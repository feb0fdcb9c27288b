"""FAT-DeepFFM benchmark: the four fused kernels (b200rec_fat_ffm_pool_fwd / _fwd / _bwd_attn /
_bwd), the attention and DNN GEMMs, and a whole FAT_DeepFFMLayer training step (forward, log-loss,
backward, lazy Adam), against the reference's op sequence (models/rank/fat_deepffm/net.py: feat
[B, NF*NF, D], max pool, the attention MLP, tile/split/stack, 741 Hadamard slice pairs, the DNN,
non-lazy Adam) restated in torch on the same GPU.

    python tools/fat_deepffm_bench.py [--V 1000000] [--batches 1000,8192,65536] [--json out.json]

Times are CUDA-event medians over --iters calls after --warmup.  The step runs in train mode, as
the trainer does (dropout on, the DNN on per-layer wgmma Linears); the GEMM rows time the eval-mode
tower, forward only.  Algorithmic bytes per sample come from
the shapes (kernel_bytes below): every gathered row once per kernel that gathers it, plus the
kernel's own inputs and outputs; the kernels' share of HBM is those bytes over their time against
the H100 SXM data sheet's 3.35 TB/s.  GEMM FLOPs are 2*M*N*K per product (forward, dX and dW in a
step).  Prints one JSON line per configuration and the card name and power limit it ran on.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

F, Dn, D = 26, 13, 10
NF = F + Dn
NN, P, R = NF * NF, NF * (NF - 1) // 2, NF * D
LAYERS = [1600, 1600]
HBM_BPS = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name()


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def make_ids(B, V, dist, seed):
    if dist == "uniform":
        g = torch.Generator(device="cuda").manual_seed(seed)
        return torch.randint(0, V, (B, F), device="cuda", generator=g)
    rng = np.random.default_rng(seed)
    return torch.tensor((rng.zipf(1.05, size=(B, F)) - 1) % V, device="cuda")


def kernel_bytes(B, U):
    """Algorithmic HBM bytes of each kernel at batch B with U distinct ids (rows of R floats; the
    backward reads a partner block per position and column, counted as its row once per position)."""
    row = R * 4
    ids_b, dense_b = F * 8, Dn * 4
    return {
        "pool_fwd": B * (ids_b + dense_b + F * row + NN * 4),
        "fwd": B * (ids_b + dense_b + F * row + NN * 4 + P * D * 4 + 4),
        "bwd_attn": B * (ids_b + dense_b + F * row + NN * 4 + 4 + P * D * 4 + NN * 4),
        "bwd": B * (ids_b + dense_b + F * row + 2 * NN * 4 + 4 + P * D * 4) + U * (row + 4) * 2,
    }


def gemm_flops(B):
    """(attention forward, DNN forward) FLOPs; a training step does 3x each (forward, dX, dW)."""
    att = 2 * B * NN * NN * 2
    sizes = [P * D] + LAYERS + [1]
    dnn = sum(2 * B * sizes[i] * sizes[i + 1] for i in range(len(sizes) - 1))
    return att, dnn


def bench_ours(V, B, dist, iters, warmup):
    from paddlerec_b200 import functional as BF
    from paddlerec_b200 import nn as bnn
    from paddlerec_b200 import ops, optim, tower
    from paddlerec_b200.rank.fat_deepffm import net
    bnn.set_matmul_precision("bf16x3")
    torch.manual_seed(0)
    layer = net.FAT_DeepFFMLayer(V, D, Dn, F, LAYERS, device="cuda")
    with torch.no_grad():   # off the saturating Constant(1.0), so the step carries gradient
        layer.cen.dense_w.normal_(0, 0.05)
    opt = optim.Adam(learning_rate=1e-4, parameters=layer.parameters())
    ids = make_ids(B, V, dist, 1)
    g = torch.Generator(device="cuda").manual_seed(2)
    dense = torch.rand(B, Dn, device="cuda", generator=g)
    label = (torch.rand(B, 1, device="cuda", generator=g) < 0.3).float()

    def step():
        opt.clear_grad()
        pred = layer(ids, dense)
        BF.log_loss_mean(pred, label).backward()
        opt.step()
    step_ms = timed(step, iters, warmup)

    W = layer.cen._fused.weight.detach()
    dw = layer.cen.dense_w.detach().reshape(Dn, R)
    pad = layer.cen._fused.pad
    pool = ops.raw_fat_ffm_pool_fwd(W, ids, dense, dw, pad, D)
    attn = torch.relu(torch.randn(B, NN, device="cuda", generator=g))
    gy1 = torch.randn(B, device="cuda", generator=g)
    dh = torch.randn(B, P * D, device="cuda", generator=g)
    dpool = torch.randn(B, NN, device="cuda", generator=g)
    groups = ops.raw_group_ids(ids, V, pad)
    U = int(groups.num[0])
    t = {
        "pool_fwd": timed(lambda: ops.raw_fat_ffm_pool_fwd(W, ids, dense, dw, pad, D), iters, warmup),
        "fwd": timed(lambda: ops.raw_fat_ffm_fwd(W, ids, dense, dw, attn, None, pad, D), iters, warmup),
        "bwd_attn": timed(lambda: ops.raw_fat_ffm_bwd_attn(W, ids, dense, dw, attn, gy1, dh, pad, D),
                          iters, warmup),
        "bwd": timed(lambda: ops.raw_fat_ffm_bwd(W, ids, dense, dw, attn, gy1, dh, dpool,
                                                 ops.raw_group_ids(ids, V, pad), pad, D),
                     iters, warmup),
    }
    fc = (layer.cen.fc.ReductionLinear, layer.cen.fc.AdditionLinear)
    lin = [m for m in layer.dnn._mlp_layers if isinstance(m, bnn.Linear)]
    h = torch.randn(B, P * D, device="cuda", generator=g)
    with torch.no_grad():
        t["attn_gemms_fwd"] = timed(lambda: tower.mlp(pool, [m.weight for m in fc],
                                                      [m.bias for m in fc], last_act=True),
                                    iters, warmup)
        t["dnn_gemms_fwd"] = timed(lambda: tower.mlp(h, [m.weight for m in lin],
                                                     [m.bias for m in lin]), iters, warmup)
    bnn.set_matmul_precision("fp32")
    kb = kernel_bytes(B, U)
    att, dnn = gemm_flops(B)
    kern_ms = sum(t[k] for k in kb)
    out = {"B": B, "dist": dist, "V": V, "D": D, "unique_ids": U,
           "step_ms": step_ms, "samples_per_s": B / (step_ms * 1e-3),
           "kernels_ms": {k: round(v, 4) for k, v in t.items()},
           "kernel_hbm_share": {k: round(kb[k] / (t[k] * 1e-3) / HBM_BPS, 3) for k in kb},
           "kernels_share_of_step": round(kern_ms / step_ms, 3),
           "attn_gemm_tflops": round(att / (t["attn_gemms_fwd"] * 1e-3) / 1e12, 1),
           "dnn_gemm_tflops": round(dnn / (t["dnn_gemms_fwd"] * 1e-3) / 1e12, 1),
           "step_gemm_tflop": round(3 * (att + dnn) / 1e12, 3)}
    del layer, opt
    torch.cuda.empty_cache()
    return out


def bench_reference(V, B, dist, iters, warmup):
    """The reference's op sequence in torch (fp32, cuBLAS GEMMs, autograd), one training step with
    non-lazy Adam over every parameter, the [V, NF*D] table included (dygraph_model.py:61-65)."""
    torch.manual_seed(0)
    dev = "cuda"
    std = 0.1 / np.sqrt(D)
    emb = torch.nn.Parameter(torch.randn(V, R, device=dev) * std)
    dense_w = torch.nn.Parameter(torch.randn(1, Dn, R, device=dev) * 0.05)
    fc = torch.nn.Sequential(torch.nn.Linear(NN, NN), torch.nn.ReLU(), torch.nn.Linear(NN, NN),
                             torch.nn.ReLU()).to(dev)
    sizes = [P * D] + LAYERS + [1]
    mods = []
    for i in range(len(sizes) - 1):
        mods.append(torch.nn.Linear(sizes[i], sizes[i + 1]))
        if i < len(sizes) - 2:
            mods.append(torch.nn.ReLU())
    dnn = torch.nn.ModuleList(mods).to(dev)
    bias = torch.nn.Parameter(torch.zeros(1, device=dev))
    drop = torch.nn.Dropout(0.5)
    params = [emb, dense_w, bias] + list(fc.parameters()) + list(dnn.parameters())
    opt = torch.optim.Adam(params, lr=1e-4)
    ids = make_ids(B, V, dist, 1)
    g = torch.Generator(device=dev).manual_seed(2)
    dense = torch.rand(B, Dn, device=dev, generator=g)
    label = (torch.rand(B, 1, device=dev, generator=g) < 0.3).float()

    def step():
        opt.zero_grad(set_to_none=True)
        feat = torch.cat([emb[ids], dense.unsqueeze(2) * dense_w], 1).reshape(-1, NN, D)
        pooled = torch.nn.functional.adaptive_max_pool1d(feat, 1).flatten(1)
        a = fc(pooled)
        a = torch.stack(torch.split(a.repeat(1, D), NN, 1), 2)
        outputs = feat * a
        y1 = outputs.sum(2).sum(1, keepdim=True)
        fa = outputs.reshape(-1, NF, NF, D)
        terms = [fa[:, i, j, :] * fa[:, j, i, :] for i in range(NF) for j in range(i + 1, NF)]
        y = torch.cat(terms, 1)
        for m in dnn:
            y = drop(m(y))
        pred = torch.sigmoid(y1 + y + bias)
        eps = 1e-4
        loss = (-label * torch.log(pred + eps) - (1 - label) * torch.log(1 - pred + eps)).mean()
        loss.backward()
        opt.step()
    ms = timed(step, iters, warmup)
    del emb, opt, params
    torch.cuda.empty_cache()
    return {"B": B, "dist": dist, "V": V, "D": D, "reference_step_ms": ms,
            "reference_samples_per_s": B / (ms * 1e-3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--V", type=int, default=1_000_000)
    ap.add_argument("--batches", default="1000,8192,65536")
    ap.add_argument("--ref-batches", default="1000,8192")
    ap.add_argument("--dists", default="uniform,zipf")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fat_deepffm_bench needs a CUDA device")
    rows = []
    info = card()
    print("card:", info, flush=True)
    for B in (int(x) for x in a.batches.split(",")):
        for dist in a.dists.split(","):
            r = bench_ours(a.V, B, dist, a.iters, a.warmup)
            r["card"] = info
            print(json.dumps(r), flush=True)
            rows.append(r)
    for B in (int(x) for x in a.ref_batches.split(",") if x):
        for dist in a.dists.split(","):
            r = bench_reference(a.V, B, dist, max(3, a.iters // 4), 2)
            r["card"] = info
            print(json.dumps(r), flush=True)
            rows.append(r)
    if a.json:
        with open(a.json, "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
