"""FFM benchmark: the fused kernels (b200rec_ffm_fwd / _bwd, lazy Adam on the wide fused rows) and a
whole FFMLayer training step, against the reference's op sequence (models/rank/ffm/net.py:99-133,
741 slice-multiply-sum pairs + add_n, non-lazy Adam) restated in torch on the same GPU.

    python tools/ffm_bench.py [--V 1000000] [--dims 9,16] [--batches 4096,65536] [--json out.json]

Times are CUDA-event medians over --iters calls after --warmup.  Algorithmic forward bytes per sample
are F*8 (ids) + Dn*4 (dense) + F*4*(R+1) (rows with w1) + 8 (y1, y2); the forward's share of HBM
bandwidth is those bytes over its time against the H100 SXM data sheet's 3.35 TB/s.  Prints one
JSON line per configuration and the card name and power limit it ran on.
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

F, Dn = 26, 13
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


def bench_ours(V, D, B, dist, iters, warmup):
    from paddlerec_b200 import functional as BF
    from paddlerec_b200 import ops, optim
    from paddlerec_b200.rank.ffm import net
    torch.manual_seed(0)
    layer = net.FFMLayer(V, D, Dn, F + Dn, device="cuda")
    with torch.no_grad():   # the reference's constant 1.0 saturates the sigmoid
        layer.ffm.dense_w.normal_(0, 0.05)
        layer.ffm.dense_w_one.normal_(0, 0.05)
    ids = make_ids(B, V, dist, 1)
    dense = torch.rand(B, Dn, device="cuda")
    label = (torch.rand(B, 1, device="cuda") < 0.3).float()
    opt = optim.Adam(learning_rate=1e-3, parameters=layer.parameters())
    fm = layer.ffm
    W = fm._fused.weight.detach()
    R = (F + Dn) * D
    dw = fm.dense_w.detach().reshape(Dn, R)
    g1 = torch.randn(B, device="cuda") * 1e-3
    out = {}
    out["fwd_ms"] = timed(lambda: ops.raw_ffm_fwd(W, ids, dense, dw, fm.dense_w_one.detach(),
                                                  layer.bias.detach(), -1, D), iters, warmup)

    def bwd():
        groups = ops.raw_group_ids(ids, V, -1)
        return groups, ops.raw_ffm_bwd(W, ids, dense, dw, g1, g1, groups, -1, D)
    out["bwd_ms"] = timed(bwd, iters, warmup)
    groups, (dW, *_rest) = bwd()
    out["unique_rows"] = int(groups.num[0])
    sr = ops.SelectedRows(groups.unique_ids, dW, groups.num, V, ncols=ops.fused_grad_cols(R))
    m, v = opt.moments(fm._fused.weight)
    out["adam_ms"] = timed(lambda: ops.raw_sparse_adam(W, m, v, sr, 1e-9, 0.9, 0.999, 1e-8, 0.9,
                                                       0.999), iters, warmup)

    def step():
        opt.clear_grad()
        BF.log_loss_mean(layer(ids, dense), label).backward()
        opt.step()
    out["step_ms"] = timed(step, iters, warmup)
    out["samples_per_s"] = B / (out["step_ms"] * 1e-3)
    fwd_bytes = B * (F * 8 + Dn * 4 + F * 4 * (R + 1) + 8)
    out["fwd_bytes"] = fwd_bytes
    out["fwd_hbm_share"] = fwd_bytes / (out["fwd_ms"] * 1e-3) / HBM_BPS
    del layer, opt, m, v, sr, dW
    torch.cuda.empty_cache()
    return out


def bench_reference(V, D, B, dist, iters, warmup):
    """net.py:99-133 op for op (embedding gathers, 741 slice * slice -> sum, add_n), sigmoid,
    log_loss mean, and paddle's default non-lazy Adam over every parameter (dense gradients)."""
    NF, R = F + Dn, (F + Dn) * D
    emb = torch.nn.Embedding(V, R).cuda()
    emb1 = torch.nn.Embedding(V, 1).cuda()
    dense_w1 = torch.nn.Parameter(torch.randn(Dn, device="cuda") * 0.05)
    dense_w = torch.nn.Parameter(torch.randn(1, Dn, R, device="cuda") * 0.05)
    bias = torch.nn.Parameter(torch.zeros(1, device="cuda"))
    params = list(emb.parameters()) + list(emb1.parameters()) + [dense_w1, dense_w, bias]
    opt = torch.optim.Adam(params, lr=1e-3)
    ids = make_ids(B, V, dist, 1)
    dense = torch.rand(B, Dn, device="cuda")
    label = (torch.rand(B, 1, device="cuda") < 0.3).float()

    def step():
        opt.zero_grad(set_to_none=True)
        y1 = emb1(ids).sum(1) + (dense * dense_w1).unsqueeze(2).sum(1)
        feat = torch.cat([emb(ids), dense.unsqueeze(2) * dense_w], 1).reshape(-1, NF, NF, D)
        terms = [(feat[:, i, j, :] * feat[:, j, i, :]).sum(1, keepdim=True)
                 for i in range(NF) for j in range(i + 1, NF)]
        pred = torch.sigmoid(y1 + torch.stack(terms, 0).sum(0) + bias)
        eps = 1e-4
        loss = (-label * torch.log(pred + eps) - (1 - label) * torch.log(1 - pred + eps)).mean()
        loss.backward()
        opt.step()
    ms = timed(step, iters, warmup)
    del emb, emb1, opt
    torch.cuda.empty_cache()
    return {"ref_step_ms": ms, "ref_samples_per_s": B / (ms * 1e-3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--V", type=int, default=1_000_000)
    ap.add_argument("--dims", default="9,16")
    ap.add_argument("--batches", default="4096,65536")
    ap.add_argument("--dists", default="uniform,zipf")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ref-max-batch", type=int, default=4096,
                    help="largest batch for the reference op sequence: each of its 1,482 slice "
                         "backwards allocates a zero tensor the size of feat [B, 39, 39*D]")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ffm_bench needs a CUDA device")
    info = card()
    print("card:", info, flush=True)
    rows = []
    for D in (int(x) for x in a.dims.split(",")):
        for B in (int(x) for x in a.batches.split(",")):
            for dist in a.dists.split(","):
                r = {"V": a.V, "D": D, "B": B, "ids": dist, "card": info}
                r.update(bench_ours(a.V, D, B, dist, a.iters, a.warmup))
                if B <= a.ref_max_batch:
                    r.update(bench_reference(a.V, D, B, dist, max(3, a.iters // 5), 1))
                rows.append(r)
                print(json.dumps(r), flush=True)
    if a.json:
        with open(a.json, "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
