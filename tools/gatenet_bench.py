"""GateNet benchmark: the embedding-gate kernels (b200rec_gate_embed_fwd / _bwd), the gated versus the
ungated wgmma tower, and a whole GateDNNLayer training step (forward, log-loss, backward, lazy Adam),
against the reference's op sequence (models/rank/gatenet/net.py:85-121: 26 per-field gathers, gate
multiply/sum/sigmoid/multiply, concat, Linear/ReLU and tanh(matmul)/multiply per layer, non-lazy
Adam) restated in torch fp32 on the same GPU.

    python tools/gatenet_bench.py [--V 1000000] [--batches 4096,65536] [--fc 512,256,256] [--json f]

Times are CUDA-event medians over --iters calls after --warmup.  Algorithmic bytes: forward
B*F*(8 + 4*D) (ids, rows) + B*Dn*4 (dense) + B*(F*D + Dn)*4 (output); backward B*F*(8 + 4*D)
(ids, re-gathered rows) + B*F*D*4 (dout) + B*F*D*4 (per-position rows).  Their share of HBM is
those bytes over the time against the H100 SXM data sheet's 3.35 TB/s.  Tower FLOPs are 2*M*K*N per
fp32 GEMM of the forward (3x for forward + dX + dW), counted once, not per bf16 plane.  Prints one
JSON line per configuration and the card name and power limit it ran on.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

F, Dn, D = 26, 13, 9
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


def tower_flops(B, fc, gated):
    sizes = [F * D + Dn] + fc + [1]
    f = sum(2 * B * sizes[i] * sizes[i + 1] for i in range(len(sizes) - 1))
    if gated:
        f += sum(2 * B * n * n for n in fc)
    return f


def reference_step(layer, ids, dense, label, opt_ref):
    """gatenet/net.py:85-121 and a non-lazy Adam, in torch fp32 (TF32 off)."""
    p = dict(layer.named_parameters())
    W = layer.embedding.weight
    embs = []
    for i in range(F):
        e = W[ids[:, i]]
        gate = (e * p["embedding_gate_weight_%d" % i]).sum(-1, keepdim=True)
        embs.append(e * torch.sigmoid(gate))
    y = torch.cat(embs + [dense], 1)
    n = len(layer._hidden_gate_weight)
    for i in range(n):
        y = torch.relu(y @ p["linear_%d.weight" % i] + p["linear_%d.bias" % i])
        y = y * torch.tanh(y @ p["hidden_gate_weight_%d" % i])
    pred = torch.sigmoid(y @ p["last_layer.weight"] + p["last_layer.bias"])
    eps = 1e-4
    loss = (-label * torch.log(pred + eps) - (1 - label) * torch.log(1 - pred + eps)).mean()
    opt_ref.zero_grad(set_to_none=True)
    loss.backward()
    opt_ref.step()


def bench(V, B, fc, dist, iters, warmup):
    from paddlerec_b200 import functional as BF
    from paddlerec_b200 import nn as bnn
    from paddlerec_b200 import ops, optim, tower
    from paddlerec_b200.rank.gatenet import net
    torch.manual_seed(0)
    ids = make_ids(B, V, dist, 5)
    dense = torch.rand(B, Dn, device="cuda")
    label = (torch.rand(B, 1, device="cuda") < 0.3).float()
    layer = net.GateDNNLayer(V, D, Dn, F, fc, True, True, device="cuda")
    gw = torch.cat(layer.embedding_gate_weight).detach()
    W = layer.embedding.weight
    r = {"B": B, "V": V, "D": D, "fc": fc, "ids": dist}
    t_fwd = timed(lambda: ops.raw_gate_embed_fwd(W, ids, gw, dense, D), iters, warmup)
    dout = torch.randn(B, F * D + Dn, device="cuda")
    t_bwd = timed(lambda: ops.raw_gate_embed_bwd(W, ids, gw, dout, D), iters, warmup)
    fwd_bytes = B * F * (8 + 4 * D) + B * Dn * 4 + B * (F * D + Dn) * 4
    bwd_bytes = B * F * (8 + 4 * D) + 2 * B * F * D * 4
    r.update(gate_embed_fwd_ms=t_fwd, gate_embed_fwd_hbm_share=fwd_bytes / (t_fwd * 1e-3) / HBM_BPS,
             gate_embed_bwd_ms=t_bwd, gate_embed_bwd_hbm_share=bwd_bytes / (t_bwd * 1e-3) / HBM_BPS)
    # tower alone, gated vs ungated, on the same input
    x = torch.randn(B, F * D + Dn, device="cuda", requires_grad=True)
    lin = [m for m in layer._mlp_layers if isinstance(m, bnn.Linear)]
    Ws = [m.weight for m in lin] + [layer.last_layer.weight]
    bs = [m.bias for m in lin] + [layer.last_layer.bias]
    dy = torch.randn(B, 1, device="cuda")
    for gated in (False, True):
        gates = layer._hidden_gate_weight if gated else None
        tf = timed(lambda: tower.mlp(x, Ws, bs, gates=gates), iters, warmup)
        tfb = timed(lambda: tower.mlp(x, Ws, bs, gates=gates).backward(dy), iters, warmup)
        fl = tower_flops(B, fc, gated)
        key = "tower_gated" if gated else "tower_ungated"
        r[key + "_fwd_ms"], r[key + "_fwd_tflops"] = tf, fl / (tf * 1e-3) / 1e12
        r[key + "_bwd_ms"] = tfb - tf
        r[key + "_bwd_tflops"] = 2 * fl / ((tfb - tf) * 1e-3) / 1e12
    # whole step, split into its parts
    opt = optim.Adam(learning_rate=1e-3, parameters=layer.parameters(), lazy_mode=True)
    prev = bnn.get_matmul_precision()
    bnn.set_matmul_precision("bf16x3")
    tower.set_overlap_dw(False)
    try:
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
        parts = []
        for it in range(warmup + iters):
            opt.clear_grad()
            ev[0].record()
            pred = layer(ids, dense)
            ev[1].record()
            loss = BF.log_loss_mean(pred, label)
            ev[2].record()
            loss.backward()
            ev[3].record()
            opt.step()
            ev[4].record()
            ev[4].synchronize()
            if it >= warmup:
                parts.append([ev[i].elapsed_time(ev[i + 1]) for i in range(4)])
        med = np.median(np.array(parts), 0)
        r.update(step_fwd_ms=med[0], step_loss_ms=med[1], step_bwd_ms=med[2], step_adam_ms=med[3],
                 step_ms=float(med.sum()))
    finally:
        bnn.set_matmul_precision(prev)
    # "before": the reference's op sequence in torch fp32 (TF32 off), non-lazy Adam, same card
    prev_tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        ref_params = [p for p in layer.parameters()]
        layer.embedding.weight.requires_grad_(True)
        opt_ref = torch.optim.Adam(ref_params, lr=1e-3)
        r["reference_torch_fp32_step_ms"] = timed(
            lambda: reference_step(layer, ids, dense, label, opt_ref), max(3, iters // 4), 2)
        layer.embedding.weight.requires_grad_(False)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev_tf32
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--V", type=int, default=1_000_000)
    ap.add_argument("--batches", default="4096,65536")
    ap.add_argument("--fc", default="512,256,256")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gatenet_bench needs a CUDA device")
    fc = [int(v) for v in a.fc.split(",")]
    rows = []
    print(json.dumps({"card": card()}))
    for B in [int(v) for v in a.batches.split(",")]:
        for dist in ("uniform", "zipf1.05"):
            r = bench(a.V, B, fc, dist, a.iters, a.warmup)
            r = {k: (round(v, 4) if isinstance(v, float) and math.isfinite(v) else v) for k, v in r.items()}
            print(json.dumps(r), flush=True)
            rows.append(r)
            torch.cuda.empty_cache()
    if a.json:
        with open(a.json, "w") as fh:
            json.dump({"card": card(), "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
