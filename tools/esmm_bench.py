"""ESMM benchmark: the head kernels (b200rec_esmm_head_fwd / _bwd) against the reference's head in
torch, the pooled lookup (b200rec_gather_pool_sum and its group_ids + segment_reduce backward), and a
whole ESMMLayer training step (forward, two log-losses, backward, lazy Adam) against the reference's
op sequence (models/multitask/esmm/net.py:85-111 and dygraph_model.py:56-74: 23 per-field gathers,
sum and concat, two Linear/ReLU chains, softmax, slice, multiply, concat, two log-losses, non-lazy
Adam) restated in torch fp32 on the same GPU.

    python tools/esmm_bench.py [--Vs 737946,100000000] [--batches 1024,65536] [--json f]

Times are CUDA-event medians over --iters calls after --warmup.  Before any time is taken, the two
paths' outputs are compared at the timed size: the six head outputs and their input gradients, the
pooled lookup, and the step's loss.  Algorithmic bytes of the pooled lookup: forward B*23*3*8 (ids)
+ B*23*3*4*D (rows) + B*23*D*4 (out); backward B*23*D*4 (dout) + U*D*4 (merged rows, U touched ids).
Their share of HBM is those bytes over the time against the H100 SXM data sheet's 3.35 TB/s.
Prints the card name and power limit, then one JSON line per configuration.
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

F, L, D, FC = 23, 3, 12, [256, 64]
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


def reference_forward(p, ids):
    """esmm/net.py:85-111 in torch fp32: 23 gathers + sums, concat, two towers, the head."""
    W = p["embedding.weight"]
    emb = [(W[ids[:, f, :]] * (ids[:, f, :] != 0).unsqueeze(-1)).sum(1) for f in range(F)]
    x = torch.cat(emb, 1)
    hs = []
    for first in (0, 3):
        y = x
        for i in range(first, first + 2):
            y = torch.relu(y @ p["linear_%d.weight" % i] + p["linear_%d.bias" % i])
        hs.append(y)
    return reference_head(hs[0], hs[1], p["linear_2.weight"], p["linear_2.bias"],
                          p["linear_5.weight"], p["linear_5.bias"])


def reference_head(h_ctr, h_cvr, W_ctr, b_ctr, W_cvr, b_cvr):
    ctr_out = torch.softmax(h_ctr @ W_ctr + b_ctr, dim=-1)
    cvr_out = torch.softmax(h_cvr @ W_cvr + b_cvr, dim=-1)
    ctr_one, cvr_one = ctr_out[:, 1:2], cvr_out[:, 1:2]
    ctcvr_one = ctr_one * cvr_one
    return ctr_out, ctr_one, cvr_out, cvr_one, torch.cat([1 - ctcvr_one, ctcvr_one], 1), ctcvr_one


def reference_loss(outs, clk, buy):
    eps = 1e-4

    def ll(p, y):
        return -y * torch.log(p + eps) - (1 - y) * torch.log(1 - p + eps)

    return (ll(outs[1], clk.float()) + ll(outs[5], buy.float())).mean()


def bench(V, B, iters, warmup):
    from paddlerec_b200 import nn as bnn
    from paddlerec_b200 import ops, optim, tower
    from paddlerec_b200.multitask.esmm import dygraph_model, net
    torch.manual_seed(0)
    g = torch.Generator(device="cuda").manual_seed(5)
    ids = torch.randint(1, V, (B, F, L), device="cuda", generator=g)
    ids[torch.rand(B, F, L, device="cuda", generator=g) < 0.3] = 0
    clk = (torch.rand(B, 1, device="cuda", generator=g) < 0.3).to(torch.int64)
    buy = clk * (torch.rand(B, 1, device="cuda", generator=g) < 0.2).to(torch.int64)
    layer = net.ESMMLayer(V, D, F, FC, FC, device="cuda")
    r = {"B": B, "V": V, "D": D, "fc": FC}
    prev_tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False

    # ---- the head alone: kernels vs the reference's torch head, checked first --------------------
    K = FC[-1]
    hs = [torch.relu(torch.randn(B, K, device="cuda", generator=g)) for _ in range(2)]
    Wb = [layer._ctr_linears[-1].weight.detach(), layer._ctr_linears[-1].bias.detach(),
          layer._cvr_linears[-1].weight.detach(), layer._cvr_linears[-1].bias.detach()]
    gs = [torch.randn(B, 2 if i % 2 == 0 else 1, device="cuda", generator=g) for i in range(6)]
    outs = ops.raw_esmm_head_fwd(hs[0], hs[1], *Wb)
    leaves = [t.clone().requires_grad_(True) for t in hs]
    ref = reference_head(leaves[0], leaves[1], *Wb)
    err = max(float((a - b).detach().abs().max()) for a, b in zip(outs, ref))
    assert err <= 1e-5, ("head forward", err)
    torch.autograd.backward(ref, gs)
    dh = ops.raw_esmm_head_bwd(gs, outs[0], outs[2], hs[0], hs[1], Wb[0], Wb[2])[:2]
    for a, b in zip(dh, leaves):
        e = float((a - b.grad).abs().max() / (b.grad.abs().max() + 1e-30))
        assert e <= 1e-4, ("head backward", e)
    r["head_fwd_ms"] = timed(lambda: ops.raw_esmm_head_fwd(hs[0], hs[1], *Wb), iters, warmup)
    r["head_bwd_ms"] = timed(lambda: ops.raw_esmm_head_bwd(gs, outs[0], outs[2], hs[0], hs[1], Wb[0],
                                                           Wb[2]), iters, warmup)

    def torch_head_step():
        lv = [t.detach().requires_grad_(True) for t in hs]
        torch.autograd.backward(reference_head(lv[0], lv[1], *Wb), gs)

    r["torch_head_fwd_ms"] = timed(lambda: reference_head(hs[0], hs[1], *Wb), iters, warmup)
    r["torch_head_fwd_bwd_ms"] = timed(torch_head_step, iters, warmup)
    r["head_fwd_hbm_share"] = (2 * B * K * 4 + 9 * B * 4) / (r["head_fwd_ms"] * 1e-3) / HBM_BPS
    r["head_bwd_hbm_share"] = (4 * B * K * 4 + 13 * B * 4) / (r["head_bwd_ms"] * 1e-3) / HBM_BPS

    # ---- the pooled lookup, forward and backward, checked first ----------------------------------
    Wt = layer.embedding.weight
    keys = ids.reshape(-1)
    offsets = torch.arange(0, B * F * L + 1, L, dtype=torch.int64, device="cuda")
    pooled, bag = ops.raw_gather_pool_sum(Wt, keys, offsets, 0)
    ref_pooled = (Wt[ids] * (ids != 0).unsqueeze(-1)).sum(2).reshape(B * F, D)
    assert float((pooled - ref_pooled).abs().max()) <= 1e-5
    dout = torch.randn(B * F, D, device="cuda", generator=g)

    def pool_bwd():
        grp = ops.raw_group_ids(keys, V, 0)
        return ops.raw_segment_reduce(dout, grp.seg_offsets, grp.sorted_pos, grp.num, grp.n,
                                      row_of_pos=bag), grp

    rows, grp = pool_bwd()
    U = int(grp.num[0])
    r["pool_fwd_ms"] = timed(lambda: ops.raw_gather_pool_sum(Wt, keys, offsets, 0), iters, warmup)
    r["pool_bwd_ms"] = timed(pool_bwd, iters, warmup)
    fwd_bytes = B * F * L * (8 + 4 * D) + B * F * D * 4
    bwd_bytes = B * F * D * 4 + U * D * 4
    r.update(pool_fwd_bytes=fwd_bytes, pool_bwd_bytes=bwd_bytes, unique_ids=U,
             pool_fwd_hbm_share=fwd_bytes / (r["pool_fwd_ms"] * 1e-3) / HBM_BPS,
             pool_bwd_hbm_share=bwd_bytes / (r["pool_bwd_ms"] * 1e-3) / HBM_BPS)

    # ---- the whole step (bf16x3 towers, lazy Adam) vs the reference's op sequence ------------------
    dm = dygraph_model.DygraphModel()
    opt = optim.Adam(learning_rate=1e-3, parameters=layer.parameters(), lazy_mode=True)
    p_ref = {k: v.detach().clone() for k, v in layer.state_dict().items()}
    prev = bnn.get_matmul_precision()
    bnn.set_matmul_precision("bf16x3")
    tower.set_overlap_dw(False)
    try:
        with torch.no_grad():
            o = layer(ids)
            ours = float(dm.create_loss(o[1], clk, o[5], buy))
        theirs = float(reference_loss(reference_forward(p_ref, ids), clk, buy))
        assert abs(ours - theirs) <= 1e-4 * abs(theirs), ("step loss", ours, theirs)

        def step():
            opt.clear_grad()
            o = layer(ids)
            dm.create_loss(o[1], clk, o[5], buy).backward()
            opt.step()

        r["step_ms"] = timed(step, iters, warmup)
    finally:
        bnn.set_matmul_precision(prev)
    ref_params = {k: v.requires_grad_(True) for k, v in p_ref.items()}
    opt_ref = torch.optim.Adam(list(ref_params.values()), lr=1e-3)

    def ref_step():
        opt_ref.zero_grad(set_to_none=True)
        reference_loss(reference_forward(ref_params, ids), clk, buy).backward()
        opt_ref.step()

    r["reference_torch_fp32_step_ms"] = timed(ref_step, max(3, iters // 4), 2)
    torch.backends.cuda.matmul.allow_tf32 = prev_tf32
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--Vs", default="737946,100000000")
    ap.add_argument("--batches", default="1024,65536")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("esmm_bench needs a CUDA device")
    rows = []
    print(json.dumps({"card": card()}), flush=True)
    for V in [int(v) for v in a.Vs.split(",")]:
        for B in [int(v) for v in a.batches.split(",")]:
            r = bench(V, B, a.iters, a.warmup)
            r = {k: (round(v, 4) if isinstance(v, float) and math.isfinite(v) else v) for k, v in r.items()}
            r["card"] = card()
            print(json.dumps(r), flush=True)
            rows.append(r)
            torch.cuda.empty_cache()
    if a.json:
        with open(a.json, "w") as fh:
            json.dump({"card": card(), "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
