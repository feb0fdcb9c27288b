#!/usr/bin/env python
"""Micro-benchmarks of the HBM-bound kernels through the C ABI (CUDA events, rotating inputs).

    python tools/kernel_sweep.py [--quick]
Prints one JSON line per (kernel, V, D, distribution): time, algorithmic GB/s, fraction of the
measured HBM peak.  Used for BASELINE config 5 (W&D gather sweep).
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from paddlerec_b200 import ops  # noqa: E402

PEAK = 6564.5
if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")):
    PEAK = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])


def ids_for(B, F, V, dist, g):
    if dist == "zipf":
        r = torch.rand(B, F, generator=g, dtype=torch.float64)
        ids = (float(V) ** r).to(torch.int64).clamp_(1, V - 1)
    else:
        ids = torch.randint(1, V, (B, F), generator=g)
    ids[torch.rand(B, F, generator=g) < 0.02] = 0
    return ids


def time_it(fn, nrot, iters=20, warm=3):
    for i in range(warm):
        fn(i % nrot)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        fn(i % nrot)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--B", type=int, default=65536)
    args = ap.parse_args()
    dev = "cuda"
    B, F, Dn = args.B, 26, 13
    g = torch.Generator().manual_seed(12345)
    Vs = [1_000_000, 100_000_000] if args.quick else [1_000_000, 10_000_000, 100_000_000]
    Ds = [16, 64] if args.quick else [16, 64, 128]
    for D in Ds:
        for V in Vs:
            if V * D * 4 > 120e9:
                continue
            W = torch.empty(V, D, device=dev).uniform_(-0.05, 0.05)
            W1 = torch.empty(V, 1, device=dev).uniform_(-0.05, 0.05)
            dw = torch.randn(Dn, D, device=dev) * 0.05
            dw1 = torch.randn(Dn, device=dev) * 0.05
            for dist in ("uniform", "zipf"):
                nrot = 4
                idl = [ids_for(B, F, V, dist, g).to(dev) for _ in range(nrot)]
                den = [torch.rand(B, Dn, generator=g).to(dev) for _ in range(nrot)]
                # fused DeepFM forward
                ms = time_it(lambda i: ops.raw_embed_fm_fwd(W, W1, idl[i], den[i], dw, dw1, 0), nrot)
                alg = B * (F * 8 + Dn * 4 + F * 4 * D + F * 4 + (F + Dn) * 4 * D + 8)
                print(json.dumps({"kernel": "embed_fm_fwd", "V": V, "D": D, "dist": dist, "ms": ms,
                                  "GBps": alg / ms / 1e6, "frac": alg / ms / 1e6 / PEAK}), flush=True)
                if D + 1 <= 32:   # fused slot layout [D emb | w1 | pad] (128-byte rows)
                    Wf = torch.zeros(V, 32, device=dev)
                    Wf[:, :D] = W
                    Wf[:, D] = W1[:, 0]
                    msf = time_it(lambda i: ops.raw_embed_fm_fwd(Wf, None, idl[i], den[i], dw, dw1,
                                                                 0, D=D), nrot)
                    print(json.dumps({"kernel": "embed_fm_fwd_fused_slots", "V": V, "D": D,
                                      "dist": dist, "ms": msf, "GBps": alg / msf / 1e6,
                                      "frac": alg / msf / 1e6 / PEAK}), flush=True)
                    # lazy Adam: two tables vs one slot table
                    gr = ops.raw_group_ids(idl[0], V, 0)
                    n = B * F
                    gW = torch.randn(n, D, device=dev)
                    gW1 = torch.randn(n, 1, device=dev)
                    gF = torch.randn(n, ops.fused_grad_cols(D), device=dev)
                    m0, v0 = torch.zeros_like(W), torch.zeros_like(W)
                    m1, v1 = torch.zeros_like(W1), torch.zeros_like(W1)
                    mf, vf = torch.zeros_like(Wf), torch.zeros_like(Wf)
                    srW = ops.SelectedRows(gr.unique_ids, gW, gr.num, V)
                    srW1 = ops.SelectedRows(gr.unique_ids, gW1, gr.num, V)
                    srF = ops.SelectedRows(gr.unique_ids, gF, gr.num, V, ncols=gF.shape[1])
                    hp = (1e-3, 0.9, 0.999, 1e-8, 0.9, 0.999)

                    def two(i):
                        ops.raw_sparse_adam(W, m0, v0, srW, *hp)
                        ops.raw_sparse_adam(W1, m1, v1, srW1, *hp)
                    ms2 = time_it(two, 1)
                    ms1 = time_it(lambda i: ops.raw_sparse_adam(Wf, mf, vf, srF, *hp), 1)
                    print(json.dumps({"kernel": "lazy_adam_two_tables", "V": V, "D": D,
                                      "dist": dist, "ms": ms2}), flush=True)
                    print(json.dumps({"kernel": "lazy_adam_fused_slots", "V": V, "D": D,
                                      "dist": dist, "ms": ms1}), flush=True)
                    del Wf, mf, vf, m0, v0, gW, gF
                # plain gather (Wide&Deep sweep, BASELINE config 5)
                ms = time_it(lambda i: ops.raw_gather(W, idl[i], -1), nrot)
                alg = B * F * (8 + 2 * 4 * D)
                print(json.dumps({"kernel": "gather", "V": V, "D": D, "dist": dist, "ms": ms,
                                  "GBps": alg / ms / 1e6, "frac": alg / ms / 1e6 / PEAK}), flush=True)
                # backward: grouping + fused FM backward (no dfeat from the tower here)
                feat, y1, y2, S = ops.raw_embed_fm_fwd(W, W1, idl[0], den[0], dw, dw1, 0)
                dfe = torch.randn_like(feat)
                gy = torch.randn(B, device=dev)
                ms_g = time_it(lambda i: ops.raw_group_ids(idl[i], V, 0), nrot)
                gr = ops.raw_group_ids(idl[0], V, 0)
                ms_b = time_it(lambda i: ops.raw_embed_fm_bwd(feat, S, dfe, gy, gy, den[0],
                                                              gr.seg_offsets, gr.sorted_pos, gr.num,
                                                              F), 1)
                alg = B * (F * 8 + (F + Dn) * 4 * D + F * 4 * D + F * 2 * 4 * D)
                print(json.dumps({"kernel": "group_ids", "V": V, "D": D, "dist": dist, "ms": ms_g}),
                      flush=True)
                print(json.dumps({"kernel": "embed_fm_bwd", "V": V, "D": D, "dist": dist,
                                  "ms": ms_b, "GBps": alg / ms_b / 1e6,
                                  "frac": alg / ms_b / 1e6 / PEAK}), flush=True)
                del feat, dfe
            del W, W1
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
