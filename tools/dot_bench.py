#!/usr/bin/env python
"""K6 (DLRM dot interaction) and the feasign fold, timed alone: CUDA events around `iters` launches
after warm-up, over a ring of inputs larger than L2 (50 MB) so every launch reads from HBM.
Reports algorithmic GB/s: forward 4*(N*d + d + P) B/sample, backward 4*(2*N*d + d + P),
hash_keys 16 (+4 with slots) B/key; the library formulation (bmm + triu gather + cat) beside it."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from paddlerec_b200 import ops  # noqa: E402


def timed(fn, n_ring, iters, warmup=3):
    for i in range(warmup):
        fn(i % n_ring)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        fn(i % n_ring)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=65536)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--v2", action="store_true", help="time the experimental B200REC_K6_V2 kernels")
    a = ap.parse_args()
    if a.v2:
        os.environ["B200REC_K6_V2"] = "1"
    dev = "cuda"
    peak = None
    mp = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(mp):
        try:
            peak = json.load(open(mp)).get("hbm_gbs")
        except Exception:
            peak = None
    for N, d in ((27, 16), (27, 64), (27, 128)):
        P = N * (N - 1) // 2
        ring = max(2, int(300e6 // (a.B * N * d * 4)) + 1)
        Ts = [torch.randn(a.B, N, d, device=dev) for _ in range(ring)]
        dRs = [torch.randn(a.B, d + P, device=dev) for _ in range(min(ring, 4))]
        iu = torch.triu_indices(N, N, 1, device=dev)
        ms_f = timed(lambda i: ops.raw_dot_interact_fwd(Ts[i]), ring, a.iters)
        ms_b = timed(lambda i: ops.raw_dot_interact_bwd(Ts[i], dRs[i % len(dRs)]), ring, a.iters)

        def lib_fwd(i):
            Z = torch.bmm(Ts[i], Ts[i].transpose(1, 2))
            return torch.cat([Ts[i][:, N - 1], Z[:, iu[0], iu[1]]], 1)
        ms_l = timed(lib_fwd, ring, a.iters)
        bf, bb = 4 * (N * d + d + P) * a.B, 4 * (2 * N * d + d + P) * a.B
        row = {"kernel": "dot_interact_v2" if a.v2 else "dot_interact", "B": a.B, "N": N, "d": d, "fwd_ms": round(ms_f, 4),
               "bwd_ms": round(ms_b, 4), "fwd_GBps": round(bf / ms_f / 1e6, 1),
               "bwd_GBps": round(bb / ms_b / 1e6, 1), "library_fwd_ms": round(ms_l, 4),
               "fwd_bytes": bf, "bwd_bytes": bb}
        if peak:
            row["fwd_frac"], row["bwd_frac"] = round(bf / ms_f / 1e6 / peak, 3), round(bb / ms_b / 1e6 / peak, 3)
        print(json.dumps(row), flush=True)
        del Ts, dRs
    n = a.B * 26 * 8
    ring = 4
    keys = [torch.randint(0, 1 << 62, (n,), device=dev) for _ in range(ring)]
    slots = (torch.arange(n, device=dev) % 26).to(torch.int32)
    for sl in (None, slots):
        ms = timed(lambda i: ops.raw_hash_keys(keys[i], 100_000_000, sl), ring, a.iters)
        by = n * (16 + (4 if sl is not None else 0))
        row = {"kernel": "hash_keys", "n": n, "slots": sl is not None, "ms": round(ms, 4),
               "GBps": round(by / ms / 1e6, 1)}
        if peak:
            row["frac"] = round(by / ms / 1e6 / peak, 3)
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
