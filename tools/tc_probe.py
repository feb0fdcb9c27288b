"""Bring-up probe for the wgmma GEMMs: every stage runs in its own process (a pipeline watchdog
trap kills the CUDA context), prints max relative error vs fp64 and kernel time.

    python tools/tc_probe.py            # all stages
    python tools/tc_probe.py fwd        # one stage in-process
"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _err(got, want):
    return float((got.double().cpu() - want.cpu()).abs().max() / (want.abs().max() + 1e-30))


def _join(planes, n):
    ld = planes.shape[1] // 2
    p = planes.double()
    return p[:, :n] + p[:, ld:ld + n]


def _time(fn, iters=10, warmup=1, repeats=1):
    """ms per call: median over `repeats` windows of `iters` back-to-back calls, after `warmup`."""
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(repeats):
        t0 = torch.cuda.Event(enable_timing=True)
        t1 = torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(iters):
            fn()
        t1.record()
        torch.cuda.synchronize()
        ts.append(t0.elapsed_time(t1) / iters)
    return sorted(ts)[len(ts) // 2]


def _card():
    """Device name and power limit, read next to the numbers they qualify."""
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                            "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = "nvidia-smi unavailable"
    return "%s, power limit / max SM clock: %s" % (torch.cuda.get_device_name(), q)


def stage(name, arg):
    import torch
    from paddlerec_b200 import ops
    dev = "cuda"
    g = torch.Generator().manual_seed(1)
    out = {"stage": name, "arg": arg}
    if name in ("fwd", "dx") and arg:
        ops.tc_debug(4, int(arg))
    if name == "fwd":
        for (M, N, K) in [(256, 64, 64), (257, 400, 624), (4096, 400, 400), (300, 1, 400)]:
            x = torch.randn(M, K, generator=g)
            W = torch.randn(K, N, generator=g) / K ** 0.5
            b = torch.randn(N, generator=g) * 0.1
            a = ops.raw_tc_split(x.to(dev))
            _, WTp = ops.raw_tc_prep_weight(W.to(dev))
            y, yp = ops.raw_tc_linear_fwd(a, K, WTp, N, b.to(dev), True, True, True)
            torch.cuda.synchronize()
            want = (x.double() @ W.double() + b.double()).clamp_min(0)
            out["%dx%dx%d" % (M, N, K)] = [_err(y, want), _err(_join(yp, N), want)]
    elif name == "dx":
        for (M, K, N) in [(256, 64, 64), (257, 624, 400), (4096, 400, 400)]:
            gy = torch.randn(M, N, generator=g)
            W = torch.randn(K, N, generator=g) / N ** 0.5
            act = torch.randn(M, K, generator=g).clamp_min(0)
            gp, _ = ops.raw_tc_split_bwd(gy.to(dev), None)
            Wp, _ = ops.raw_tc_prep_weight(W.to(dev))
            ap = ops.raw_tc_split(act.to(dev))
            dx, dxp, db = ops.raw_tc_linear_bwd_dx(gp, N, Wp, K, ap, True, True, True)
            torch.cuda.synchronize()
            want = (gy.double() @ W.double().t()) * (act.double() > 0)
            out["%dx%dx%d" % (M, K, N)] = [_err(dx, want), _err(_join(dxp, K), want),
                                            _err(db, want.sum(0))]
    elif name == "dw":
        if arg:
            lbo_a, lbo_b, sbo = (int(v) for v in arg.split(","))
            ops.tc_debug(1, lbo_a); ops.tc_debug(2, lbo_b); ops.tc_debug(3, sbo)
        for (M, K, N) in [(64, 128, 64), (256, 128, 208), (257, 624, 400), (8192, 400, 400)]:
            a = torch.randn(M, K, generator=g)
            gy = torch.randn(M, N, generator=g)
            ap = ops.raw_tc_split(a.to(dev))
            gp, _ = ops.raw_tc_split_bwd(gy.to(dev), None)
            dW = ops.raw_tc_linear_bwd_dw(ap, K, gp, N)
            torch.cuda.synchronize()
            out["%dx%dx%d" % (M, K, N)] = _err(dW, a.double().t() @ gy.double())
    elif name == "perf":
        # the K-major calls of bench.py's DeepFM tower at its batch: forward 624->400 and 400->400
        # (bias, ReLU, planes, column of ones), dX into masked planes at output widths 400 and
        # 624, dX into fp32 at 624 (the gradient of the tower input); plus the dW kernel
        M = 65536
        out["card"] = _card()
        res = {}
        tm = dict(iters=20, warmup=3, repeats=5)
        for (K, N) in [(624, 400), (400, 400)]:
            x = torch.randn(M, K, device=dev)
            W = torch.randn(K, N, device=dev) / K ** 0.5
            b = torch.randn(N, device=dev) * 0.1
            a = ops.raw_tc_split(x)
            Wp, WTp = ops.raw_tc_prep_weight(W)
            gp, _ = ops.raw_tc_split_bwd(torch.randn(M, N, device=dev), None)
            fl = 3 * 2.0 * M * K * N
            for bn in ([0] if not arg else [int(v) for v in arg.split(",")]):
                ops.tc_debug(0, bn)
                for bk in (64, 32):
                    ops.tc_debug(4, bk)
                    tag = "%dx%d bn%d bk%d" % (K, N, bn, bk)
                    t = _time(lambda: ops.raw_tc_linear_fwd(a, K, WTp, N, b, True, False, True,
                                                            ones_col=True), **tm)
                    res["fwd " + tag] = [round(t, 4), round(fl / t / 1e9, 1)]
                    t = _time(lambda: ops.raw_tc_linear_bwd_dx(gp, N, Wp, K, a, False, True, False),
                              **tm)
                    res["dx  " + tag] = [round(t, 4), round(fl / t / 1e9, 1)]
                    t = _time(lambda: ops.raw_tc_linear_bwd_dx(gp, N, Wp, K, a, False, True, True),
                              **tm)
                    res["dx+colsum " + tag] = [round(t, 4), round(fl / t / 1e9, 1)]
                    t = _time(lambda: ops.raw_tc_linear_bwd_dx(gp, N, Wp, K, None, True, False, False),
                              **tm)
                    res["dx f32 " + tag] = [round(t, 4), round(fl / t / 1e9, 1)]
                t = _time(lambda: ops.raw_tc_linear_bwd_dw(a, K, gp, N), **tm)
                res["dw  %dx%d bn%d" % (K, N, bn)] = [round(t, 4), round(fl / t / 1e9, 1)]
            ops.tc_debug(0, 0)
            ops.tc_debug(4, 32)
            # library reference: the three bf16 GEMMs of the round-1 path
            a2 = torch.randn(M, 2 * K, device=dev).to(torch.bfloat16)
            w2 = torch.randn(2 * K, N, device=dev).to(torch.bfloat16)
            wl = torch.randn(K, N, device=dev).to(torch.bfloat16)
            y = torch.empty(M, N, device=dev)

            def lib():
                torch.mm(a2, w2, out_dtype=torch.float32, out=y)
                torch.addmm(y, a2[:, :K], wl, out_dtype=torch.float32, out=y)
            t = _time(lib)
            res["cublas fwd %dx%d" % (K, N)] = [round(t, 4), round(fl / t / 1e9, 1)]
        out.update(res)
        out["unit"] = "[ms, TFLOP/s of bf16 MMA work]"
    print(json.dumps(out), flush=True)


def main():
    if len(sys.argv) > 1:
        stage(sys.argv[1], sys.argv[2] if len(sys.argv) > 2 else "")
        return
    plan = [("fwd", "32"), ("fwd", "64"), ("dx", "32"), ("dx", "64"), ("dw", ""), ("perf", "")]
    # descriptor candidates for the MN-major operands if the default is wrong: (lbo_a, lbo_b, sbo)
    sweep = [("dw", "1024,1024,4096"), ("dw", "4096,4096,2048"), ("dw", "2048,2048,1024"),
             ("dw", "1024,1024,2048")]
    results = []
    for name, arg in plan + sweep:
        if name == "dw" and arg and any(r.get("stage") == "dw" and r.get("ok") for r in results):
            continue
        t0 = time.time()
        try:
            p = subprocess.run([sys.executable, os.path.abspath(__file__), name, arg],
                               capture_output=True, text=True, timeout=300)
            line = [l for l in p.stdout.splitlines() if l.startswith("{")]
            r = json.loads(line[-1]) if line else {"stage": name, "arg": arg, "rc": p.returncode,
                                                   "stderr": p.stderr[-1500:]}
        except subprocess.TimeoutExpired:
            r = {"stage": name, "arg": arg, "timeout": True}
        vals = [v for k, v in r.items() if "x" in k and isinstance(v, (float, list))]
        flat = [x for v in vals for x in (v if isinstance(v, list) else [v])]
        r["ok"] = bool(flat) and all(x < 5e-5 for x in flat) if name != "perf" else True
        r["secs"] = round(time.time() - t0, 1)
        results.append(r)
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
