"""Persistent and grid-stride kernels at sizes where every CTA (or warp, or lane group) loops.

The unit tests in test_gpu_kernels.py run these kernels where the grid is not yet capped, so each
CTA makes one pass or none.  Here every size is computed from the launcher's grid formula and the
device's SM count (the library reads the same attribute, b200rec.cu:32-43), and each test asserts
that every CTA / warp / lane group makes at least MIN_ITERS passes of its loop.  The C++ constants
are mirrored below with the line that defines them: if one changes, the iteration assertions fail
instead of the test silently shrinking back into the one-pass regime.

Every value is compared ELEMENT-WISE with a float64 reference of the same operation computed on the
GPU.  fp32 sums are held to
    |got - want| <= k * 2^-24 * sum|terms|        (per element)
where k is the longest chain of fp32 roundings the kernel's summation order can put on that
element; each test's docstring derives its k from the kernel's loop structure.  Copies, gathers and
single correctly-rounded products are compared with torch.equal, and the paths documented as
fixed-order are run twice and must be bit-identical.
"""
import math
import os

import numpy as np
import pytest
import torch

from oracle import nets
from oracle import optim as ooptim
from tests.test_gpu_fat_deepffm import _fat_smem, _gamma, _oracle

pytestmark = pytest.mark.gpu

DEV = "cuda"
U = 2.0 ** -24            # unit roundoff of fp32
MIN_ITERS = 3

# ---- C++ constants mirrored here (file:line of the definition) ---------------------------------
DIN_TILE = 64             # din_attn.cuh:28   kDinTile; grid = min(tiles, SM) din_attn.cuh:627-630,693-694
DIN_H1, DIN_H2 = 80, 40   # din_attn.cuh:26-27
SEG_THREADS = 256         # segreduce.cuh:17  kSegThreads; light grid min(ceil(n/GPB), 64*SM) :160-161
HOT_THRESHOLD = 64        # segreduce.cuh:26  kHotThreshold
HOT_CHUNK = 2048          # segreduce.cuh:27  kHotChunk
ROW_THREADS = 256         # gather_scatter.cuh:18 kGatherThreads; grids min(ceil(n/GPB), 64*SM)
#                           gather_scatter.cuh:132-134 (pool), :328-330 and :349-351 (row updates)
FWD_THREADS = 128         # embed_fm.cuh:56-57 FwdGeom; grid min(tiles, SM*ctas_per_sm) :596
FWD_CTAS_PER_SM = 8       # embed_fm.cuh:39 K1Config default ctas_per_sm
BWD_THREADS = 256         # embed_fm.cuh:634 kBwdThreads (dense-part samples per CTA = 256/TPR :675)
BWD_DENSE_CTAS_PER_SM = 2  # embed_fm.cuh:792 bwd_dense_grid() = 2*SM
DENSE_CHUNK = 8           # embed_fm.cuh:666 kDenseChunk
BWD_WARPS = 8             # embed_fm.cuh:676 kWarps = kBwdThreads/32
RED_LANES = 32            # embed_fm.cuh:758 kRedLanes; 4-in-flight loop while g + 3*32 < G :768
DOT_WARPS = 4             # dot_interact.cuh:24 kDotWarps; shrink while > 96 KB b200rec.cu:607-608
DOT_CTAS_PER_SM = 8       # b200rec.cu:612
CROSS_ROW_SLICES = 264    # cross.cuh:42 kCrossRowSlices
TOWER_ROW_SLICES = 528    # tower.cuh:337 kTowerRowSlices; TX/TY tower.cuh:382-384
TOWER_THREADS = 256       # tower.cuh:21
TOWER_UNROLL = 4          # tower.cuh:103 kBwdUnroll
STREAM_CTAS_PER_SM = 16   # b200rec.cu:577,589,642 (cvm, hash_keys: 256-thread CTAs)
FFM_THREADS = 256         # ffm.cuh:19  kFfmThreads
FFM_MAX_FIELDS = 64       # ffm.cuh:20  kFfmMaxFields
FFM_FWD_MAX_CTAS_PER_SM = 2048 // FFM_THREADS  # ffm.cuh:176-179 grid = min(B, SM*per_sm), per_sm from
#                           the occupancy call: at most 2048 threads per SM
FFM_HOT_CHUNK = 1024      # ffm.cuh:244 kFfmHotChunk; items pack c | (chunks << 16) :287
FFM_MAX_CHUNKS = 32767    # ffm.cuh:465 B*F < 32767 * kFfmHotChunk
FFM_MAX_SLICES = 256      # ffm.cuh:257 slices = min(256, ceil(B/256))
FFM_LIGHT_CTAS_PER_SM = 16  # ffm.cuh:429 light grid min(ceil(n/8), 16*SM)
FFM_HOT_CTAS_PER_SM = 8   # ffm.cuh:434 hot / combine grid min(max_items, 8*SM)
WIDE_CTAS_PER_SM = 64     # gather_scatter.cuh:399, 428 wide-row grids min(ceil(n/8), 64*SM)
FAT_POOL_THREADS = 256    # fat_ffm.cuh:322-324 pool grid min(ceil(B*NF^2/256), 16*SM) of 256 threads
FAT_POOL_CTAS_PER_SM = 16
FAT_SAMPLE_MAX_CTAS_PER_SM = 2048 // FFM_THREADS  # fat_ffm.cuh:350-353 grid = min(B, SM*per_sm),
#                           per_sm from the occupancy call: at most 2048 threads per SM
FAT_MAX_POSITIONS = FFM_MAX_CHUNKS * FFM_HOT_CHUNK  # fat_ffm.cuh:370 B*F < 32767 * kFfmHotChunk
#                           FatSmem, fat_ffm.cuh:70-81, is mirrored by test_gpu_fat_deepffm._fat_smem


def _ops():
    from paddlerec_b200 import ops
    return ops


def _sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cdiv(a, b):
    return -(-a // b)


def row_shape(D):
    """pick_row_shape, common.cuh:223-232: (VEC floats per lane, TPR lanes per row)."""
    vec = 4 if D % 4 == 0 else (2 if D % 2 == 0 else 1)
    chunks = D // vec
    tpr = 1
    while tpr < chunks:
        tpr <<= 1
    return vec, tpr


def assert_loops(what, iters):
    """Every CTA / warp / lane group of `what` makes at least MIN_ITERS passes."""
    print("[iterations] %s: %d" % (what, iters))
    assert iters >= MIN_ITERS, "%s: only %d passes per CTA; the size no longer makes the grid loop" % (
        what, iters)


def assert_within(got, want, bound, what):
    """Element-wise |got - want| <= bound (all float64 on the device)."""
    got = got.double()
    assert got.shape == want.shape, (what, got.shape, want.shape)
    err = (got - want).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        i = int(torch.argmax((err - bound).reshape(-1)))
        raise AssertionError("%s: %d / %d entries out of bound; worst at flat index %d: got %.9g want "
                             "%.9g bound %.3g" % (what, int(bad.sum()), bad.numel(), i,
                                                  float(got.reshape(-1)[i]), float(want.reshape(-1)[i]),
                                                  float(bound.reshape(-1)[i])))


@pytest.fixture(autouse=True)
def hbm_budget(request):
    """Each test allocates at most ~12 GB; skip when the shared GPU has less free."""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < 14e9:
        pytest.skip("needs ~14 GB of free HBM (%.1f GB free)" % (free / 1e9))
    torch.cuda.reset_peak_memory_stats()
    yield
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    print("[peak] %s: %.2f GB" % (request.node.name, peak / 1e9))
    assert peak <= 12.5e9, "%s allocated %.1f GB" % (request.node.name, peak / 1e9)


def seg_chain(counts, D):
    """Longest fp32 chain of one merged row in launch_seg_reduce (segreduce.cuh): a segment of
    <= 64 positions is summed sequentially by one lane group (k = count); a hot one is cut into
    2048-position chunks, each summed by GPB groups striding the chunk (ceil(2048/GPB) adds), a
    log2(GPB)-level shared-memory tree, and seg_combine_kernel adds the chunk partials in order
    (one add per chunk)."""
    _, tpr = row_shape(D)
    gpb = SEG_THREADS // tpr
    hot = counts > HOT_THRESHOLD
    k_hot = _cdiv(HOT_CHUNK, gpb) + int(math.log2(gpb)) + (counts + HOT_CHUNK - 1) // HOT_CHUNK
    return torch.where(hot, k_hot, counts).double()


# ================================================================================================
# 1. DIN attention (din_attn.cuh): forward scores kernel and fused backward, persistent over tiles
# ================================================================================================
def _din_params(E, g):
    W1 = torch.randn(4 * E, DIN_H1, generator=g, device=DEV) / (4 * E) ** 0.5
    b1 = torch.randn(DIN_H1, generator=g, device=DEV) * 0.1
    W2 = torch.randn(DIN_H1, DIN_H2, generator=g, device=DEV) / DIN_H1 ** 0.5
    b2 = torch.randn(DIN_H2, generator=g, device=DEV) * 0.1
    W3 = torch.randn(DIN_H2, 1, generator=g, device=DEV) / DIN_H2 ** 0.5
    b3 = torch.randn(1, generator=g, device=DEV) * 0.1
    return [W1, b1, W2, b2, W3, b3]


def _din_reference(hist, tseq, mask, params, dout, L_tiles_k):
    """fp64 on the device, chunked over samples.  Returns, per output and gradient:
      want  nets.din_attention_unit and its autograd gradients;
      bound k * 2^-24 * M + Ep, where M is the output recomputed with every factor replaced by its
            absolute value (the sum|terms| of its own summation, chain length k from L_tiles_k) and
            Ep is the first-order propagation, position by position, of the fp32 errors of the
            factors the kernels recompute (z1, z2, the softmax weights w, <dout, h>, da, dz2, g).
    Forward error model (u = 2^-24; sigmoid by __expf, add and divide: 4u absolute on z <= 1):
      a1 = h Wac + (h*t) Wd + tb      e_a1 = (3E + 4) u M_a1   (tb: E-term addmm; 2E fmas)
      z1 = sigmoid(a1)                e_z1 = e_a1 / 4 + 4u     (sigmoid' <= 1/4)
      a2 = z1 W2 + b2                 e_a2 = 82 u M_a2 + e_z1 |W2|
      z2, s = scale (z2 W3 + b3)      e_s  = scale (44 u M_s + e_z2 |W3|)
      w = softmax(s)                  |dw_l| <= w_l (2 max_l e_s + (ceil(L/128) + 12) u)"""
    B, L, E = hist.shape
    scale = E ** -0.5
    P64 = [p.double().requires_grad_(True) for p in params]
    W1, b1, W2, b2, W3, b3 = [p.detach() for p in P64]
    Wa, Wb, Wc, Wd = W1[:E], W1[E:2 * E], W1[2 * E:3 * E], W1[3 * E:]
    aWac, aWd, aWbc, aW2, aW3 = (Wa + Wc).abs(), Wd.abs(), (Wb - Wc).abs(), W2.abs(), W3.abs().reshape(-1)
    f64 = dict(dtype=torch.float64, device=DEV)
    want = {"out": torch.empty(B, E, **f64), "dhist": torch.empty(B, L, E, **f64),
            "dtseq": torch.empty(B, E, **f64)}
    bound = {k: torch.empty_like(v) for k, v in want.items()}
    pgrad = [torch.zeros_like(p) for p in P64]
    acc = {k: torch.zeros(E, DIN_H1, **f64) for k in ("MWa", "EWa", "MWb", "EWb", "MWd", "EWd")}
    acc.update({k: torch.zeros(DIN_H1, **f64) for k in ("Mb1", "Eb1")})
    acc.update({k: torch.zeros(DIN_H1, DIN_H2, **f64) for k in ("MW2", "EW2")})
    acc.update({k: torch.zeros(DIN_H2, **f64) for k in ("Mb2", "Eb2", "MW3", "EW3")})
    acc.update({k: torch.zeros((), **f64) for k in ("Mb3", "Eb3")})
    wsum = torch.empty(B, **f64)
    k_out, k_dhist, k_dtseq, k_cta, k_B, k_P = L_tiles_k
    chunk = max(1, (1 << 24) // (L * 4 * E))
    for s in range(0, B, chunk):
        e = min(B, s + chunk)
        h = hist[s:e].double().requires_grad_(True)
        t = tseq[s:e].double().requires_grad_(True)
        m = mask[s:e] if mask is not None else None
        go = dout[s:e].double()
        o = nets.din_attention_unit(h, t, m, *P64)
        gs = torch.autograd.grad(o, [h, t] + P64, go)
        want["out"][s:e] = o.detach()
        want["dhist"][s:e] = gs[0]
        want["dtseq"][s:e] = gs[1]
        for a, gg in zip(pgrad, gs[2:]):
            a += gg
        with torch.no_grad():
            h, t = h.detach(), t.detach()
            tt = t.unsqueeze(1).expand_as(h)
            ah, at, aht = h.abs(), t.abs(), (h * tt).abs()
            c = torch.cat([h, tt, h - tt, h * tt], 2)
            z1 = torch.sigmoid(c @ W1 + b1)
            z2 = torch.sigmoid(z1 @ W2 + b2)
            sc = (z2 @ W3 + b3).squeeze(2)
            if m is not None:
                sc = sc + m.reshape(sc.shape).double()
            w = torch.softmax(sc * scale, 1)
            wsum[s:e] = w.sum(1)
            live = w > 0
            # forward errors
            Ma1 = ah @ aWac + aht @ aWd + (at @ aWbc + b1.abs()).unsqueeze(1)
            ez1 = (3 * E + 4) * U * Ma1 / 4 + 4 * U
            ez2 = (82 * U * (z1 @ aW2 + b2.abs()) + ez1 @ aW2) / 4 + 4 * U
            es = scale * (44 * U * (z2 @ aW3 + b3.abs()) + ez2 @ aW3) * live
            dlw = 2 * es.max(1, keepdim=True).values + (_cdiv(L, 128) + 12) * U
            Ew = w * dlw
            # backward values, magnitudes M and propagated errors Ep
            dw = (h * go.unsqueeze(1)).sum(2)
            Mdw = (ah * go.abs().unsqueeze(1)).sum(2)
            Edw = (E + 6) * U * Mdw
            dot = (w * dw).sum(1, keepdim=True)
            Edot = (Ew * dw.abs() + w * Edw).sum(1, keepdim=True) + (_cdiv(L, 128) + 8) * U * (w * dw.abs()).sum(1, keepdim=True)
            da = scale * w * (dw - dot)
            Mda = scale * w * (Mdw + (w * Mdw).sum(1, keepdim=True))
            Eda = scale * (Ew * (dw.abs() + dot.abs()) + w * (Edw + Edot)) + 3 * U * Mda
            d2 = z2 * (1 - z2)
            Mdz2 = Mda.unsqueeze(2) * aW3 * d2
            dz2 = da.unsqueeze(2) * W3.reshape(-1) * d2
            Edz2 = (Eda.unsqueeze(2) * d2 + da.abs().unsqueeze(2) * ez2) * aW3 + 4 * U * Mdz2
            d1 = z1 * (1 - z1)
            q = dz2 @ W2.t()
            Mq = Mdz2 @ aW2.t()
            Mg = Mq * d1
            Eg = (Edz2 @ aW2.t() + 41 * U * Mq) * d1 + q.abs() * ez1 + 2 * U * Mg
            # outputs
            bound["out"][s:e] = k_out * U * (w.unsqueeze(2) * ah).sum(1) + (Ew.unsqueeze(2) * ah).sum(1)
            MgWd, EgWd = Mg @ aWd.t(), Eg @ aWd.t()
            bound["dhist"][s:e] = (k_dhist * U * (w.unsqueeze(2) * go.abs().unsqueeze(1) + Mg @ aWac.t()
                                                  + MgWd * tt.abs())
                                   + Ew.unsqueeze(2) * go.abs().unsqueeze(1) + Eg @ aWac.t() + EgWd * tt.abs())
            bound["dtseq"][s:e] = (k_dtseq * U * ((MgWd * ah).sum(1) + Mg.sum(1) @ aWbc.t())
                                   + (EgWd * ah).sum(1) + Eg.sum(1) @ aWbc.t())
            flat = lambda x: x.reshape(-1, x.shape[-1])  # noqa: E731
            acc["MWa"] += flat(ah).t() @ flat(Mg)
            acc["EWa"] += flat(ah).t() @ flat(Eg)
            acc["MWb"] += at.t() @ Mg.sum(1)
            acc["EWb"] += at.t() @ Eg.sum(1)
            acc["MWd"] += flat(aht).t() @ flat(Mg)
            acc["EWd"] += flat(aht).t() @ flat(Eg)
            acc["Mb1"] += Mg.sum((0, 1))
            acc["Eb1"] += Eg.sum((0, 1))
            acc["MW2"] += flat(z1).t() @ flat(Mdz2)
            acc["EW2"] += flat(z1).t() @ flat(Edz2) + flat(ez1).t() @ flat(dz2.abs())
            acc["Mb2"] += Mdz2.sum((0, 1))
            acc["Eb2"] += Edz2.sum((0, 1))
            acc["MW3"] += (z2 * Mda.unsqueeze(2)).sum((0, 1))
            acc["EW3"] += (z2 * Eda.unsqueeze(2) + ez2 * da.abs().unsqueeze(2)).sum((0, 1))
            acc["Mb3"] += Mda.sum()
            acc["Eb3"] += Eda.sum()
    a = acc
    bWa = k_cta * U * a["MWa"] + a["EWa"]
    bWb = k_B * U * a["MWb"] + a["EWb"]
    bound["dW1"] = torch.cat([bWa, bWb, bWa + bWb + U * (a["MWa"] + a["MWb"]), k_cta * U * a["MWd"] + a["EWd"]], 0)
    bound["db1"] = k_B * U * a["Mb1"] + a["Eb1"]
    bound["dW2"] = k_cta * U * a["MW2"] + a["EW2"]
    bound["db2"] = k_cta * U * a["Mb2"] + a["Eb2"]
    bound["dW3"] = (k_cta * U * a["MW3"] + a["EW3"]).reshape(-1, 1)
    bound["db3"] = (k_P * U * a["Mb3"] + a["Eb3"]).reshape(1)
    for k, gg in zip(("dW1", "db1", "dW2", "db2", "dW3", "db3"), pgrad):
        want[k] = gg
    return want, bound, wsum


def _din_case(B, L, E, seed):
    """Runs the fused forward + backward (ops.din_attention) on B samples of L positions with a
    mask of variable lengths, and checks every output and gradient element-wise against
    nets.din_attention_unit in fp64 (bounds: _din_reference).

    Loop: P = B*L positions in 64-position tiles, grid = min(tiles, SM) persistent CTAs
    (din_attn.cuh:627-630, 693-694); each CTA runs `tpc` tiles and the backward keeps
    aWac/aWd/aW2/ab2/aW3 in registers across all of them (din_attn.cuh:331-343).

    Summation chains k (on top of the propagated factor errors):
      out          L-term fma chain over the history (din_softmax_pool_kernel) + 1
      dhist        80-term GEMMs (g Wac^T, g Wd^T) + 3 fmas
      dtseq        L positions (atomics, any order) + 80 (g Wd^T) + 80 (addmm with dtb) + 2
      dWa, dWd, dW2, db2, dW3   64 positions per tile x tpc tiles in a CTA's registers, then the
                   grid partials in order (din_reduce_partials_kernel) + 16 (shuffles, products)
      dWb, db1     B samples (torch matmul / sum over dtb) + L (dtb atomics) + 2
      db3          B*L (torch sum of da) + 2
    The softmax weights must sum to 1 within (ceil(L/128) + 10) roundings (128-thread sum, 5-level
    shuffle, 4 warp partials, one division, one multiply per weight), and masked positions get
    exactly 0."""
    ops = _ops()
    SM = _sm()
    P = B * L
    tiles = _cdiv(P, DIN_TILE)
    grid = min(tiles, SM)
    tpc = _cdiv(tiles, grid)
    assert_loops("din scores fwd/bwd B=%d L=%d E=%d: tiles per CTA" % (B, L, E), tiles // grid)
    g = torch.Generator(device=DEV).manual_seed(seed)
    hist = torch.randn(B, L, E, generator=g, device=DEV) * 0.5
    tseq = torch.randn(B, E, generator=g, device=DEV) * 0.5
    lens = torch.randint(1, L + 1, (B,), generator=g, device=DEV)
    lens[0] = L
    lens[1 % B] = 1
    mask = torch.where(torch.arange(L, device=DEV).unsqueeze(0) < lens.unsqueeze(1), 0,
                       int(-1e9)).to(torch.int64).unsqueeze(2)
    params = _din_params(E, g)
    dout = torch.randn(B, E, generator=g, device=DEV)

    dev_in = [t.clone().requires_grad_(True) for t in [hist, tseq] + params]
    out = ops.din_attention(dev_in[0], dev_in[1], mask, *dev_in[2:])
    out.backward(dout)
    _, w = ops.raw_din_attn_fwd(hist, tseq, mask, *params)
    torch.cuda.synchronize()

    ks = (L + 1, DIN_H1 + 3, L + 2 * DIN_H1 + 2, DIN_TILE * tpc + grid + 16, B + L + 2, P + 2)
    want, bound, wsum_ref = _din_reference(hist, tseq, mask, params, dout, ks)
    got = {"out": out, "dhist": dev_in[0].grad, "dtseq": dev_in[1].grad}
    got.update(zip(("dW1", "db1", "dW2", "db2", "dW3", "db3"), [p.grad for p in dev_in[2:]]))
    for name in ("out", "dhist", "dtseq", "dW1", "db1", "dW2", "db2", "dW3", "db3"):
        assert_within(got[name], want[name], bound[name] + 1e-30, "DIN %s B=%d L=%d E=%d" % (name, B, L, E))
    # softmax weights: normalised, masked positions exactly zero
    assert_within(w.double().sum(1), torch.ones_like(wsum_ref),
                  torch.full_like(wsum_ref, (_cdiv(L, 128) + 10) * U), "DIN sum of weights")
    masked = mask.squeeze(2) != 0
    assert bool((w[masked] == 0).all()), "masked history positions must get weight exactly 0"
    # the fixed-order weight gradients are bit-reproducible (dtseq / dtb use atomics: excluded)
    r1 = ops.raw_din_attn_bwd(hist, tseq, *params[:5], w, dout)
    r2 = ops.raw_din_attn_bwd(hist, tseq, *params[:5], w, dout)
    kernel_rows = torch.cat([torch.arange(E), torch.arange(3 * E, 4 * E)]).to(DEV)  # Wa, Wd of dW1
    assert torch.equal(r1[2][kernel_rows], r2[2][kernel_rows]), "DIN dWac/dWd differ between runs"
    for i in (4, 5, 6):          # dW2, db2, dW3
        assert torch.equal(r1[i], r2[i]), "DIN fixed-order weight gradient %d differs between runs" % i
    assert torch.equal(r1[0], r2[0]), "dhist is per position (no atomics): must be reproducible"


def test_din_bench_shape():
    """The DIN benchmark shape: B=4096, L=100, E=128, ~48 tiles per CTA."""
    _din_case(4096, 100, 128, seed=1)


@pytest.mark.parametrize("E", [4, 20, 36, 100])
def test_din_partial_register_tiles(E):
    """E not a multiple of 16: the last of the kreps = ceil(E/16) k-rows of the aWac/aWd register
    tiles is partial (din_attn.cuh:344, 522-525, 604-606).  L=61 makes tiles straddle samples."""
    L = 61
    B = _cdiv((3 * _sm() + _sm() // 2) * DIN_TILE, L)
    _din_case(B, L, E, seed=E)


def test_din_longest_history():
    """L = 8192 (the maximum: a 32 KB softmax row in shared memory) with enough samples that the
    grid loops."""
    L = 8192
    B = _cdiv((3 * _sm() + _sm() // 2) * DIN_TILE, L)
    _din_case(B, L, 32, seed=8192)


# ================================================================================================
# 2. Segment reduce (segreduce.cuh): hot path with several 2048-position chunks + combine
# ================================================================================================
HOT_LENS = [64, 65, 2048, 2049, 6145, 150001]


def _hot_stream(n_uniform, V, g):
    """Ids with segments of exactly HOT_LENS positions (ids 11..16), uniform traffic, and 5000
    padding ids (0) shuffled in between, so padding sits inside the hot runs."""
    parts = [torch.full((n,), 11 + i, dtype=torch.int64, device=DEV) for i, n in enumerate(HOT_LENS)]
    parts.append(torch.randint(100, V, (n_uniform,), generator=g, device=DEV))
    parts.append(torch.zeros(5000, dtype=torch.int64, device=DEV))
    ids = torch.cat(parts)
    return ids[torch.randperm(ids.numel(), generator=g, device=DEV)]


def _check_segment_rows(ops, gr, rows_fn, contrib, valid_ids, D, what):
    """rows_fn() -> merged rows; contrib [n_valid, D] fp64 per-position terms in position order;
    checks against index_add in fp64 with the seg_chain bound, then bit-reproducibility."""
    uniq, inv, counts = torch.unique(valid_ids, return_inverse=True, return_counts=True)
    Uq = uniq.numel()
    assert int(gr.num[0]) == Uq
    assert torch.equal(gr.unique_ids[:Uq], uniq)
    want = torch.zeros(Uq, D, dtype=torch.float64, device=DEV).index_add_(0, inv, contrib)
    mag = torch.zeros(Uq, D, dtype=torch.float64, device=DEV).index_add_(0, inv, contrib.abs())
    k = seg_chain(counts, D).unsqueeze(1)
    rows = rows_fn()
    assert_within(rows[:Uq], want, k * U * mag + 1e-30, what)
    assert torch.equal(rows[:Uq], rows_fn()[:Uq]), what + ": not bit-reproducible"
    return counts


@pytest.mark.parametrize("D", [1, 2, 3, 9, 16, 40, 128])
def test_segment_reduce_hot_chunks(D):
    """raw_segment_reduce on segments of 64 (light), 65, 2048, 2049 (hot, 1-2 chunks), 6145
    (4 chunks) and 150001 (74 chunks) positions plus uniform traffic and padding; every VEC/TPR
    family.  Bound: seg_chain (light: count adds; hot: ceil(2048/GPB) + log2(GPB) + chunks)."""
    ops = _ops()
    chunks = [_cdiv(n, HOT_CHUNK) for n in HOT_LENS if n > HOT_THRESHOLD]
    assert_loops("seg_combine_kernel: chunks added for the 6145-position id", chunks[-2])
    assert_loops("seg_combine_kernel: chunks added for the 150001-position id", chunks[-1])
    g = torch.Generator(device=DEV).manual_seed(D)
    V = 1_000_000
    ids = _hot_stream(100_000, V, g)
    n = ids.numel()
    dOut = torch.randn(n, D, generator=g, device=DEV)
    gr = ops.raw_group_ids(ids, V, 0)
    valid = ids != 0
    counts = _check_segment_rows(
        ops, gr, lambda: ops.raw_segment_reduce(dOut, gr.seg_offsets, gr.sorted_pos, gr.num, n),
        dOut[valid].double(), ids[valid], D, "segment_reduce D=%d" % D)
    assert sorted(counts[counts > 1000].tolist()) == [2048, 2049, 6145, 150001]


def test_segment_reduce_light_kernel_loops():
    """D=16 with U >= 3 * 64*SM CTAs * 64 groups distinct ids: every lane group of
    seg_light_kernel walks >= 3 segments (segreduce.cuh:47-48, 160-161); hot ids ride along."""
    ops = _ops()
    D = 16
    _, tpr = row_shape(D)
    gpb = SEG_THREADS // tpr
    cap = 64 * _sm() * gpb
    Uq = 3 * cap + 1001
    g = torch.Generator(device=DEV).manual_seed(16)
    V = 4 * Uq
    ids = torch.cat([torch.randperm(V - 100, generator=g, device=DEV)[:Uq] + 100,
                     _hot_stream(0, V, g)])
    ids = ids[torch.randperm(ids.numel(), generator=g, device=DEV)]
    n = ids.numel()
    grid = min(_cdiv(n, gpb), 64 * _sm())
    assert_loops("seg_light_kernel: segments per lane group", Uq // (grid * gpb))
    dOut = torch.randn(n, D, generator=g, device=DEV)
    gr = ops.raw_group_ids(ids, V, 0)
    valid = ids != 0
    _check_segment_rows(
        ops, gr, lambda: ops.raw_segment_reduce(dOut, gr.seg_offsets, gr.sorted_pos, gr.num, n),
        dOut[valid].double(), ids[valid], D, "segment_reduce light loop")


# ================================================================================================
# 3. embed_fm backward at B=65536 with Zipf ids (hot ids of tens of thousands of positions)
# ================================================================================================
@pytest.mark.parametrize("D", [9, 16, 40])
@pytest.mark.parametrize("Dn", [0, 8, 13, 17])
def test_embed_fm_bwd_zipf(D, Dn):
    """raw_embed_fm_bwd, two-table and fused_cols layouts, B=65536 x F=26, Zipf ids over V=1e6.

    Sparse rows: per position the kernel forms fmaf(gy2, S - feat, dfeat) (2 roundings of
    |gy2|(|S| + |feat|) + |dfeat|) and merges them in seg_chain order: k = seg_chain + 2.  dW1 is
    the same merge of gy1 (k = seg_chain).
    Dense part (embed_fm_bwd_dense_kernel): each lane accumulates iters = ceil(B / (2*SM*SPB))
    samples, then log2(32/TPR) shuffles, 8 warp partials in order, and reduce_partials_kernel adds
    ceil(G/32) partials per lane and 32 lanes: k = iters + 5 + 8 + ceil(G/32) + 32 + 3 for
    fmaf(x, fmaf(g2, S - fe, dd), acc) terms of magnitude |x|(|g2|(|S| + |fe|) + |dd|)."""
    ops = _ops()
    SM = _sm()
    B, F, V = 65536, 26, 1_000_000
    vec, tpr = row_shape(D)
    spb = BWD_THREADS // tpr
    G = BWD_DENSE_CTAS_PER_SM * SM
    assert_loops("embed_fm_bwd_dense_kernel D=%d: samples per lane" % D, B // (G * spb))
    red_iters = len(range(0, G - 3 * RED_LANES, 4 * RED_LANES))
    assert red_iters >= 1, "reduce_partials_kernel's 4-loads-in-flight branch is no longer reached"
    g = torch.Generator(device=DEV).manual_seed(1000 * D + Dn)
    r = torch.rand(B, F, generator=g, device=DEV, dtype=torch.float64)
    ids = (V ** r).to(torch.int64).clamp_(1, V - 1)
    ids[torch.rand(B, F, generator=g, device=DEV) < 0.02] = 0
    N = F + Dn
    feat = torch.randn(B, N, D, generator=g, device=DEV) * 0.1
    S = torch.randn(B, D, generator=g, device=DEV)
    dfeat = torch.randn(B, N, D, generator=g, device=DEV) * 0.01
    gy1 = torch.randn(B, generator=g, device=DEV)
    gy2 = torch.randn(B, generator=g, device=DEV)
    dense = torch.rand(B, Dn, generator=g, device=DEV)
    dense[torch.rand(B, Dn, generator=g, device=DEV) < 0.3] = 0
    gr = ops.raw_group_ids(ids, V, 0)
    args = (feat, S, dfeat, gy1, gy2, dense, gr.seg_offsets, gr.sorted_pos, gr.num, F)

    flat = ids.reshape(-1)
    valid = flat != 0
    b_of = torch.arange(B, device=DEV).repeat_interleave(F)[valid]
    fe = feat[:, :F].reshape(-1, D)[valid].double()
    dd = dfeat[:, :F].reshape(-1, D)[valid].double()
    g2 = gy2.double()[b_of].unsqueeze(1)
    Sb = S.double()[b_of]
    uniq, inv, counts = torch.unique(flat[valid], return_inverse=True, return_counts=True)
    Uq = uniq.numel()
    hot_chunks = _cdiv(int(counts.max()), HOT_CHUNK)
    assert_loops("embed_fm_bwd seg_combine_kernel: chunks of the hottest id", hot_chunks)
    z = lambda *s: torch.zeros(*s, dtype=torch.float64, device=DEV)  # noqa: E731
    want = z(Uq, D).index_add_(0, inv, g2 * (Sb - fe) + dd)
    mag = z(Uq, D).index_add_(0, inv, g2.abs() * (Sb.abs() + fe.abs()) + dd.abs())
    del fe, dd, Sb
    want1 = z(Uq).index_add_(0, inv, gy1.double()[b_of])
    mag1 = z(Uq).index_add_(0, inv, gy1.double().abs()[b_of])
    k = seg_chain(counts, D)

    dW, dW1, ddw, ddw1 = ops.raw_embed_fm_bwd(*args)
    assert_within(dW[:Uq], want, (k + 2).unsqueeze(1) * U * mag + 1e-30, "dW rows D=%d Dn=%d" % (D, Dn))
    assert_within(dW1[:Uq], want1, k * U * mag1 + 1e-30, "dW1 rows D=%d Dn=%d" % (D, Dn))
    if Dn > 0:
        x = dense.double().unsqueeze(2)
        fd, dfd = feat[:, F:].double(), dfeat[:, F:].double()
        g2b = gy2.double().reshape(B, 1, 1)
        Sd = S.double().unsqueeze(1)
        wdw = (x * (g2b * (Sd - fd) + dfd)).sum(0)
        mdw = (x * (g2b.abs() * (Sd.abs() + fd.abs()) + dfd.abs())).sum(0)
        kd = _cdiv(B, G * spb) + int(math.log2(32 // tpr)) + BWD_WARPS + _cdiv(G, RED_LANES) + RED_LANES
        assert_within(ddw, wdw, (kd + 3) * U * mdw + 1e-30, "ddense_w D=%d Dn=%d" % (D, Dn))
        wd1 = (dense.double() * gy1.double().unsqueeze(1)).sum(0)
        md1 = (dense.double() * gy1.double().abs().unsqueeze(1)).sum(0)
        kd1 = _cdiv(B, G * spb) + 5 + BWD_WARPS + _cdiv(G, RED_LANES) + RED_LANES + 1
        assert_within(ddw1, wd1, kd1 * U * md1 + 1e-30, "ddense_w1 D=%d Dn=%d" % (D, Dn))
    # deterministic, and the fused layout [D | g1 | zeros] holds exactly the same numbers
    dW_b, dW1_b, ddw_b, ddw1_b = ops.raw_embed_fm_bwd(*args)
    assert torch.equal(dW[:Uq], dW_b[:Uq]) and torch.equal(dW1[:Uq], dW1_b[:Uq])
    assert torch.equal(ddw, ddw_b) and torch.equal(ddw1, ddw1_b)
    Gc = ops.fused_grad_cols(D)
    dWf, none, ddw_f, _ = ops.raw_embed_fm_bwd(*args, fused_cols=Gc)
    assert none is None
    assert torch.equal(dWf[:Uq, :D], dW[:Uq]) and torch.equal(dWf[:Uq, D], dW1[:Uq])
    assert not dWf[:Uq, D + 1:].any(), "zero_pad columns of the fused rows must be written as 0"
    assert torch.equal(ddw_f, ddw)


# ================================================================================================
# 4. DLRM dot interaction (dot_interact.cuh): one warp per sample, persistent grid
# ================================================================================================
def _dot_warps(N, d, bwd):
    """dot_interact_launch, b200rec.cu:605-608 (v1 path)."""
    pitch = d + 1
    per_warp = 4 * (N * pitch + (N * N if bwd else 0))
    warps = DOT_WARPS
    while warps > 1 and warps * per_warp > 96 * 1024:
        warps >>= 1
    return warps


def _dot_ref(T, dR, self_interaction, chunk=4096):
    """nets.dot_interact in fp64 (value and autograd gradient) and the same on |T| with |dR| as
    the magnitude, chunked over samples."""
    outs = [[], [], [], []]
    for s in range(0, T.shape[0], chunk):
        for j, src in enumerate((T[s:s + chunk], T[s:s + chunk].abs())):
            Tl = src.double().requires_grad_(True)
            R = nets.dot_interact(Tl, self_interaction)
            gT, = torch.autograd.grad(R, Tl, (dR[s:s + chunk] if j == 0 else dR[s:s + chunk].abs()).double())
            outs[j].append(R.detach())
            outs[2 + j].append(gT)
    return [torch.cat(o) for o in outs]


@pytest.mark.parametrize("B,N,d", [(65536, 27, 16), (16384, 128, 4), (8192, 27, 256)])
@pytest.mark.parametrize("self_interaction", [False, True])
def test_dot_interact_fwd_bwd(B, N, d, self_interaction):
    """Forward: each pair is a d-term fma chain (k = d) of magnitude sum|T_i||T_j|.  Backward:
    dT[i,c] = sum_j dZ[i,j] T[j,c] (+ dR for the x row): k = N + 1.  No atomics: bit-identical on
    a second run."""
    ops = _ops()
    SM = _sm()
    for bwd in (False, True):
        warps = _dot_warps(N, d, bwd)
        grid = min(_cdiv(B, warps), DOT_CTAS_PER_SM * SM)
        assert_loops("dot_interact %s B=%d N=%d d=%d (%d warps/CTA): samples per warp"
                     % ("bwd" if bwd else "fwd", B, N, d, warps), B // (grid * warps))
    g = torch.Generator(device=DEV).manual_seed(B + N + d + self_interaction)
    T = torch.randn(B, N, d, generator=g, device=DEV)
    dR = torch.randn(B, ops.dot_interact_width(N, d, self_interaction), generator=g, device=DEV)
    R = ops.raw_dot_interact_fwd(T, self_interaction)
    dT = ops.raw_dot_interact_bwd(T, dR, self_interaction)
    wR, mR, wT, mT = _dot_ref(T, dR, self_interaction)
    assert_within(R, wR, d * U * mR + 1e-30, "dot_interact fwd")
    assert_within(dT, wT, (N + 1) * U * mT + 1e-30, "dot_interact bwd")
    assert torch.equal(R[:, :d], T[:, N - 1])
    assert torch.equal(ops.raw_dot_interact_fwd(T, self_interaction), R)
    assert torch.equal(ops.raw_dot_interact_bwd(T, dR, self_interaction), dT)


@pytest.mark.skipif(os.environ.get("B200REC_TEST_EXPERIMENTAL") != "1",
                    reason="experimental K6 v2 kernels: opt in with B200REC_TEST_EXPERIMENTAL=1")
@pytest.mark.parametrize("self_interaction", [False, True])
def test_dot_interact_v2_matches_v1_when_warps_loop(self_interaction, monkeypatch):
    """v2's cp.async double buffer is only used when a warp loops: B=65536 makes every warp run
    ~15 samples.  Same products in the same order: bit-identical to v1."""
    ops = _ops()
    B, N, d = 65536, 27, 16
    g = torch.Generator(device=DEV).manual_seed(27 + self_interaction)
    T = torch.randn(B, N, d, generator=g, device=DEV)
    dR = torch.randn(B, ops.dot_interact_width(N, d, self_interaction), generator=g, device=DEV)
    monkeypatch.delenv("B200REC_K6_V2", raising=False)
    R1, dT1 = ops.raw_dot_interact_fwd(T, self_interaction), ops.raw_dot_interact_bwd(T, dR, self_interaction)
    monkeypatch.setenv("B200REC_K6_V2", "1")
    R2, dT2 = ops.raw_dot_interact_fwd(T, self_interaction), ops.raw_dot_interact_bwd(T, dR, self_interaction)
    assert torch.equal(R1, R2) and torch.equal(dT1, dT2)


# ================================================================================================
# 5. CrossNet K3 (cross.cuh): row slices accumulate the bias gradient over many rows
# ================================================================================================
@pytest.mark.parametrize("C", [1560, 351])
def test_cross_v2_at_scale(C):
    """B=65536: each of the 264 row slices of cross_v2_bwd_kernel walks ~248 rows.
    dxw = dout*x0 and dx0 = dout*(xw + bias) are single correctly-rounded fp32 operations: equal to
    torch's fp32 result bit for bit (hence within 2^-24 relative of fp64).
    out = fmaf(x0, xw + bias, xl): 2 roundings of |x0|(|xw| + |bias|) + |xl|.
    dbias: each slice adds ceil(B/264) rows in order, reduce_partials_kernel adds ceil(264/32)
    per lane then 32 lanes: k = ceil(B/264) + 9 + 32 + 1 of sum|dout x0|."""
    ops = _ops()
    B = 65536
    vec = 4 if C % 4 == 0 else 1
    assert_loops("cross_v2_bwd_kernel C=%d: rows per slice" % C, B // CROSS_ROW_SLICES)
    total = B * (C // vec)
    grid = min(_cdiv(total, 256), 16 * _sm())
    assert_loops("cross_v2_fwd_kernel C=%d: elements per thread" % C, total // (grid * 256))
    g = torch.Generator(device=DEV).manual_seed(C)
    x0, xl, xw, dout = (torch.randn(B, C, generator=g, device=DEV) for _ in range(4))
    bias = torch.randn(C, generator=g, device=DEV)
    out = ops.raw_cross_v2_fwd(x0, xl, xw, bias)
    d = lambda t: t.double()  # noqa: E731
    assert_within(out, d(xl) + d(x0) * (d(xw) + d(bias)),
                  2 * U * (d(x0).abs() * (d(xw).abs() + d(bias).abs()) + d(xl).abs()), "cross fwd")
    del out
    dxw, dx0, dbias = ops.raw_cross_v2_bwd(dout, x0, xw, bias)
    assert torch.equal(dxw, dout * x0)
    assert torch.equal(dx0, dout * (xw + bias))
    k = _cdiv(B, CROSS_ROW_SLICES) + _cdiv(CROSS_ROW_SLICES, RED_LANES) + RED_LANES + 1
    prod = d(dout) * d(x0)
    assert_within(dbias, prod.sum(0), k * U * prod.abs().sum(0), "cross dbias C=%d" % C)
    assert torch.equal(ops.raw_cross_v2_bwd(dout, x0, xw, bias)[2], dbias)


# ================================================================================================
# 6. tower_relu_bwd_split (tower.cuh): 4-row unrolled main loop + tail, db through 528 slices
# ================================================================================================
@pytest.mark.parametrize("N", [1, 7, 400])
@pytest.mark.parametrize("masked", [False, True])
def test_tower_split_bwd_at_scale(N, masked):
    """raw_tc_split_bwd at M=65536: g = dy * (mask_hi > 0) written as bf16 planes [hi | lo] (bit
    exact: the same two roundings torch does) and db = column sums of g.  A thread walks
    rows = M / row_step rows (row_step = 528 * TY), >= 3 passes of the 4-row unrolled loop plus the
    tail; reduce_partials_kernel runs its 4-in-flight loop over the 528 partials.
    db: k = ceil(M/row_step) + TY (block rows in order) + ceil(528/32) + 32 of sum|g|."""
    ops = _ops()
    M = 65536
    ld = ops.plane_ld(N)
    v4 = N % 4 == 0 and ld % 4 == 0
    chunks = N // 4 if v4 else N
    tx = 32
    while tx < chunks and tx < TOWER_THREADS:
        tx <<= 1
    ty = TOWER_THREADS // tx
    row_step = min(TOWER_ROW_SLICES, M) * ty
    assert_loops("tower_relu_bwd_split N=%d: unrolled 4-row passes per thread" % N,
                 (M // row_step) // TOWER_UNROLL)
    assert (M // row_step) % TOWER_UNROLL != 0, "the tail loop should run too"
    assert_loops("reduce_partials_kernel over %d partials: 4-in-flight passes of lane 0"
                 % TOWER_ROW_SLICES, len(range(0, TOWER_ROW_SLICES - 3 * RED_LANES, 4 * RED_LANES)))
    g = torch.Generator(device=DEV).manual_seed(N + masked)
    dy = torch.randn(M, N, generator=g, device=DEV)
    mp = ops.raw_tc_split(torch.randn(M, N, generator=g, device=DEV).clamp_min(0)) if masked else None
    gp, db = ops.raw_tc_split_bwd(dy, mp)
    gw = torch.where(mp[:, :N].float() > 0, dy, torch.zeros_like(dy)) if masked else dy
    hi = gw.to(torch.bfloat16)
    lo = (gw - hi.float()).to(torch.bfloat16)
    assert torch.equal(gp[:, :N], hi) and torch.equal(gp[:, ld:ld + N], lo)
    k = _cdiv(M, row_step) + ty + _cdiv(TOWER_ROW_SLICES, RED_LANES) + RED_LANES
    assert_within(db, gw.double().sum(0), k * U * gw.double().abs().sum(0), "split bwd db N=%d" % N)
    assert torch.equal(ops.raw_tc_split_bwd(dy, mp)[1], db)
    if masked and N == 400:       # the older entry point shares the launcher: same planes and db
        act = ops.raw_tower_split(torch.randn(M, N, generator=g, device=DEV), None, True)
        dz, db2 = ops.raw_tower_relu_bwd_split(dy, act)
        gw2 = torch.where(act[:, :N].float() > 0, dy, torch.zeros_like(dy))
        hi2 = gw2.to(torch.bfloat16)
        assert torch.equal(dz[:, :N], hi2) and torch.equal(dz[:, N:], (gw2 - hi2.float()).to(torch.bfloat16))
        assert_within(db2, gw2.double().sum(0), k * U * gw2.double().abs().sum(0), "tower bwd db")


# ================================================================================================
# 7. Row updates (gather_scatter.cuh) at U ~ 3x the grid's capacity, against oracle/optim.py
# ================================================================================================
@pytest.mark.parametrize("D", [9, 16])
def test_row_updates_at_scale(D):
    """row_update_kernel / row_adagrad_kernel: grid = min(ceil(U/GPB), 64*SM), so each lane group
    updates >= 3 rows.  Bounds (per element, u = 2^-24):
      sgd      fmaf(-lr, g, w) with lr rounded to fp32: 2u (|w| + |lr g|)
      adam     m: 3 roundings + 2 fp32 parameters per step -> 10u of m's magnitude after 2 steps;
               v: 12u (all terms positive); w: per step 1u |w| plus the update lr_t m/(sqrt v + eps)
               with m's error and 16 roundings (sqrt, add, div, mul, sub, lr_t, eps_t, half of v's)
      adagrad  g2sum: (D + 8)u per step (positive terms); w: per step 1u |w| + (D + 16)u |lr g s|
      rows_to_dense  zeros + g: exact copies
    Untouched rows (and their moments) must stay bit-identical."""
    ops = _ops()
    vec, tpr = row_shape(D)
    gpb = ROW_THREADS // tpr
    cap = 64 * _sm() * gpb
    Uq = 3 * cap + 77
    grid = min(_cdiv(Uq, gpb), 64 * _sm())
    assert_loops("row updates D=%d: rows per lane group" % D, Uq // (grid * gpb))
    V = Uq + Uq // 4
    g = torch.Generator(device=DEV).manual_seed(D)
    rows = torch.randperm(V, generator=g, device=DEV)[:Uq].sort().values
    val = torch.randn(Uq, D, generator=g, device=DEV)
    num = torch.tensor([Uq, Uq], dtype=torch.int32, device=DEV)
    sr = ops.SelectedRows(rows, val, num, V)
    untouched = torch.ones(V, dtype=torch.bool, device=DEV)
    untouched[rows] = False
    W0 = torch.randn(V, D, generator=g, device=DEV)
    Wh = W0[rows].double().cpu().numpy()
    gh = val.double().cpu().numpy()
    idx = np.arange(Uq)
    t64 = lambda a: torch.from_numpy(a).to(DEV)  # noqa: E731

    dense = sr.to_dense()
    assert torch.equal(dense[rows], val) and not dense[untouched].any()
    del dense

    W = W0.clone()
    ops.raw_sparse_sgd(W, sr, 0.1)
    want = t64(ooptim.sgd(Wh, idx, gh, 0.1))
    assert_within(W[rows], want, 2 * U * (want.abs() + 0.1 * t64(gh).abs()), "sgd")
    assert torch.equal(W[untouched], W0[untouched])

    W, m, v = W0.clone(), torch.zeros_like(W0), torch.zeros_like(W0)
    Wr, mr, vr = Wh, np.zeros_like(Wh), np.zeros_like(Wh)
    mm = np.zeros_like(Wh)
    upd_mag = np.zeros_like(Wh)
    b1, b2, eps, lr = 0.9, 0.999, 1e-8, 1e-3
    for t in (1, 2):
        ops.raw_sparse_adam(W, m, v, sr, lr, b1, b2, eps, b1 ** t, b2 ** t)
        Wr, mr, vr = ooptim.adam_lazy(Wr, mr, vr, idx, gh, lr, b1, b2, eps, t)
        mm = b1 * mm + (1 - b1) * np.abs(gh)
        lr_t = lr * np.sqrt(1 - b2 ** t) / (1 - b1 ** t)
        upd_mag += lr_t * (10 * mm + 16 * np.abs(mr)) / (np.sqrt(vr) + eps * np.sqrt(1 - b2 ** t))
    assert_within(m[rows], t64(mr), 10 * U * t64(mm), "adam m")
    assert_within(v[rows], t64(vr), 12 * U * t64(vr), "adam v")
    assert_within(W[rows], t64(Wr), U * (2 * t64(np.abs(Wr)) + t64(upd_mag)), "adam W")
    assert torch.equal(W[untouched], W0[untouched])
    assert not m[untouched].any() and not v[untouched].any()

    W, g2 = W0.clone(), torch.zeros(V, device=DEV)
    Wr, g2r = Wh, np.zeros(Uq)
    upd_mag = np.zeros_like(Wh)
    lr, g0, lo, hi = 0.05, 3.0, -2.5, 2.5
    for _ in range(2):
        upd_mag += (D + 16) * lr * np.abs(gh) * np.sqrt(g0 / (g0 + g2r))[:, None]
        ops.raw_sparse_adagrad(W, g2, sr, lr, g0, lo, hi)
        Wr, g2r = ooptim.adagrad_row(Wr, g2r, idx, gh, lr, g0, lo, hi)
    assert_within(g2[rows], t64(g2r), 2 * (D + 8) * U * t64(g2r), "adagrad g2sum")
    assert_within(W[rows], t64(Wr), U * (2 * t64(np.abs(Wr)) + t64(upd_mag)), "adagrad W")
    assert torch.equal(W[untouched], W0[untouched]) and not g2[untouched].any()


# ================================================================================================
# 8. gather_pool_sum (gather_scatter.cuh) forward with n_bags ~ 3x capacity, and its backward
# ================================================================================================
@pytest.mark.parametrize("D", [9, 16])
def test_gather_pool_sum_at_scale(D):
    """gather_pool_kernel: one lane group per bag, grid = min(ceil(n_bags/GPB), 64*SM), so each group
    pools >= 3 bags.  A bag of len keys is a chain of len adds: k = len of sum|W rows|.  Empty bags
    are exactly 0; padding and out-of-range keys are skipped (and counted).  Backward: the pooled
    gradient through raw_segment_reduce(row_of_pos=bag_of_pos) with a hot key of many chunks,
    seg_chain bound, bit-reproducible."""
    ops = _ops()
    vec, tpr = row_shape(D)
    gpb = ROW_THREADS // tpr
    cap = 64 * _sm() * gpb
    n_bags = 3 * cap + 123
    grid = min(_cdiv(n_bags, gpb), 64 * _sm())
    assert_loops("gather_pool_kernel D=%d: bags per lane group" % D, n_bags // (grid * gpb))
    V = 100_000
    g = torch.Generator(device=DEV).manual_seed(D)
    lens = torch.randint(0, 6, (n_bags,), generator=g, device=DEV)
    lens[::97] = 0
    offsets = torch.zeros(n_bags + 1, dtype=torch.int64, device=DEV)
    offsets[1:] = torch.cumsum(lens, 0)
    nnz = int(offsets[-1])
    keys = torch.randint(0, V, (nnz,), generator=g, device=DEV)
    keys[::25] = 17
    keys[5::1001] = V + 3
    W = torch.randn(V, D, generator=g, device=DEV)
    ops.raw_oob_count()
    out, bag_of_pos = ops.raw_gather_pool_sum(W, keys, offsets, 0)
    assert ops.raw_oob_count() == int((keys >= V).sum())
    bag = torch.arange(n_bags, device=DEV).repeat_interleave(lens)
    assert torch.equal(bag_of_pos[:nnz], bag.to(torch.int32))
    ok = (keys != 0) & (keys < V)
    Wd = W.double()
    want = torch.zeros(n_bags, D, dtype=torch.float64, device=DEV).index_add_(0, bag[ok], Wd[keys[ok]])
    mag = torch.zeros_like(want).index_add_(0, bag[ok], Wd[keys[ok]].abs())
    assert_within(out, want, lens.double().unsqueeze(1) * U * mag + 1e-30, "gather_pool_sum D=%d" % D)
    assert not out[lens == 0].any()
    # backward
    dout = torch.randn(n_bags, D, generator=g, device=DEV)
    gr = ops.raw_group_ids(keys, V, 0)
    counts = _check_segment_rows(
        ops, gr, lambda: ops.raw_segment_reduce(dout, gr.seg_offsets, gr.sorted_pos, gr.num, nnz,
                                                row_of_pos=bag_of_pos),
        dout.double()[bag[ok]], keys[ok], D, "gather_pool_sum backward D=%d" % D)
    assert_loops("pooled backward: chunks of the hot key", _cdiv(int(counts.max()), HOT_CHUNK))


# ================================================================================================
# 9. embed_fm forward (embed_fm.cuh): persistent tiles with the double-buffered id prefetch
# ================================================================================================
@pytest.mark.parametrize("D", [9, 16, 40])
@pytest.mark.parametrize("fused", [False, True])
def test_embed_fm_fwd_at_scale(D, fused):
    """B >= 65536 (more for D=16, so that every CTA runs >= 3 tiles: grid = min(tiles, 8*SM),
    tile = 128/TPR samples), V=1e6.  The WHOLE feat is compared with torch.equal (gathers are
    copies; dense rows one fp32 product).  S: N-term sums, k = N of sum|feat|; y1: N terms, one of
    which a product, k = N + 2; y2 = 0.5 sum_d (S_d^2 - Q_d): the S error doubles through the
    square, so k = 4N + 2D + 8 of 0.5 sum_d ((sum_f |feat|)^2 + Q_d)."""
    ops = _ops()
    SM = _sm()
    F, Dn, V = 26, 13, 1_000_000
    N = F + Dn
    _, tpr = row_shape(D)
    spb = FWD_THREADS // tpr
    B = max(65536, 3 * FWD_CTAS_PER_SM * SM * spb)
    tiles = _cdiv(B, spb)
    grid = min(tiles, FWD_CTAS_PER_SM * SM)
    assert_loops("embed_fm_fwd_kernel D=%d B=%d: tiles per CTA" % (D, B), tiles // grid)
    g = torch.Generator(device=DEV).manual_seed(D + 100 * fused)
    ids = torch.randint(1, V, (B, F), generator=g, device=DEV)
    ids[torch.rand(B, F, generator=g, device=DEV) < 0.02] = 0
    dense = torch.rand(B, Dn, generator=g, device=DEV)
    W = torch.randn(V, D, generator=g, device=DEV) * 0.1
    W1 = torch.randn(V, 1, generator=g, device=DEV) * 0.1
    dense_w = torch.randn(Dn, D, generator=g, device=DEV) * 0.1
    dense_w1 = torch.randn(Dn, generator=g, device=DEV) * 0.1
    ops.raw_oob_count()
    if fused:
        Wf = torch.full((V, ops.fused_slot(D)), 123.0, device=DEV)
        Wf[:, :D] = W
        Wf[:, D] = W1[:, 0]
        feat, y1, y2, S = ops.raw_embed_fm_fwd(Wf, None, ids, dense, dense_w, dense_w1, 0, D=D)
        del Wf
    else:
        feat, y1, y2, S = ops.raw_embed_fm_fwd(W, W1, ids, dense, dense_w, dense_w1, 0)
    live = (ids != 0).unsqueeze(2)
    assert torch.equal(feat[:, :F], W[ids] * live)
    assert torch.equal(feat[:, F:], dense.unsqueeze(2) * dense_w.unsqueeze(0))
    assert ops.raw_oob_count() == 0
    f = feat.double()
    assert_within(S, f.sum(1), N * U * f.abs().sum(1), "S")
    t1 = torch.cat([(W1[ids, 0] * (ids != 0)).double(), dense.double() * dense_w1.double()], 1)
    assert_within(y1, t1.sum(1), (N + 2) * U * t1.abs().sum(1), "y1")
    Sd, Q = f.sum(1), f.square().sum(1)
    A = f.abs().sum(1)
    assert_within(y2, 0.5 * (Sd.square() - Q).sum(1),
                  (4 * N + 2 * D + 8) * U * 0.5 * (A.square() + Q).sum(1), "y2")


# ================================================================================================
# 10. hash_keys and cvm (grid-stride over 16*SM CTAs of 256 threads)
# ================================================================================================
def test_hash_keys_at_scale():
    """n = 4M keys: every thread folds >= 3 keys.  Bit-exact against oracle/readers.hash_keys."""
    from oracle import readers
    ops = _ops()
    n = 4 << 20
    assert_loops("hash_keys_kernel: keys per thread", n // (STREAM_CTAS_PER_SM * _sm() * 256))
    rng = np.random.default_rng(4)
    keys = rng.integers(0, 1 << 63, n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, n, dtype=np.uint64)
    keys[::1000] = 0
    slots = rng.integers(0, 26, n).astype(np.int32)
    kd = torch.from_numpy(keys).to(DEV)
    for V, sl, rz in ((1_000_003, slots, True), ((1 << 40) + 7, None, False)):
        got = ops.raw_hash_keys(kd, V, None if sl is None else torch.from_numpy(sl).to(DEV), rz)
        assert np.array_equal(got.cpu().numpy(), readers.hash_keys(keys, V, sl, rz))


@pytest.mark.parametrize("use_cvm", [False, True])
def test_cvm_at_scale(use_cvm):
    """N = 1.7M rows of D+2 = 13: every thread handles >= 3 elements.  Copies are bit-exact; the
    two log columns: logf(x + 1) is within 1 ulp after one rounded add, so each is within
    2u(1 + |log|) and their difference within 4u(1 + |log(x0+1)| + |log(x1+1)|)."""
    ops = _ops()
    N, D = 1_700_000, 11
    out_w = D + 2 if use_cvm else D
    assert_loops("cvm_fwd_kernel: elements per thread", N * out_w // (STREAM_CTAS_PER_SM * _sm() * 256))
    g = torch.Generator(device=DEV).manual_seed(11)
    x = torch.rand(N, D + 2, generator=g, device=DEV) * 5
    y = ops.raw_cvm_fwd(x, use_cvm)
    assert torch.equal(y[:, -D:], x[:, 2:])
    if use_cvm:
        ref = nets.cvm(x.double(), True)
        l0, l1 = torch.log1p(x[:, 0].double()), torch.log1p(x[:, 1].double())
        bound = (4 * U * (1 + l0.abs() + l1.abs())).unsqueeze(1).expand(N, 2)
        assert_within(y[:, :2], ref[:, :2], bound, "cvm log columns")
    sc = torch.rand(N, 2, generator=g, device=DEV) * 3
    dy = torch.randn(N, out_w, generator=g, device=DEV)
    assert_loops("cvm_bwd_kernel: elements per thread", N * (D + 2) // (STREAM_CTAS_PER_SM * _sm() * 256))
    dx = ops.raw_cvm_bwd(dy, sc, D, use_cvm)
    assert torch.equal(dx[:, :2], sc) and torch.equal(dx[:, 2:], dy[:, -D:])


# ================================================================================================
# 11. FFM (ffm.cuh): persistent forward, light / hot / combine backward, dense-gradient slices
# ================================================================================================
def ffm_staged_cols(R):
    """ffm_staged_cols, ffm.cuh:22: [R | w1 | pad] rounded up to 4 floats."""
    return (R + 1 + 3) // 4 * 4


def ffm_fwd_smem(F, Dn, D, nbuf):
    """FfmFwdSmem(F, Dn, D, nbuf).total, ffm.cuh:26-36."""
    NF = F + Dn
    R, P = NF * D, NF * (NF - 1) // 2
    a16 = lambda x: (x + 15) // 16 * 16  # noqa: E731
    off_pairs = a16(Dn * R * 4)
    off_red = a16(off_pairs + P * 4)
    off_buf = off_red + 16 * (FFM_THREADS // 32 + 4)
    return off_buf + nbuf * F * ffm_staged_cols(R) * 4


def _ffm_feat(W, ids, dense, dense_w, s, e, D, pad):
    """Samples s:e in fp64: e[b, n, :] [b, NF, R] (table rows, zero for padding and out-of-range
    ids; dense rows x * dense_w), the first-order table terms [b, F] and x [b, Dn]."""
    V = W.shape[0]
    F, Dn = ids.shape[1], dense.shape[1]
    R = (F + Dn) * D
    idb = ids[s:e]
    ok = ((idb >= 0) & (idb < V) & (idb != pad)).unsqueeze(2)
    rows = W[idb.clamp(0, V - 1), :R + 1].double() * ok
    x = dense[s:e].double()
    feat = torch.cat([rows[:, :, :R], x.unsqueeze(2) * dense_w.double().unsqueeze(0)], 1)
    return feat, rows[:, :, R], x


def _ffm_table(V, R, g):
    """Fused rows [R emb | w1 | 123...]: the slot's padding must never be read."""
    ops = _ops()
    W = torch.full((V, ops.fused_slot(R)), 123.0, device=DEV)
    W[:, :R + 1] = torch.randn(V, R + 1, generator=g, device=DEV) * 0.1
    return W


@pytest.mark.parametrize("F,Dn,D,B,nbuf", [
    (26, 13, 22, None, 2),     # the largest double-buffered shape at F=26, Dn=13
    (26, 13, 23, None, 1),     # the smallest single-buffered one
    (26, 13, 16, 65536, 2),
    (26, 0, 9, None, 2),       # no dense fields
    (40, 24, 1, None, 2),      # F+Dn = 64 fields: P = 2016 pairs, 8 per thread
    (26, 13, 1, None, 2),
])
def test_ffm_fwd_at_scale(F, Dn, D, B, nbuf):
    """ffm_fwd_kernel: persistent CTAs, grid = min(B, SM*per_sm) with per_sm <= 2048/256 = 8
    (ffm.cuh:176-179), so B >= 3*8*SM + 17 makes every CTA take >= 3 samples: with two buffers
    every CTA stages into both and prefetches across iterations.  The buffering the case gets is
    asserted from the FfmFwdSmem mirror against the device's opt-in shared-memory limit.
    y2: each pair is a D-fma dot (D roundings), scaled by sa*sc (1) and fma'd into the thread's
    accumulator of ceil(P/256) pairs, then 5 shuffle levels and 8 warp partials in order:
    k = D + ceil(P/256) + 15 of sum over pairs of |e[n, block m]| . |e[m, block n]|.
    y1: F adds of w1, Dn fmas of x*dense_w1, one add of the two and one of the bias: k = F + Dn + 2.
    Padding, negative and >= V ids stage zero rows; raw_oob_count counts each out-of-range
    position exactly once; a second run is bit-identical."""
    ops = _ops()
    SM = _sm()
    NF = F + Dn
    R, P = NF * D, NF * (NF - 1) // 2
    assert NF <= FFM_MAX_FIELDS
    limit = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    if nbuf == 2:
        assert ffm_fwd_smem(F, Dn, D, 2) <= limit, "F=%d Dn=%d D=%d no longer double-buffered" % (F, Dn, D)
    else:
        assert ffm_fwd_smem(F, Dn, D, 2) > limit >= ffm_fwd_smem(F, Dn, D, 1), \
            "F=%d Dn=%d D=%d is no longer the single-buffered case" % (F, Dn, D)
    B = B or 3 * FFM_FWD_MAX_CTAS_PER_SM * SM + 17
    assert_loops("ffm_fwd_kernel F=%d Dn=%d D=%d (%d buffers): samples per CTA" % (F, Dn, D, nbuf),
                 B // (FFM_FWD_MAX_CTAS_PER_SM * SM))
    V, pad = 20_000, 0
    g = torch.Generator(device=DEV).manual_seed(1000 * D + NF)
    W = _ffm_table(V, R, g)
    ids = torch.randint(1, V, (B, F), generator=g, device=DEV)
    r = torch.rand(B, F, generator=g, device=DEV)
    ids[r < 0.03] = pad
    ids[(r >= 0.03) & (r < 0.035)] = -1 - torch.randint(0, 5, (B, F), generator=g, device=DEV)[
        (r >= 0.03) & (r < 0.035)]
    ids[(r >= 0.035) & (r < 0.04)] = V + torch.randint(0, 5, (B, F), generator=g, device=DEV)[
        (r >= 0.035) & (r < 0.04)]
    n_oob = int(((ids < 0) | (ids >= V)).sum())
    assert n_oob > 0 and int((ids == pad).sum()) > 0
    dense = torch.rand(B, Dn, generator=g, device=DEV)
    dense_w = torch.randn(Dn, R, generator=g, device=DEV) * 0.1
    dense_w1 = torch.randn(Dn, generator=g, device=DEV) * 0.1
    bias = torch.tensor([0.3], device=DEV)

    ops.raw_oob_count()
    y1, y2 = ops.raw_ffm_fwd(W, ids, dense, dense_w, dense_w1, bias, pad, D)
    assert ops.raw_oob_count() == n_oob

    f64 = dict(dtype=torch.float64, device=DEV)
    w1, m1, w2, m2 = (torch.empty(B, **f64) for _ in range(4))
    iu = torch.triu_indices(NF, NF, 1, device=DEV)
    chunk = max(1, (1 << 24) // (NF * R))
    for s in range(0, B, chunk):
        e = min(B, s + chunk)
        feat, first, x = _ffm_feat(W, ids, dense, dense_w, s, e, D, pad)
        e4 = feat.view(e - s, NF, NF, D)
        prod = e4[:, iu[0], iu[1]] * e4[:, iu[1], iu[0]]
        w2[s:e], m2[s:e] = prod.sum((1, 2)), prod.abs().sum((1, 2))
        t1 = torch.cat([first, x * dense_w1.double()], 1)
        w1[s:e], m1[s:e] = t1.sum(1) + float(bias), t1.abs().sum(1) + abs(float(bias))
    del feat, e4, prod
    what = "ffm fwd F=%d Dn=%d D=%d B=%d" % (F, Dn, D, B)
    assert_within(y2, w2, (D + _cdiv(P, FFM_THREADS) + 15) * U * m2 + 1e-30, what + " y2")
    assert_within(y1, w1, (F + Dn + 2) * U * m1 + 1e-30, what + " y1")
    y1b, y2b = ops.raw_ffm_fwd(W, ids, dense, dense_w, dense_w1, bias, pad, D)
    assert ops.raw_oob_count() == n_oob
    assert torch.equal(y1, y1b) and torch.equal(y2, y2b), what + ": not bit-reproducible"


FFM_BWD_LENS = [64, 65, 1024, 1025, 2048, 2049, 150001]   # ids 1..7; 150001 = 147 hot chunks
FFM_LIGHT_LO = 10_000                                     # light traffic uses ids FFM_LIGHT_LO..V-1


def _ffm_bwd_ids(B, F, V, g):
    """[B, F] ids: ids 1..7 with exactly FFM_BWD_LENS positions; 3*8*SM + 50 ids (100, 101, ...)
    of 65-300 positions each; 5000 padding positions (id 0, so padding sits inside the hot runs);
    40 positions each of V+3 and -2; the rest uniform over [FFM_LIGHT_LO, V), all shuffled."""
    n = B * F
    n_hot = 3 * FFM_HOT_CTAS_PER_SM * _sm() + 50
    parts = [torch.full((c,), 1 + i, dtype=torch.int64, device=DEV) for i, c in enumerate(FFM_BWD_LENS)]
    lens = torch.randint(HOT_THRESHOLD + 1, 301, (n_hot,), generator=g, device=DEV)
    parts.append(torch.arange(100, 100 + n_hot, device=DEV).repeat_interleave(lens))
    parts.append(torch.zeros(5000, dtype=torch.int64, device=DEV))
    parts.append(torch.full((40,), V + 3, dtype=torch.int64, device=DEV))
    parts.append(torch.full((40,), -2, dtype=torch.int64, device=DEV))
    used = sum(p.numel() for p in parts)
    parts.append(torch.randint(FFM_LIGHT_LO, V, (n - used,), generator=g, device=DEV))
    ids = torch.cat(parts)
    return ids[torch.randperm(n, generator=g, device=DEV)].reshape(B, F)


def ffm_bwd_chain(counts):
    """Longest fp32 chain of the columns < R of one gradient row, from its segment length
    (ffm.cuh:265-365); every term g2 * partner is itself up to 2 roundings (a dense partner is
    x * dense_w).  Light (<= 64 positions): one lane adds the segment in order, len + 2.  Hot, one
    chunk: each of 8 warps adds ceil(len/8) positions, the 8 warp sums meet in order,
    ceil(len/8) + 8 + 2.  Several chunks: 1024/8 = 128 per warp, 8 warp sums, then the combine
    adds the chunk partials in order, 128 + 8 + chunks + 2."""
    wpb = FFM_THREADS // 32
    chunks = (counts + FFM_HOT_CHUNK - 1) // FFM_HOT_CHUNK
    k_one = (counts + wpb - 1) // wpb + wpb + 2
    k_many = FFM_HOT_CHUNK // wpb + wpb + chunks + 2
    return torch.where(counts <= HOT_THRESHOLD, counts + 2,
                       torch.where(chunks == 1, k_one, k_many)).double()


@pytest.mark.parametrize("Dn,D,B", [(13, 9, 65536), (13, 16, 65536), (13, 16, 65536 - 100),
                                    (0, 9, 65536)])
def test_ffm_bwd_at_scale(Dn, D, B):
    """raw_ffm_bwd at B*F = 1.7M positions, F=26, V=200k, ids built by _ffm_bwd_ids so that
    every light warp walks >= 3 distinct ids, every hot CTA takes >= 3 work items, and the combine
    adds the 147 chunks of the 150001-position id.  Every row of every distinct id is checked
    element-wise against the per-position contributions g2[b] * e[b, m, block f] (m != f) and
    g1[b] merged in fp64 with index_add, bound ffm_bwd_chain(len) for columns < R and 2 less for
    column R (g1 terms are not rounded); columns R+1..G-1 must be exactly 0.
    Dense gradients (ffm.cuh:367-408): each of the `slices` = min(256, ceil(B/256)) slices sums
    per_slice samples with fmaf(g2*x, partner, acc) (+2 roundings per term, +1 for a dense partner's
    x*dense_w), then the slice partials are added in order: ddense_w k = per_slice + 3 + slices,
    ddense_w1 k = per_slice + 1 + slices, dbias k = per_slice + slices.  B = 65436 leaves the last
    slice short.  Every output is bit-identical on a second run."""
    ops = _ops()
    SM = _sm()
    F, V, pad = 26, 200_000, 0
    NF = F + Dn
    R = NF * D
    G = ffm_staged_cols(R)
    n = B * F
    g = torch.Generator(device=DEV).manual_seed(100 * D + Dn + B)
    ids = _ffm_bwd_ids(B, F, V, g)
    flat = ids.reshape(-1)
    valid = (flat >= 0) & (flat < V) & (flat != pad)
    uniq, inv, counts = torch.unique(flat[valid], return_inverse=True, return_counts=True)
    Uq = uniq.numel()
    # the loop counts the construction gives
    assert sorted(counts[counts > 300].tolist()) == sorted(c for c in FFM_BWD_LENS if c > 300)
    wpb = FFM_THREADS // 32
    n_light = int((counts <= HOT_THRESHOLD).sum())
    assert n_light >= 3 * FFM_LIGHT_CTAS_PER_SM * SM * wpb
    lgrid = min(_cdiv(n, wpb), FFM_LIGHT_CTAS_PER_SM * SM)
    assert_loops("ffm_bwd_light_kernel: distinct ids per warp", Uq // (lgrid * wpb))
    hot = counts[counts > HOT_THRESHOLD]
    n_items = int(((hot + FFM_HOT_CHUNK - 1) // FFM_HOT_CHUNK).sum())
    max_items = n // (HOT_THRESHOLD + 1) + 1
    hgrid = min(max_items, FFM_HOT_CTAS_PER_SM * SM)
    assert_loops("ffm_bwd_hot_kernel: work items per CTA", n_items // hgrid)
    assert_loops("ffm_bwd_combine_kernel: chunks of the 150001-position id",
                 _cdiv(FFM_BWD_LENS[-1], FFM_HOT_CHUNK))
    slices = min(FFM_MAX_SLICES, _cdiv(B, 256))
    per_slice = _cdiv(B, slices)
    assert_loops("ffm_bwd_dense_kernel: samples per slice", per_slice)

    W = _ffm_table(V, R, g)
    dense = torch.rand(B, Dn, generator=g, device=DEV)
    dense_w = torch.randn(Dn, R, generator=g, device=DEV) * 0.1
    gy1 = torch.randn(B, generator=g, device=DEV)
    gy2 = torch.randn(B, generator=g, device=DEV)
    groups = ops.raw_group_ids(ids, V, pad)
    assert int(groups.num[0]) == Uq
    assert torch.equal(groups.unique_ids[:Uq], uniq), "the gradient rows must be exactly the valid ids"
    out = ops.raw_ffm_bwd(W, ids, dense, dense_w, gy1, gy2, groups, pad, D)
    out2 = ops.raw_ffm_bwd(W, ids, dense, dense_w, gy1, gy2, groups, pad, D)
    what = "ffm bwd Dn=%d D=%d B=%d" % (Dn, D, B)
    assert torch.equal(out[0][:Uq], out2[0][:Uq]), what + ": rows not bit-reproducible"
    for a, b in zip(out[1:], out2[1:]):
        assert torch.equal(a, b), what + ": dense gradients not bit-reproducible"
    del out2
    dW, ddw, ddw1, db = out

    f64 = dict(dtype=torch.float64, device=DEV)
    pos_row = torch.full((n,), -1, dtype=torch.int64, device=DEV)
    pos_row[valid] = inv
    want, mag = torch.zeros(Uq, R + 1, **f64), torch.zeros(Uq, R + 1, **f64)
    wdw, mdw = torch.zeros(Dn, NF, D, **f64), torch.zeros(Dn, NF, D, **f64)
    wd1, md1 = torch.zeros(Dn, **f64), torch.zeros(Dn, **f64)
    ar = torch.arange(NF, device=DEV)
    off = (ar[:F].unsqueeze(1) != ar).double().reshape(1, F, NF, 1)          # m != f
    offd = (ar[F:].unsqueeze(1) != ar).double().unsqueeze(2)                  # m != F+k
    chunk = 1024
    for s in range(0, B, chunk):
        e = min(B, s + chunk)
        b = e - s
        feat, _, x = _ffm_feat(W, ids, dense, dense_w, s, e, D, pad)
        e4 = feat.view(b, NF, NF, D)                       # e4[b, m, f] = e[b, m, block f]
        g2, g1 = gy2[s:e].double(), gy1[s:e].double()
        t = e4.transpose(1, 2)[:, :F] * off * g2.view(b, 1, 1, 1)
        t = torch.cat([t.reshape(b * F, R), g1.repeat_interleave(F).unsqueeze(1)], 1)
        r = pos_row[s * F:e * F]
        ok = r >= 0
        want.index_add_(0, r[ok], t[ok])
        mag.index_add_(0, r[ok], t[ok].abs())
        del t
        if Dn:
            term = e4[:, :, F:] * (g2.unsqueeze(1) * x).view(b, 1, Dn, 1)    # [b, m, k, D]
            wdw += term.sum(0).transpose(0, 1) * offd
            mdw += term.abs().sum(0).transpose(0, 1) * offd
            wd1 += (g1.unsqueeze(1) * x).sum(0)
            md1 += (g1.abs().unsqueeze(1) * x.abs()).sum(0)
    del feat, e4
    k = ffm_bwd_chain(counts).unsqueeze(1)
    for r0 in range(0, Uq, 32768):
        sl = slice(r0, min(Uq, r0 + 32768))
        bound = k[sl] * U * mag[sl]
        bound[:, R] -= 2 * U * mag[sl, R]
        assert_within(dW[sl, :R + 1], want[sl], bound + 1e-30, what + " rows %d.." % r0)
    assert not dW[:Uq, R + 1:G].any(), what + ": the padding columns of the rows must be 0"
    del want, mag
    if Dn:
        assert_within(ddw, wdw.reshape(Dn, R), (per_slice + 3 + slices) * U * mdw.reshape(Dn, R) + 1e-30,
                      what + " ddense_w")
        assert_within(ddw1, wd1, (per_slice + 1 + slices) * U * md1 + 1e-30, what + " ddense_w1")
    assert_within(db, gy1.double().sum().reshape(1),
                  (per_slice + slices) * U * gy1.double().abs().sum().reshape(1), what + " dbias")


def test_ffm_bwd_chunk_packing_limit():
    """Work items pack chunk | (chunks << 16) into one int32 (ffm.cuh:287), which the launcher
    bounds by B*F < 32767*1024 (ffm.cuh:465).  At F=1, Dn=0, D=1 and B*F = 32767*1024 - 1, id 1
    takes 32766*1024 + 512 positions (32767 chunks: chunk index 32766, chunks << 16 =
    2,147,418,112), all with gy1 = 1.0; the other 511 positions go to distinct ids.  Each full chunk
    sums to exactly 1024 (8 warps of 128 ones), and every partial total of the combine is an even
    integer below 2^25, so id 1's g1 column must be exactly 32766*1024 + 512: a dropped or
    duplicated chunk shows.  The single-position rows hold their gy1 exactly.  dbias:
    k = per_slice + slices.  One more position, with every buffer sized for it, is refused with
    B200REC_ERR_INVALID naming B*F."""
    import ctypes
    from paddlerec_b200 import _lib
    ops = _ops()
    lib = _lib.load()
    SM = _sm()
    n_max = FFM_MAX_CHUNKS * FFM_HOT_CHUNK        # the first B*F the launcher refuses
    n = n_max - 1
    n_a = (FFM_MAX_CHUNKS - 1) * FFM_HOT_CHUNK + FFM_HOT_CHUNK // 2
    chunks = _cdiv(n_a, FFM_HOT_CHUNK)
    assert chunks == FFM_MAX_CHUNKS and chunks - 1 < 1 << 16 and chunks << 16 == 2_147_418_112
    assert n_a < 1 << 25 and n_a % 2 == 0
    hgrid = min(n // (HOT_THRESHOLD + 1) + 1, FFM_HOT_CTAS_PER_SM * SM)
    assert_loops("ffm_bwd_hot_kernel at the packing limit: work items per CTA", chunks // hgrid)
    V, A = 1024, 1
    R = 1
    G = ffm_staged_cols(R)
    g = torch.Generator(device=DEV).manual_seed(32767)
    ids = torch.full((n_max, 1), 2, dtype=torch.int64, device=DEV)
    body = torch.cat([torch.full((n_a,), A, dtype=torch.int64, device=DEV),
                      torch.arange(2, 2 + n - n_a, device=DEV)])
    ids[:n, 0] = body[torch.randperm(n, generator=g, device=DEV)]
    del body
    gy1 = torch.where(ids[:, 0] == A, 1.0, torch.randn(n_max, generator=g, device=DEV))
    gy2 = torch.randn(n_max, generator=g, device=DEV)
    W = _ffm_table(V, R, g)
    dense = torch.empty(n_max, 0, device=DEV)
    dense_w = torch.empty(0, R, device=DEV)
    groups = ops.raw_group_ids(ids[:n], V, -1)
    Uq = int(groups.num[0])
    assert Uq == 1 + n - n_a
    assert torch.equal(groups.unique_ids[:Uq], torch.arange(1, 1 + Uq, device=DEV))
    dW, _, _, db = ops.raw_ffm_bwd(W, ids[:n], dense[:n], dense_w, gy1[:n], gy2[:n], groups, -1, 1)
    assert float(dW[0, R]) == float(n_a), "g1 of the 32767-chunk id: %r, want %d" % (float(dW[0, R]), n_a)
    want1 = torch.zeros(V, device=DEV)
    rest = ids[:n, 0] != A
    want1[ids[:n, 0][rest]] = gy1[:n][rest]
    assert torch.equal(dW[1:Uq, R], want1[2:1 + Uq])
    assert not dW[:Uq, :R].any() and not dW[:Uq, R + 1:G].any()
    slices = min(FFM_MAX_SLICES, _cdiv(n, 256))
    g1 = gy1[:n].double()
    assert_within(db, g1.sum().reshape(1), (_cdiv(n, slices) + slices) * U * g1.abs().sum().reshape(1),
                  "dbias at the packing limit")

    nbytes = ctypes.c_size_t(0)
    assert lib.b200rec_ffm_bwd_workspace_bytes(n_max, 1, 0, R, ctypes.byref(nbytes)) == 0
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=DEV)
    seg = torch.zeros(n_max + 1, dtype=torch.int32, device=DEV)
    pos = torch.zeros(n_max, dtype=torch.int32, device=DEV)
    num = torch.tensor([Uq, n_max], dtype=torch.int32, device=DEV)
    out = torch.zeros(V, G, device=DEV)
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    rc = lib.b200rec_ffm_bwd(P(W), W.stride(0), P(ids), None, None, P(gy1), P(gy2), P(seg), P(pos),
                             P(num), P(out), G, None, None, P(db), n_max, 1, 0, R, V, -1, P(ws),
                             nbytes.value, None)
    assert rc == -1 and b"B*F" in lib.b200rec_last_error(), (rc, lib.b200rec_last_error())


# ================================================================================================
# 12. Wide-row optimizers (gather_scatter.cuh:294-353): one warp per row of > 32 vector chunks
# ================================================================================================
ROW_GUARD = 4   # rows of every table / state buffer before and after the V rows the call sees


def row_shape_for(D, ldw, ld_rows, byte_offsets):
    """pick_row_shape_for, gather_scatter.cuh:359-376: (VEC, TPR), TPR = 0 for the wide kernels."""
    vec = 4 if D % 4 == 0 else (2 if D % 2 == 0 else 1)
    while vec > 1 and (D % vec or ldw % vec or ld_rows % vec or any(o % (4 * vec) for o in byte_offsets)):
        vec >>= 1
    chunks = D // vec
    tpr = 1
    while tpr < chunks:
        tpr <<= 1
    return vec, (0 if chunks > 32 else tpr)


# name: (columns updated, table row stride, gradient row stride, first column of the view, VEC, TPR)
WIDE_CASES = {
    "ffm_d9": (352, 384, 352, 0, 4, 0),     # FFM's G at D=9, ldw = fused_slot(R)
    "ffm_d16": (628, 640, 628, 0, 4, 0),    # FFM's G at D=16
    "vec1": (625, 640, 625, 0, 1, 0),
    "cvm_view": (624, 628, 626, 2, 2, 0),   # [show, click, emb] rows: columns 2.. of table and grad
    "cvm_view_narrow": (16, 20, 18, 2, 2, 8),   # the same view on the lane-group kernels
}


@pytest.mark.parametrize("case", list(WIDE_CASES))
def test_wide_row_optimizers_at_scale(case):
    """row_update_wide_kernel (SGD, lazy Adam, rows_to_dense) and row_adagrad_wide_kernel: grid =
    min(ceil(n/8), 64*SM) warps of one row each (gather_scatter.cuh:399, 428), so U >= 3*8*64*SM
    rows make every warp update >= 3 rows; each lane steps through the row 32*VEC floats at a
    time.  Widths: FFM's G at D=9 and D=16 with ldw = fused_slot(R) and separate [V, slot] moments
    (optim.Adam on FFMLayer), 625 (VEC 1), and a [show, click, emb] column view 2 floats into the
    table and the gradient (VEC narrowed to 2; optim._table_parts), also at 16 columns on the
    lane-group kernels (row_update_kernel / row_adagrad_kernel, >= 3 rows per group).
    Bounds as test_row_updates_at_scale, except AdaGrad's g2sum on the wide kernel: each lane fmas
    ceil(D/(32*VEC))*VEC squares, 5 shuffle levels, the division by D and the add:
    k = ceil(D/(32*VEC))*VEC + 5 + 2 per step.  Out-of-range ids among the unique rows (-3, -1, V,
    V+2) are skipped; untouched rows, moments, g2sum, the guard rows around the V rows and the
    columns outside the view are bit-identical."""
    ops = _ops()
    SM = _sm()
    Dw, ldw, ldr, c0, vec, tpr = WIDE_CASES[case]
    assert row_shape_for(Dw, ldw, ldr, [4 * c0, 4 * ROW_GUARD * ldw]) == (vec, tpr)
    assert row_shape_for(Dw, Dw, ldr, [4 * c0, 4 * ROW_GUARD * Dw]) == (vec, tpr)   # rows_to_dense
    gpb = ROW_THREADS // (tpr or 32)
    Uq = 3 * WIDE_CTAS_PER_SM * SM * gpb + 77
    V = Uq + Uq // 8
    oob = torch.tensor([-3, -1, V, V + 2], device=DEV)
    n = Uq + oob.numel()
    grid = min(_cdiv(n, gpb), WIDE_CTAS_PER_SM * SM)
    assert_loops("%s (%s): rows per %s" % ("row_update_kernel" if tpr else "row_update_wide_kernel",
                                           case, "lane group" if tpr else "warp"), n // (grid * gpb))
    g = torch.Generator(device=DEV).manual_seed(Dw + c0)
    rows = torch.cat([torch.randperm(V, generator=g, device=DEV)[:Uq].sort().values, oob])
    rows = rows[torch.randperm(n, generator=g, device=DEV)]
    ok = (rows >= 0) & (rows < V)
    val_full = torch.randn(n, ldr, generator=g, device=DEV)
    num = torch.tensor([n, n], dtype=torch.int32, device=DEV)
    sr = ops.SelectedRows(rows, val_full[:, c0:], num, V, ncols=Dw)
    ids = rows[ok]
    gv = val_full[ok, c0:c0 + Dw]
    cols = slice(c0, c0 + Dw)
    inner = slice(ROW_GUARD, ROW_GUARD + V)
    W0_full = torch.randn(V + 2 * ROW_GUARD, ldw, generator=g, device=DEV)
    W0 = W0_full[inner, cols]
    ch = 32768

    def outside_unchanged(full, full0, c=cols):
        chk = full.clone()
        if full.dim() == 2:
            chk[ROW_GUARD + ids, c] = full0[ROW_GUARD + ids, c]
        else:
            chk[ROW_GUARD + ids] = full0[ROW_GUARD + ids]
        return torch.equal(chk, full0)

    # rows_to_dense: zeros + g, exact copies
    dW_full = torch.zeros(V + 2 * ROW_GUARD, Dw, device=DEV)
    ops.raw_rows_to_dense(sr, dW_full[inner])
    assert torch.equal(dW_full[ROW_GUARD + ids], gv), "rows_to_dense " + case
    assert outside_unchanged(dW_full, torch.zeros_like(dW_full), slice(None)), "rows_to_dense " + case
    del dW_full

    W_full = W0_full.clone()
    ops.raw_sparse_sgd(W_full[inner, cols], sr, 0.1)
    for s in range(0, ids.numel(), ch):
        i, gg = ids[s:s + ch], gv[s:s + ch].double()
        want = W0[i].double() - 0.1 * gg
        assert_within(W_full[inner, cols][i], want, 2 * U * (want.abs() + 0.1 * gg.abs()), "sgd " + case)
    assert outside_unchanged(W_full, W0_full), "sgd " + case

    W_full = W0_full.clone()
    m_full, v_full = torch.zeros_like(W0_full), torch.zeros_like(W0_full)
    b1, b2, eps, lr = 0.9, 0.999, 1e-8, 1e-3
    for t in (1, 2):
        ops.raw_sparse_adam(W_full[inner, cols], m_full[inner, cols], v_full[inner, cols], sr, lr, b1, b2,
                            eps, b1 ** t, b2 ** t)
    for s in range(0, ids.numel(), ch):
        i, gg = ids[s:s + ch], gv[s:s + ch].double()
        Wr, mr, vr = W0[i].double(), torch.zeros_like(gg), torch.zeros_like(gg)
        mm, upd = torch.zeros_like(gg), torch.zeros_like(gg)
        for t in (1, 2):                      # oracle/optim.py adam_lazy, with its error magnitudes
            lr_t = lr * math.sqrt(1 - b2 ** t) / (1 - b1 ** t)
            den = eps * math.sqrt(1 - b2 ** t)
            mr = b1 * mr + (1 - b1) * gg
            vr = b2 * vr + (1 - b2) * gg * gg
            Wr = Wr - lr_t * mr / (vr.sqrt() + den)
            mm = b1 * mm + (1 - b1) * gg.abs()
            upd += lr_t * (10 * mm + 16 * mr.abs()) / (vr.sqrt() + den)
        assert_within(m_full[inner, cols][i], mr, 10 * U * mm, "adam m " + case)
        assert_within(v_full[inner, cols][i], vr, 12 * U * vr, "adam v " + case)
        assert_within(W_full[inner, cols][i], Wr, U * (2 * Wr.abs() + upd), "adam W " + case)
    assert outside_unchanged(W_full, W0_full), "adam W " + case
    assert outside_unchanged(m_full, torch.zeros_like(m_full)), "adam m " + case
    assert outside_unchanged(v_full, torch.zeros_like(v_full)), "adam v " + case
    del m_full, v_full

    W_full = W0_full.clone()
    g2_full = torch.zeros(V + 2 * ROW_GUARD, device=DEV)
    lr, g0, lo, hi = 0.05, 3.0, -2.5, 2.5
    for _ in range(2):
        ops.raw_sparse_adagrad(W_full[inner, cols], g2_full[inner], sr, lr, g0, lo, hi)
    k_g2 = (_cdiv(Dw, 32 * vec) * vec + 5 + 2) if tpr == 0 else Dw + 8
    for s in range(0, ids.numel(), ch):
        i, gg = ids[s:s + ch], gv[s:s + ch].double()
        Wr, g2r, upd = W0[i].double(), torch.zeros(i.numel(), dtype=torch.float64, device=DEV), 0
        for _ in range(2):                    # oracle/optim.py adagrad_row
            sc = (g0 / (g0 + g2r)).sqrt().unsqueeze(1)
            upd = upd + (Dw + 16) * lr * gg.abs() * sc
            Wr = (Wr - lr * gg * sc).clamp(lo, hi)
            g2r = g2r + (gg * gg).mean(1)
        assert_within(g2_full[inner][i], g2r, 2 * k_g2 * U * g2r, "adagrad g2sum " + case)
        assert_within(W_full[inner, cols][i], Wr, U * (2 * Wr.abs() + upd), "adagrad W " + case)
    assert outside_unchanged(W_full, W0_full), "adagrad W " + case
    assert outside_unchanged(g2_full, torch.zeros_like(g2_full)), "adagrad g2sum " + case


# ================================================================================================
# 13. FAT-DeepFFM (fat_ffm.cuh): max pool, persistent forward and dattn, FatBwd on FFM's backward
# ================================================================================================
def _fat_e(W, ids, dense, dense_w, s, e, D, pad):
    """Samples s:e as E [b, NF, NF, D] in fp32, exactly as the kernels form it: E[b, n, m] is
    block m of row n, i.e. of the table row (zero for padding and out-of-range ids) or of the
    fp32 product dense * dense_w."""
    V = W.shape[0]
    F, Dn = ids.shape[1], dense.shape[1]
    NF = F + Dn
    idb = ids[s:e]
    ok = ((idb >= 0) & (idb < V) & (idb != pad)).unsqueeze(2)
    rows = torch.where(ok, W[idb.clamp(0, V - 1), :NF * D], 0.0)
    return torch.cat([rows, dense[s:e].unsqueeze(2) * dense_w.unsqueeze(0)], 1).view(e - s, NF, NF, D)


def _fat_closed_form(E32, attn, gy1, dh, dpool=None, bias=None):
    """FAT-DeepFFM's interaction and its gradients in fp64, in closed form, for the samples of E32.
    With A = attn as [b, NF, NF], ^T swapping n and m, DH = dh spread symmetrically with a zero
    diagonal and `first` the one-hot of the first index where E equals its block maximum:
        pool  = max_d E                          (fp32, exact)
        y1    = sum A.E + bias
        h     = (A.E)[n<m] . (A^T.E^T)[n<m]
        dattn = sum_d E . (gy1 + DH.A^T.E^T)
        de    = A.(gy1 + DH.A^T.E^T) + first.dpool      (only when dpool is given)
    Returns (pool, values, magnitudes); the magnitudes are the same expressions on absolute values
    (first unchanged): the sum of |terms| each output adds."""
    b, NF, _, D = E32.shape
    P = NF * (NF - 1) // 2
    iu = torch.triu_indices(NF, NF, 1, device=DEV)
    top = E32.amax(-1, keepdim=True)
    pool = top.reshape(b, NF * NF)
    if dpool is not None:
        at = (E32 == top).to(torch.int8).argmax(-1, keepdim=True)
        first = torch.zeros(E32.shape, dtype=torch.float64, device=DEV).scatter_(-1, at, 1.0)
    out = []
    for f in (lambda t: t.double(), lambda t: t.double().abs()):
        E = f(E32)
        A = f(attn).view(b, NF, NF, 1)
        DH = torch.zeros(E.shape, dtype=torch.float64, device=DEV)
        d = f(dh).view(b, P, D)
        DH[:, iu[0], iu[1]] = d
        DH[:, iu[1], iu[0]] = d
        S = A * E
        St = S.transpose(1, 2)
        ds = f(gy1).view(b, 1, 1, 1) + DH * St
        r = {"y1": S.sum((1, 2, 3)) + (0.0 if bias is None else f(bias)),
             "h": (S[:, iu[0], iu[1]] * St[:, iu[0], iu[1]]).reshape(b, P * D),
             "dattn": (E * ds).sum(3).reshape(b, NF * NF)}
        if dpool is not None:
            r["de"] = A * ds + first * f(dpool).view(b, NF, NF, 1)
        out.append(r)
    return pool, out[0], out[1]


def _fat_chunk(NF, D):
    return max(1, (1 << 22) // (NF * NF * D))


def test_fat_closed_form_matches_autograd_oracle():
    """The closed form above equals _oracle (autograd over the reference's operations) exactly, on
    inputs quantised to multiples of 1/4 so that every fp64 sum is exact in any order.  Table
    blocks hold ties, among them all-nonpositive blocks with both -0.0 and +0.0; dense values
    include -0.0 and 0; padding and out-of-range ids are mixed in."""
    B, F, Dn, D, V, pad = 300, 5, 3, 4, 50, 3
    NF, R = F + Dn, (F + Dn) * D
    g = torch.Generator(device=DEV).manual_seed(13)
    q = lambda lo, hi, *s: torch.randint(lo, hi, s, generator=g, device=DEV) / 4  # noqa: E731
    W = _ffm_table(V, R, g)
    W[:, :R] = q(-8, 9, V, R)
    W[:, R] = 7.0
    W[::2, :D] = -q(1, 9, (V + 1) // 2, D)
    W[::2, 1], W[::2, 3] = -0.0, 0.0
    ids = torch.randint(0, V, (B, F), generator=g, device=DEV)
    ids[::11, 0], ids[::13, 1], ids[::17, 2] = pad, -1, V + 2
    dense = torch.tensor([-1, -0.5, -0.0, 0.0, 0.5, 1.0], device=DEV)[
        torch.randint(0, 6, (B, Dn), generator=g, device=DEV)]
    dense_w = q(-8, 9, Dn, R)
    attn, gy1, dh, dpool = q(0, 5, B, NF * NF), q(-4, 5, B), q(-4, 5, B, NF * (NF - 1) // 2 * D), \
        q(-4, 5, B, NF * NF)
    bias = torch.tensor([0.25], device=DEV)
    ties = W[:, :R].view(V, NF, D)
    hit = (ties == ties.amax(-1, keepdim=True)).to(torch.int8)
    assert bool((hit.argmax(-1) != D - 1 - hit.flip(-1).argmax(-1)).any()), "no tied table block"

    pool, r, _ = _fat_closed_form(_fat_e(W, ids, dense, dense_w, 0, B, D, pad), attn, gy1, dh, dpool,
                                  bias)
    ref = _oracle(W, ids, dense, dense_w, attn, bias, gy1, dh, dpool, D, pad)
    ok = ((ids >= 0) & (ids < V) & (ids != pad)).reshape(-1)
    de = r["de"].reshape(B, NF, R)
    dW = torch.zeros(V, R, dtype=torch.float64, device=DEV).index_add_(
        0, ids.reshape(-1)[ok], de[:, :F].reshape(B * F, R)[ok])
    ddw = torch.einsum("bk,bkr->kr", dense.double(), de[:, F:])
    assert torch.equal(pool.double(), ref["pool"])
    for k in ("y1", "h", "dattn"):
        assert torch.equal(r[k], ref[k]), k
    assert torch.equal(dW, ref["dW"]) and torch.equal(ddw, ref["ddw"])


def _fat_sample_ids(B, F, V, pad, g):
    """[B, F] ids over [1, V): 3% padding, 0.5% negative, 0.5% >= V."""
    ids = torch.randint(1, V, (B, F), generator=g, device=DEV)
    r = torch.rand(B, F, generator=g, device=DEV)
    ids[r < 0.03] = pad
    neg, big = (r >= 0.03) & (r < 0.035), (r >= 0.035) & (r < 0.04)
    ids[neg] = -1 - torch.randint(0, 5, (B, F), generator=g, device=DEV)[neg]
    ids[big] = V + torch.randint(0, 5, (B, F), generator=g, device=DEV)[big]
    return ids


@pytest.mark.parametrize("F,Dn,D,B,nbuf", [
    (26, 13, 21, None, 2),     # the largest double-buffered shape at F=26, Dn=13
    (26, 13, 22, None, 1),     # the smallest single-buffered one
    (26, 13, 36, None, 1),     # the largest D that fits at all
    (26, 13, 10, 65536, 2),    # the benchmark shape
    (40, 24, 7, None, 2),      # NF = 64: 16 attention entries per thread, P = 2016 pairs
    (26, 0, 10, None, 2),      # no dense fields
    (1, 1, 3, None, 2),        # NF = 2: only B ~ 405k makes the pool's grid loop
    (1, 0, 4, None, 2),        # NF = 1: P = 0, h and dh have no elements
])
def test_fat_sample_kernels_at_scale(F, Dn, D, B, nbuf):
    """fat_ffm_pool_kernel and fat_ffm_sample_kernel<fwd / bwd>.  The pool runs one thread per
    (sample, block) on min(ceil(B*NF^2/256), 16*SM) CTAs (fat_ffm.cuh:322-324); the sample kernels
    run persistent CTAs, grid = min(B, SM*per_sm) with per_sm <= 8 (fat_ffm.cuh:350-353).  B
    defaults to the larger of 3*8*SM + 17 and the pool's 3-pass size, so every CTA takes >= 3
    samples (with two buffers, every CTA stages into both and prefetches across iterations) and
    every pool thread >= 3 blocks.  The buffering each case gets is asserted from the FatSmem
    mirror against the device's opt-in shared-memory limit.
    Against _fat_closed_form, bounds as test_gpu_fat_deepffm._check_all derives them:
    pool bit for bit; y1 gamma(ceil(NF^2/256)*(D+1) + 14) (per thread ceil(NF^2/256) blocks of D
    adds and one fma, 5 shuffles, 8 warp sums, the bias); h gamma(5); dattn gamma(D+5).
    Padding, negative and >= V ids read as zero rows; the pool counts each out-of-range position
    once, fwd and bwd_attn count none.  The w1 column (7.0) and the slot padding (123.0) must not
    leak.  A second run of each kernel is bit-identical."""
    ops = _ops()
    SM = _sm()
    NF = F + Dn
    R, P, NN = NF * D, NF * (NF - 1) // 2, NF * NF
    limit = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    if nbuf == 2:
        assert _fat_smem(F, Dn, D, 2) <= limit, "F=%d Dn=%d D=%d no longer double-buffered" % (F, Dn, D)
    else:
        assert _fat_smem(F, Dn, D, 2) > limit >= _fat_smem(F, Dn, D, 1), \
            "F=%d Dn=%d D=%d is no longer single-buffered" % (F, Dn, D)
    if D == 36:
        assert _fat_smem(F, Dn, D + 1, 1) > limit, "D=37 fits: D=36 is no longer the largest shape"
    B = B or max(3 * FAT_SAMPLE_MAX_CTAS_PER_SM * SM + 17,
                 _cdiv(3 * FAT_POOL_CTAS_PER_SM * SM * FAT_POOL_THREADS, NN))
    what = "fat F=%d Dn=%d D=%d B=%d" % (F, Dn, D, B)
    assert_loops("fat_ffm_sample_kernel %s (%d buffers): samples per CTA" % (what, nbuf),
                 B // (FAT_SAMPLE_MAX_CTAS_PER_SM * SM))
    pgrid = min(_cdiv(B * NN, FAT_POOL_THREADS), FAT_POOL_CTAS_PER_SM * SM)
    assert_loops("fat_ffm_pool_kernel %s: blocks per thread" % what, B * NN // (pgrid * FAT_POOL_THREADS))
    V, pad = 20_000, 0
    g = torch.Generator(device=DEV).manual_seed(1000 * D + NF)
    W = _ffm_table(V, R, g)
    W[:, R] = 7.0
    ids = _fat_sample_ids(B, F, V, pad, g)
    n_oob = int(((ids < 0) | (ids >= V)).sum())
    assert n_oob > 0 and int((ids == pad).sum()) > 0
    dense = torch.rand(B, Dn, generator=g, device=DEV) * 2 - 0.5
    dense_w = torch.randn(Dn, R, generator=g, device=DEV) * 0.1
    attn = torch.relu(torch.randn(B, NN, generator=g, device=DEV) + 0.3)
    gy1 = torch.randn(B, generator=g, device=DEV)
    dh = torch.randn(B, P * D, generator=g, device=DEV)
    bias = torch.tensor([0.3], device=DEV)

    ops.raw_oob_count()
    pool = ops.raw_fat_ffm_pool_fwd(W, ids, dense, dense_w, pad, D)
    assert ops.raw_oob_count() == n_oob
    y1, h = ops.raw_fat_ffm_fwd(W, ids, dense, dense_w, attn, bias, pad, D)
    dattn = ops.raw_fat_ffm_bwd_attn(W, ids, dense, dense_w, attn, gy1, dh, pad, D)
    assert ops.raw_oob_count() == 0
    assert torch.equal(pool, ops.raw_fat_ffm_pool_fwd(W, ids, dense, dense_w, pad, D)), what + " pool"
    y1b, hb = ops.raw_fat_ffm_fwd(W, ids, dense, dense_w, attn, bias, pad, D)
    assert torch.equal(y1, y1b) and torch.equal(h, hb), what + ": fwd not bit-reproducible"
    del hb
    assert torch.equal(dattn, ops.raw_fat_ffm_bwd_attn(W, ids, dense, dense_w, attn, gy1, dh, pad, D)), \
        what + ": dattn not bit-reproducible"
    ops.raw_oob_count()

    k_y1 = _gamma(_cdiv(NN, 256) * (D + 1) + 14)
    chunk = _fat_chunk(NF, D)
    for s in range(0, B, chunk):
        e = min(B, s + chunk)
        E = _fat_e(W, ids, dense, dense_w, s, e, D, pad)
        want_pool, r, m = _fat_closed_form(E, attn[s:e], gy1[s:e], dh[s:e], bias=bias)
        at = "%s samples %d.." % (what, s)
        assert torch.equal(pool[s:e], want_pool), at + " pool"
        assert_within(y1[s:e], r["y1"], k_y1 * m["y1"] + 1e-30, at + " y1")
        assert_within(h[s:e], r["h"], _gamma(5) * m["h"] + 1e-30, at + " h")
        assert_within(dattn[s:e], r["dattn"], _gamma(D + 5) * m["dattn"] + 1e-30, at + " dattn")


FAT_TIED_ID = 1 + FFM_BWD_LENS.index(150001)


def _fat_tied_inputs(W, V, Dn, R, D, NF, B, g):
    """Quantised inputs full of ties: table and dense_w entries in {-2, -1.75, ..., 2}; every third
    table row (and ids 1..7) gets one block of nonpositive values holding -0.0 and +0.0 at two
    different columns; dense values from {-1, -0.5, -0.0, 0, 0.5, 1}."""
    W[:, :R] = torch.randint(-8, 9, (V, R), generator=g, device=DEV) / 4
    ar = torch.arange(V, device=DEV)
    sel = ar[(ar % 3 == 0) | (ar <= len(FFM_BWD_LENS))]
    m = sel % NF
    j0 = (sel // NF) % D
    j1 = (j0 + 1 + (sel // 7) % (D - 1)) % D
    cols = m.unsqueeze(1) * D + torch.arange(D, device=DEV)
    W[sel.unsqueeze(1), cols] = -(torch.randint(1, 9, (sel.numel(), D), generator=g, device=DEV) / 4)
    W[sel, m * D + j0] = -0.0
    W[sel, m * D + j1] = 0.0
    dense = torch.tensor([-1, -0.5, -0.0, 0.0, 0.5, 1.0], device=DEV)[
        torch.randint(0, 6, (B, Dn), generator=g, device=DEV)]
    dense_w = torch.randint(-8, 9, (Dn, R), generator=g, device=DEV) / 4
    return dense, dense_w


@pytest.mark.parametrize("Dn,D,B,tied", [
    (13, 10, 65536, False),    # the benchmark shape: 256 full slices
    (13, 10, 65536 - 100, False),   # a short last slice
    (13, 10, 65536, True),     # tied block maxima: the first maximum takes the pool gradient
    (0, 4, 65536, False),      # no dense fields
    (13, 1, 65536, False),     # every column is its block's maximum
])
def test_fat_bwd_at_scale(Dn, D, B, tied):
    """raw_fat_ffm_bwd (FatBwd on ffm_bwd_light / hot / combine / dense kernels) at B*F = 1.7M
    positions, F=26, V=200k, with _ffm_bwd_ids' stream: every light warp walks >= 3 distinct ids,
    every hot CTA takes >= 3 work items, and the combine adds the 147 chunks of the
    150001-position id.  Every row of every distinct id is checked element-wise against the
    per-position de of _fat_closed_form merged in fp64 with index_add, bound gamma(ffm_bwd_chain
    + 4): FFM's chain with 6 roundings per term instead of 2 (the partner product, dh fma, attn
    product, the dense product, the pool add).  Columns R..G-1 (the w1 column and the padding)
    must be exactly 0.  Dense gradients over `slices` = min(256, ceil(B/256)) slices of per_slice
    samples: ddense_w gamma(per_slice + slices + 6), dbias gamma(per_slice + slices).  Every
    output is bit-identical on a second run.
    tied: table and dense_w entries are multiples of 1/4 in [-2, 2], some table blocks hold both
    -0.0 and +0.0 as their maximum, dense values include -0.0 and 0, and the inputs are asserted
    to hold blocks whose first and last maxima differ for a light id, a single-chunk hot id and
    the 150001-position id: a last-maximum rule moves dpool to another column of their rows."""
    ops = _ops()
    SM = _sm()
    F, V, pad = 26, 200_000, 0
    NF = F + Dn
    R, P, NN = NF * D, NF * (NF - 1) // 2, NF * NF
    G = ffm_staged_cols(R)
    n = B * F
    assert n < FAT_MAX_POSITIONS
    g = torch.Generator(device=DEV).manual_seed(100 * D + Dn + B + tied)
    ids = _ffm_bwd_ids(B, F, V, g)
    flat = ids.reshape(-1)
    valid = (flat >= 0) & (flat < V) & (flat != pad)
    uniq, inv, counts = torch.unique(flat[valid], return_inverse=True, return_counts=True)
    Uq = uniq.numel()
    assert sorted(counts[counts > 300].tolist()) == sorted(c for c in FFM_BWD_LENS if c > 300)
    wpb = FFM_THREADS // 32
    assert int((counts <= HOT_THRESHOLD).sum()) >= 3 * FFM_LIGHT_CTAS_PER_SM * SM * wpb
    lgrid = min(_cdiv(n, wpb), FFM_LIGHT_CTAS_PER_SM * SM)
    assert_loops("ffm_bwd_light_kernel<FatBwd>: distinct ids per warp", Uq // (lgrid * wpb))
    hot = counts[counts > HOT_THRESHOLD]
    n_items = int(((hot + FFM_HOT_CHUNK - 1) // FFM_HOT_CHUNK).sum())
    hgrid = min(n // (HOT_THRESHOLD + 1) + 1, FFM_HOT_CTAS_PER_SM * SM)
    assert_loops("ffm_bwd_hot_kernel<FatBwd>: work items per CTA", n_items // hgrid)
    assert_loops("ffm_bwd_combine_kernel: chunks of the 150001-position id",
                 _cdiv(FFM_BWD_LENS[-1], FFM_HOT_CHUNK))
    slices = min(FFM_MAX_SLICES, _cdiv(B, 256))
    per_slice = _cdiv(B, slices)
    assert_loops("ffm_bwd_dense_kernel<FatBwd>: samples per slice", per_slice)

    W = _ffm_table(V, R, g)
    W[:, R] = 7.0
    if tied:
        dense, dense_w = _fat_tied_inputs(W, V, Dn, R, D, NF, B, g)
        blk = W[uniq, :R].view(Uq, NF, D)
        hit = (blk == blk.amax(-1, keepdim=True)).to(torch.int8)
        split = (hit.argmax(-1) != D - 1 - hit.flip(-1).argmax(-1)).any(1)
        assert bool(split[counts <= HOT_THRESHOLD].any()), "no light id with a tied block"
        assert bool(split[(counts > HOT_THRESHOLD) & (counts <= FFM_HOT_CHUNK)].any()), \
            "no single-chunk hot id with a tied block"
        assert bool(split[uniq == FAT_TIED_ID].all()), "the 150001-position id has no tied block"
        del blk, hit
    else:
        dense = torch.rand(B, Dn, generator=g, device=DEV) * 2 - 0.5
        dense_w = torch.randn(Dn, R, generator=g, device=DEV) * 0.1
    attn = torch.relu(torch.randn(B, NN, generator=g, device=DEV) + 0.3)
    gy1 = torch.randn(B, generator=g, device=DEV)
    dh = torch.randn(B, P * D, generator=g, device=DEV)
    dpool = torch.randn(B, NN, generator=g, device=DEV)
    groups = ops.raw_group_ids(ids, V, pad)
    assert int(groups.num[0]) == Uq
    assert torch.equal(groups.unique_ids[:Uq], uniq), "the gradient rows must be exactly the valid ids"
    args = (W, ids, dense, dense_w, attn, gy1, dh, dpool, groups, pad, D)
    dW, ddw, db = ops.raw_fat_ffm_bwd(*args)
    dW2, ddw2, db2 = ops.raw_fat_ffm_bwd(*args)
    what = "fat bwd Dn=%d D=%d B=%d%s" % (Dn, D, B, " tied" if tied else "")
    assert torch.equal(dW[:Uq], dW2[:Uq]), what + ": rows not bit-reproducible"
    assert torch.equal(ddw, ddw2) and torch.equal(db, db2), what + ": dense gradients not bit-reproducible"
    del dW2
    assert dW.shape[1] == G and not dW[:Uq, R:].any(), what + ": columns R.. of the rows must be 0"

    f64 = dict(dtype=torch.float64, device=DEV)
    pos_row = torch.full((n,), -1, dtype=torch.int64, device=DEV)
    pos_row[valid] = inv
    want, mag = torch.zeros(Uq, R, **f64), torch.zeros(Uq, R, **f64)
    wdw, mdw = torch.zeros(Dn, R, **f64), torch.zeros(Dn, R, **f64)
    chunk = _fat_chunk(NF, D)
    for s in range(0, B, chunk):
        e = min(B, s + chunk)
        b = e - s
        E = _fat_e(W, ids, dense, dense_w, s, e, D, pad)
        _, r, m = _fat_closed_form(E, attn[s:e], gy1[s:e], dh[s:e], dpool[s:e])
        de, dm = r["de"].view(b, NF, R), m["de"].view(b, NF, R)
        rr = pos_row[s * F:e * F]
        ok = rr >= 0
        want.index_add_(0, rr[ok], de[:, :F].reshape(b * F, R)[ok])
        mag.index_add_(0, rr[ok], dm[:, :F].reshape(b * F, R)[ok])
        if Dn:
            x = dense[s:e].double()
            wdw += torch.einsum("bk,bkr->kr", x, de[:, F:])
            mdw += torch.einsum("bk,bkr->kr", x.abs(), dm[:, F:])
    del E, r, m, de, dm
    k = _gamma(ffm_bwd_chain(counts) + 4).unsqueeze(1)
    for r0 in range(0, Uq, 32768):
        sl = slice(r0, min(Uq, r0 + 32768))
        assert_within(dW[sl, :R], want[sl], k[sl] * mag[sl] + 1e-30, what + " rows %d.." % r0)
    del want, mag
    if Dn:
        assert_within(ddw, wdw, _gamma(per_slice + slices + 6) * mdw + 1e-30, what + " ddense_w")
    assert_within(db, gy1.double().sum().reshape(1),
                  _gamma(per_slice + slices) * gy1.double().abs().sum().reshape(1), what + " dbias")


def test_fat_bwd_chunk_packing_limit():
    """FatBwd on the work-item packing of test_ffm_bwd_chunk_packing_limit: items pack
    chunk | (chunks << 16) into one int32 (ffm.cuh:287), which the launcher bounds by
    B*F < 32767*1024 (fat_ffm.cuh:370).  F=1, Dn=0, D=1: NF = 1, so P = 0 and dh has no elements.
    At B*F = 32767*1024 - 1, id 1 takes 32766*1024 + 512 positions (32767 chunks), all with
    attn = gy1 = dpool = 1: each contributes attn*gy1 + dpool = 2 (with D = 1 every column is its
    block's maximum).  A full chunk sums to exactly 2048 (8 warps of 128 twos), every partial total
    of the combine is a multiple of 1024 below 2^26, so fp32 holds each one exactly and id 1's row
    must be exactly 2*n_a: a dropped or duplicated chunk shows.  The other 511 positions go to
    distinct ids, each row one attn*gy1 + dpool (gamma(2)).  dbias: gamma(per_slice + slices).  One
    more position, with every buffer sized for it, is refused with B200REC_ERR_INVALID naming B*F."""
    import ctypes
    from paddlerec_b200 import _lib
    ops = _ops()
    lib = _lib.load()
    SM = _sm()
    n_max = FAT_MAX_POSITIONS                     # the first B*F the launcher refuses
    n = n_max - 1
    n_a = (FFM_MAX_CHUNKS - 1) * FFM_HOT_CHUNK + FFM_HOT_CHUNK // 2
    chunks = _cdiv(n_a, FFM_HOT_CHUNK)
    assert chunks == FFM_MAX_CHUNKS and chunks << 16 == 2_147_418_112
    assert 2 * n_a < 1 << 26
    hgrid = min(n // (HOT_THRESHOLD + 1) + 1, FFM_HOT_CTAS_PER_SM * SM)
    assert_loops("ffm_bwd_hot_kernel<FatBwd> at the packing limit: work items per CTA", chunks // hgrid)
    V, A, D = 1024, 1, 1
    R = D
    G = ffm_staged_cols(R)
    g = torch.Generator(device=DEV).manual_seed(32768)
    ids = torch.full((n_max, 1), 2, dtype=torch.int64, device=DEV)
    body = torch.cat([torch.full((n_a,), A, dtype=torch.int64, device=DEV),
                      torch.arange(2, 2 + n - n_a, device=DEV)])
    ids[:n, 0] = body[torch.randperm(n, generator=g, device=DEV)]
    del body
    hot = ids[:, 0] == A
    attn = torch.where(hot, 1.0, torch.rand(n_max, generator=g, device=DEV)).unsqueeze(1)
    gy1 = torch.where(hot, 1.0, torch.randn(n_max, generator=g, device=DEV))
    dpool = torch.where(hot, 1.0, torch.randn(n_max, generator=g, device=DEV)).unsqueeze(1)
    dh = torch.empty(n_max, 0, device=DEV)
    W = _ffm_table(V, R, g)
    W[:, R] = 7.0
    dense = torch.empty(n_max, 0, device=DEV)
    dense_w = torch.empty(0, R, device=DEV)
    groups = ops.raw_group_ids(ids[:n], V, -1)
    Uq = int(groups.num[0])
    assert Uq == 1 + n - n_a
    assert torch.equal(groups.unique_ids[:Uq], torch.arange(1, 1 + Uq, device=DEV))
    dW, _, db = ops.raw_fat_ffm_bwd(W, ids[:n], dense[:n], dense_w, attn[:n], gy1[:n], dh[:n], dpool[:n],
                                    groups, -1, D)
    assert float(dW[0, 0]) == 2.0 * n_a, "row of the 32767-chunk id: %r, want %d" % (float(dW[0, 0]), 2 * n_a)
    rest = ~hot[:n]
    at, g1, dp = attn[:n, 0][rest].double(), gy1[:n][rest].double(), dpool[:n, 0][rest].double()
    want = torch.zeros(V, dtype=torch.float64, device=DEV)
    mag = torch.zeros(V, dtype=torch.float64, device=DEV)
    want[ids[:n, 0][rest]] = at * g1 + dp
    mag[ids[:n, 0][rest]] = (at * g1).abs() + dp.abs()
    assert_within(dW[1:Uq, 0], want[2:1 + Uq], _gamma(2) * mag[2:1 + Uq] + 1e-30, "single-position rows")
    assert not dW[:Uq, R:G].any()
    slices = min(FFM_MAX_SLICES, _cdiv(n, 256))
    g1 = gy1[:n].double()
    assert_within(db, g1.sum().reshape(1), _gamma(_cdiv(n, slices) + slices) * g1.abs().sum().reshape(1),
                  "dbias at the packing limit")

    nbytes = ctypes.c_size_t(0)
    assert lib.b200rec_fat_ffm_bwd_workspace_bytes(n_max, 1, 0, D, ctypes.byref(nbytes)) == 0
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=DEV)
    seg = torch.zeros(n_max + 1, dtype=torch.int32, device=DEV)
    pos = torch.zeros(n_max, dtype=torch.int32, device=DEV)
    num = torch.tensor([Uq, n_max], dtype=torch.int32, device=DEV)
    out = torch.zeros(V, G, device=DEV)
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    rc = lib.b200rec_fat_ffm_bwd(P(W), W.stride(0), P(ids), None, None, P(attn), P(gy1), None, P(dpool),
                                 P(seg), P(pos), P(num), P(out), G, None, P(db), n_max, 1, 0, D, V, -1,
                                 P(ws), nbytes.value, None)
    assert rc == -1 and b"B*F" in lib.b200rec_last_error(), (rc, lib.b200rec_last_error())
