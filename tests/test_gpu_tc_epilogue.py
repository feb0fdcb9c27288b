"""The K-major GEMM's staged epilogue (csrc/tc_gemm.cuh) bit for bit against torch.

The raw fp32 accumulator of a product comes from the same kernel: the same call with fp32 output
and no bias, ReLU, mask, addend or CrossNet.  Every epilogue kind must then equal what torch
computes from that accumulator in fp32 (the element-wise order of the kernel: + bias, + addend,
aux store, CrossNet fma, ReLU, mask), with hi = bf16(v) and lo = bf16(v - hi) rounded to nearest.
Only the CrossNet fma is held to 1 ulp of the correctly rounded x0 * u + xl (torch rounds the
product and the sum separately).  Values compare with torch.equal, which does not tell -0 from +0:
a last k-block skips the k-steps that would multiply TMA's zero fill, and that can change only the
sign of an exact zero.

Every output buffer starts as NaN; afterwards the rows past M, the fp32 columns past N and the
plane columns between N and the pitch (other than the column of ones) must still hold NaN.  Pitches
that are not multiples of 4 take the epilogue's element-wise path.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
EXTRA_ROWS = 5          # rows past M in every output buffer


def _ops():
    from paddlerec_b200 import ops
    return ops


def _lib():
    from paddlerec_b200 import _lib
    return _lib


# mirrors of the launcher (csrc/tc_gemm.cuh): kBM, kTileBN and pick_bn, the grid of
# launch_kmajor_tiles
BM = 128
TILE_BN = [16, 64, 128, 208, 256]


def pick_bn(n):
    best, best_cost = 256, None
    for bn in TILE_BN:
        cost = (n + bn - 1) // bn * (bn + 64)
        if best_cost is None or cost <= best_cost:
            best, best_cost = bn, cost
    return best


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _nan(rows, cols, dtype):
    return torch.full((rows, cols), float("nan"), dtype=dtype, device=DEV)


def _split(v):
    hi = v.to(torch.bfloat16)
    lo = (v - hi.float()).to(torch.bfloat16)
    return hi, lo


def _check_planes(p, v, M, N, ldp, ones_col=False):
    """planes p [M + EXTRA_ROWS, 2 ldp] hold split(v) in [:M, :N], NaN everywhere else they may not
    write (the column of ones excepted)."""
    hi, lo = _split(v)
    assert torch.equal(p[:M, :N], hi)
    assert torch.equal(p[:M, ldp:ldp + N], lo)
    pad0 = N + (1 if ones_col else 0)
    if ones_col:
        assert torch.all(p[:M, N].float() == 1) and torch.all(p[:M, ldp + N].float() == 0)
    assert torch.isnan(p[:M, pad0:ldp].float()).all()
    assert torch.isnan(p[:M, ldp + pad0:].float()).all()
    assert torch.isnan(p[M:].float()).all()


def _check_f32(y, v, M, N):
    assert torch.equal(y[:M, :N], v)
    assert torch.isnan(y[:M, N:]).all() and torch.isnan(y[M:]).all()


def _odd(n):
    """An odd pitch > n: rows not aligned for the epilogue's 8- and 16-byte accesses."""
    return n + 3 if n % 2 == 0 else n + 2


def _planes_of(x):
    ops = _ops()
    return ops.raw_tc_split(x)


def _fwd(a, K, WTp, N, M, bias=None, relu=False, ld_f32=0, ldp=0, ones_col=False):
    """b200rec_tc_linear_fwd into NaN-filled buffers; ld_f32 / ldp = 0: that output is off."""
    L = _lib()
    y = _nan(M + EXTRA_ROWS, ld_f32, torch.float32) if ld_f32 else None
    p = _nan(M + EXTRA_ROWS, 2 * ldp, torch.bfloat16) if ldp else None
    L.check(L.load().b200rec_tc_linear_fwd(
        L.ptr(a), a.shape[1] // 2, L.ptr(WTp), WTp.shape[1] // 2, L.ptr(bias), int(relu), L.ptr(y),
        ld_f32, L.ptr(p), ldp, int(ones_col), M, N, K, _ops()._stream()), "tc_linear_fwd")
    return y, p


def _dx(gp, N, Wp, K, M, mask=None, addend=None, ld_f32=0, ldp=0, dbias=False):
    """b200rec_tc_linear_bwd_dx (output width K, reduction N) into NaN-filled buffers."""
    L, ops = _lib(), _ops()
    y = _nan(M + EXTRA_ROWS, ld_f32, torch.float32) if ld_f32 else None
    p = _nan(M + EXTRA_ROWS, 2 * ldp, torch.bfloat16) if ldp else None
    db = torch.full((K,), float("nan"), device=DEV) if dbias else None
    ws = ops._tc_bwd_ws(M, K, N, DEV)
    L.check(L.load().b200rec_tc_linear_bwd_dx(
        L.ptr(gp), gp.shape[1] // 2, L.ptr(Wp), Wp.shape[1] // 2, L.ptr(mask),
        mask.shape[1] // 2 if mask is not None else 0, L.ptr(addend), L.ptr(y), ld_f32, L.ptr(p),
        ldp, L.ptr(db), M, K, N, L.ptr(ws), ws.numel(), ops._stream()), "tc_linear_bwd_dx")
    return y, p, db


def _raw_fwd(a, K, WTp, N, M):
    y, _ = _fwd(a, K, WTp, N, M, ld_f32=N)
    return y[:M, :N].clone()


def _operands(M, N, K, seed):
    ops = _ops()
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=g).to(DEV)
    W = (torch.randn(K, N, generator=g) / math.sqrt(K)).to(DEV)
    b = (torch.randn(N, generator=g) * 0.1).to(DEV)
    a = _planes_of(x)
    Wp, WTp = ops.raw_tc_prep_weight(W)
    return a, Wp, WTp, b, g


def _with_bk(bk, fn):
    ops = _ops()
    ops.tc_debug(4, bk)
    try:
        return fn()
    finally:
        ops.tc_debug(4, 64)


# K whose last 64-wide k-block holds 1, 2, 3, 4 k-steps (and 1 or 2 of a 32-wide one), K not a
# multiple of 16; M not a multiple of 128; N below, at and above a tile, odd, and 1
SHAPES = [
    (300, 400, 80), (300, 400, 96), (300, 400, 112), (300, 400, 128),
    (257, 37, 70), (257, 37, 100), (129, 1, 48), (129, 1, 40), (200, 208, 624), (131, 130, 9),
]


@pytest.mark.parametrize("bk", [32, 64])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_fwd_kinds_bit_exact(M, N, K, bk):
    """Forward: bias + ReLU into fp32 and planes (with the column of ones), no bias, and pitches
    that force the element-wise path."""
    a, _, WTp, b, _ = _operands(M, N, K, M * 31 + N * 7 + K)

    def run():
        raw = _raw_fwd(a, K, WTp, N, M)
        v = torch.clamp_min(raw + b, 0.0)
        ldp = (N + 1 + 7) // 8 * 8
        y, p = _fwd(a, K, WTp, N, M, bias=b, relu=True, ld_f32=N + 4, ldp=ldp, ones_col=True)
        _check_f32(y, v, M, N)
        _check_planes(p, v, M, N, ldp, ones_col=True)
        # no bias, no ReLU, odd pitches: every access element-wise
        y, p = _fwd(a, K, WTp, N, M, ld_f32=N + 1, ldp=_odd(N))
        _check_f32(y, raw, M, N)
        _check_planes(p, raw, M, N, _odd(N))
        # planes only, bias without ReLU
        _, p = _fwd(a, K, WTp, N, M, bias=b, ldp=(N + 7) // 8 * 8)
        _check_planes(p, raw + b, M, N, (N + 7) // 8 * 8)
        torch.cuda.synchronize()

    _with_bk(bk, run)


@pytest.mark.parametrize("bk", [32, 64])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_dx_kinds_bit_exact(M, N, K, bk):
    """dX (output width N here, reduction K): the ReLU mask into planes with column sums, fp32
    without a mask, fp32 + addend, and a mask pitch that forces the element-wise path."""
    # the dX GEMM reduces over the layer's output width: operands g [M, K] and W [N, K]
    a, _, WTp, _, g = _operands(M, N, K, M * 17 + N * 5 + K)
    act = torch.randn(M, N, generator=g).clamp_min(0).to(DEV)
    act[:, ::3] = 0.0
    mask = _planes_of(act)
    addend = torch.randn(M, N, generator=g).to(DEV)

    def run():
        raw = _raw_fwd(a, K, WTp, N, M)
        keep = mask[:M, :N].float() > 0
        v = torch.where(keep, raw, torch.zeros_like(raw))
        ldp = (N + 7) // 8 * 8
        y, p, db = _dx(a, K, WTp, N, M, mask=mask, ld_f32=N + 4, ldp=ldp, dbias=True)
        _check_f32(y, v, M, N)
        _check_planes(p, v, M, N, ldp)
        assert torch.allclose(db.double(), v.double().sum(0),
                              atol=1e-5 * float(v.abs().sum(0).max()) + 1e-30, rtol=0)
        _, _, db2 = _dx(a, K, WTp, N, M, mask=mask, ldp=ldp, dbias=True)
        assert torch.equal(db, db2)       # fixed-order column sums
        y, _, _ = _dx(a, K, WTp, N, M, ld_f32=N)
        _check_f32(y, raw, M, N)
        y, _, _ = _dx(a, K, WTp, N, M, addend=addend, ld_f32=N + 1)
        _check_f32(y, raw + addend, M, N)
        # a mask whose rows are not 8-byte aligned: element-wise mask reads
        ldo = _odd(N)
        odd = torch.empty(M, 2 * ldo, dtype=torch.bfloat16, device=DEV)
        odd[:, :N] = mask[:, :N]
        odd[:, ldo:ldo + N] = mask[:, ldp:ldp + N]
        y, p, _ = _dx(a, K, WTp, N, M, mask=odd, ld_f32=N, ldp=ldo)
        _check_f32(y, v, M, N)
        _check_planes(p, v, M, N, ldo)
        torch.cuda.synchronize()

    _with_bk(bk, run)


@pytest.mark.parametrize("M,C", [(300, 400), (129, 37), (200, 1)])
def test_cross_bit_exact(M, C):
    """CrossNet: aux u = acc + bias exactly; out = fma(x0, u, xl) within 1 ulp of the correctly
    rounded value, and the planes of out exactly the split of the fp32 out."""
    L = _lib()
    a, _, WTp, b, g = _operands(M, C, C, M + 3 * C)
    x0 = torch.randn(M, C, generator=g).to(DEV)
    xl = torch.randn(M, C, generator=g).to(DEV)
    raw = _raw_fwd(a, C, WTp, C, M)
    for ld, ldp in [(C, (C + 1 + 7) // 8 * 8), (C + 1, _odd(C))]:
        x0p = torch.zeros(M, ld, device=DEV)
        xlp = torch.zeros(M, ld, device=DEV)
        x0p[:, :C], xlp[:, :C] = x0, xl
        u = _nan(M + EXTRA_ROWS, ld, torch.float32)
        out = _nan(M + EXTRA_ROWS, ld, torch.float32)
        p = _nan(M + EXTRA_ROWS, 2 * ldp, torch.bfloat16)
        ones = ldp > C and ldp % 8 == 0
        L.check(L.load().b200rec_tc_cross_fwd(
            L.ptr(a), a.shape[1] // 2, L.ptr(WTp), WTp.shape[1] // 2, L.ptr(b), L.ptr(x0p),
            L.ptr(xlp), ld, L.ptr(u), L.ptr(out), ld, L.ptr(p), ldp, int(ones), M, C,
            _ops()._stream()), "tc_cross_fwd")
        torch.cuda.synchronize()
        uv = raw + b
        _check_f32(u, uv, M, C)
        want = (x0.double() * uv.double() + xl.double()).float()
        got = out[:M, :C]
        ulp = (torch.nextafter(want.abs(), torch.full_like(want, math.inf)) - want.abs())
        assert bool(((got - want).abs() <= ulp).all())
        assert torch.isnan(out[:M, C:]).all() and torch.isnan(out[M:]).all()
        _check_planes(p, got.contiguous(), M, C, ldp, ones_col=ones)


@pytest.mark.parametrize("bk", [32, 64])
def test_staging_reused_across_tiles(bk):
    """Every CTA of the persistent grid runs at least 3 tiles, so each warp's staging chunks and
    column-sum rows are reused from tile to tile; forward and masked dX with column sums."""
    N, K = 400, 400
    bn = pick_bn(N)
    tiles_n = (N + bn - 1) // bn
    tiles_m = (3 * _sms() + tiles_n - 1) // tiles_n + 1
    M = tiles_m * BM - 50
    tiles = tiles_m * tiles_n
    grid = min(tiles, _sms())
    assert tiles // grid >= 3, (tiles, grid)
    a, _, WTp, b, g = _operands(M, N, K, 4242)
    act = torch.randn(M, N, generator=g).clamp_min(0).to(DEV)
    mask = _planes_of(act)

    def run():
        raw = _raw_fwd(a, K, WTp, N, M)
        v = torch.clamp_min(raw + b, 0.0)
        ldp = (N + 1 + 7) // 8 * 8
        y, p = _fwd(a, K, WTp, N, M, bias=b, relu=True, ld_f32=N, ldp=ldp, ones_col=True)
        _check_f32(y, v, M, N)
        _check_planes(p, v, M, N, ldp, ones_col=True)
        vm = torch.where(mask[:M, :N].float() > 0, raw, torch.zeros_like(raw))
        ldp = (N + 7) // 8 * 8
        _, p, db = _dx(a, K, WTp, N, M, mask=mask, ldp=ldp, dbias=True)
        _check_planes(p, vm, M, N, ldp)
        _, _, db2 = _dx(a, K, WTp, N, M, mask=mask, ldp=ldp, dbias=True)
        assert torch.equal(db, db2)
        assert torch.allclose(db.double(), vm.double().sum(0),
                              atol=1e-5 * float(vm.abs().sum(0).max()), rtol=0)
        torch.cuda.synchronize()

    _with_bk(bk, run)
