"""wgmma / TMA tower GEMMs (csrc/tc_gemm.cuh) through the C ABI vs an fp64 product of the
same fp32 operands.  Split precision (bf16x3) drops only the lo*lo term and the residual of the
residual: ~2^-17 per product, so 5e-5 of the output's max-norm is a tight bar (TF32 would be 5e-4).
Edge cases: M, N, K not multiples of the tile (128 x BN x 64), N = 1, K = 1, forced narrow tiles,
every epilogue (bias, ReLU, planes / fp32 / both, ReLU mask + bias column-sum, CrossNet)."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _ops():
    from paddlerec_b200 import ops
    return ops


def _join(planes, n):
    """planes [R, 2*ld] -> fp64 hi + lo of the logical [R, n] matrix."""
    ld = planes.shape[1] // 2
    p = planes.double()
    return p[:, :n] + p[:, ld:ld + n]


def _err(got, want):
    return float((got.double().cpu() - want.cpu()).abs().max() / (want.abs().max() + 1e-30))


SHAPES = [(257, 400, 624), (128, 400, 400), (300, 1, 400), (1000, 208, 64), (129, 16, 8),
          (4096, 624, 400), (513, 40, 1560), (64, 400, 1)]


@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("relu", [False, True])
def test_tc_linear_fwd(M, N, K, relu):
    ops = _ops()
    g = torch.Generator().manual_seed(M * 7 + N * 3 + K)
    x = torch.randn(M, K, generator=g)
    W = torch.randn(K, N, generator=g) / K ** 0.5
    b = torch.randn(N, generator=g) * 0.1
    want = x.double() @ W.double() + b.double()
    if relu:
        want = want.clamp_min(0)
    a = ops.raw_tc_split(x.to(DEV))
    assert _err(_join(a, K), x.double()) < 2e-5           # the split itself
    Wp, WTp = ops.raw_tc_prep_weight(W.to(DEV))
    assert _err(_join(Wp, N), W.double()) < 2e-5
    assert _err(_join(WTp, K), W.double().t()) < 2e-5
    y, yp = ops.raw_tc_linear_fwd(a, K, WTp, N, b.to(DEV), relu, True, True)
    torch.cuda.synchronize()
    assert _err(y, want) < 5e-5
    assert _err(_join(yp, N), want) < 5e-5
    # no bias, planes only
    y2, yp2 = ops.raw_tc_linear_fwd(a, K, WTp, N, None, relu, False, True)
    want2 = x.double() @ W.double()
    if relu:
        want2 = want2.clamp_min(0)
    assert y2 is None and _err(_join(yp2, N), want2) < 5e-5


@pytest.mark.parametrize("bn", [16, 64, 128, 224])
@pytest.mark.parametrize("bk", [32, 64])
def test_tc_linear_fwd_tile_shapes(bn, bk):
    """Forced tile widths (rounded up to a compiled one: 16, 64, 128, 256) and both k-block / swizzle
    variants (64 B and 128 B rows); the three calls emit fp32 only, planes only and both."""
    ops = _ops()
    g = torch.Generator().manual_seed(bn)
    M, N, K = 700, 400, 624
    x = torch.randn(M, K, generator=g)
    W = torch.randn(K, N, generator=g) / K ** 0.5
    a = ops.raw_tc_split(x.to(DEV))
    _, WTp = ops.raw_tc_prep_weight(W.to(DEV))
    ops.tc_debug(0, bn)
    ops.tc_debug(4, bk)
    try:
        y, _ = ops.raw_tc_linear_fwd(a, K, WTp, N, None, False, True, False)
        _, yp = ops.raw_tc_linear_fwd(a, K, WTp, N, None, False, False, True)
        y2, yp2 = ops.raw_tc_linear_fwd(a, K, WTp, N, None, False, True, True)
        torch.cuda.synchronize()
    finally:
        ops.tc_debug(0, 0)
        ops.tc_debug(4, 64)
    want = x.double() @ W.double()
    assert _err(y, want) < 5e-5 and _err(_join(yp, N), want) < 5e-5
    assert torch.equal(y, y2) and torch.equal(yp[:, :N], yp2[:, :N])


@pytest.mark.parametrize("M,K,N", [(257, 624, 400), (5000, 400, 400), (300, 127, 1)])
def test_tc_bias_row_from_ones_column(M, K, N):
    """ones_col: the operand planes carry hi[:, K] = 1, the forward GEMM must ignore it (its tensor
    map stops at K) and the dW GEMM over K+1 rows returns colsum(g) as the extra row."""
    ops = _ops()
    g_ = torch.Generator().manual_seed(M + K)
    x = torch.randn(M, K, generator=g_)
    W = torch.randn(K, N, generator=g_) / K ** 0.5
    gy = torch.randn(M, N, generator=g_)
    a = ops.raw_tc_split(x.to(DEV), ones_col=True)
    _, WTp = ops.raw_tc_prep_weight(W.to(DEV), want_w=False)
    y, yp = ops.raw_tc_linear_fwd(a, K, WTp, N, None, False, True, True, ones_col=True)
    assert _err(y, x.double() @ W.double()) < 5e-5
    ld = yp.shape[1] // 2
    assert ld >= N + 1
    assert torch.all(yp[:, N].float() == 1) and torch.all(yp[:, ld + N].float() == 0)
    gp, _ = ops.raw_tc_split_bwd(gy.to(DEV), None)
    dW, db = ops.raw_tc_linear_bwd_dw(a, K, gp, N, bias_row=True)
    torch.cuda.synchronize()
    assert _err(dW, x.double().t() @ gy.double()) < 5e-5
    assert _err(db, gy.double().sum(0)) < 5e-5


@pytest.mark.parametrize("M,K,N", [(257, 624, 400), (1000, 400, 400), (300, 400, 1), (4096, 400, 624),
                                   (130, 9, 33)])
@pytest.mark.parametrize("masked", [False, True])
def test_tc_linear_bwd_dx(M, K, N, masked):
    """dx = g @ W^T; masked: by the hi plane of the layer input, + column sums (bias gradient)."""
    ops = _ops()
    g_ = torch.Generator().manual_seed(M + K + N)
    gy = torch.randn(M, N, generator=g_)
    W = torch.randn(K, N, generator=g_) / N ** 0.5
    act = torch.randn(M, K, generator=g_).clamp_min(0)     # a ReLU output: ~half zeros
    gp, db_top = ops.raw_tc_split_bwd(gy.to(DEV), None)
    assert _err(db_top, gy.double().sum(0)) < 1e-5
    Wp, _ = ops.raw_tc_prep_weight(W.to(DEV))
    ap = ops.raw_tc_split(act.to(DEV))
    want = gy.double() @ W.double().t()
    if masked:
        want = want * (act.double() > 0)
        dx, dxp, db = ops.raw_tc_linear_bwd_dx(gp, N, Wp, K, ap, True, True, True)
        torch.cuda.synchronize()
        assert _err(db, want.sum(0)) < 5e-5
        assert _err(_join(dxp, K), want) < 5e-5
    else:
        dx, dxp, db = ops.raw_tc_linear_bwd_dx(gp, N, Wp, K, None, True, False, False)
        torch.cuda.synchronize()
        assert dxp is None and db is None
    assert _err(dx, want) < 5e-5


@pytest.mark.parametrize("M,K,N", [(257, 624, 400), (4096, 400, 400), (1000, 400, 1), (8192, 624, 400),
                                   (33, 9, 33), (70000, 128, 64)])
def test_tc_linear_bwd_dw(M, K, N):
    ops = _ops()
    g_ = torch.Generator().manual_seed(M + 2 * K + N)
    a = torch.randn(M, K, generator=g_)
    gy = torch.randn(M, N, generator=g_)
    ap = ops.raw_tc_split(a.to(DEV))
    gp, _ = ops.raw_tc_split_bwd(gy.to(DEV), None)
    dW = ops.raw_tc_linear_bwd_dw(ap, K, gp, N)
    torch.cuda.synchronize()
    assert _err(dW, a.double().t() @ gy.double()) < 5e-5
    dW2 = ops.raw_tc_linear_bwd_dw(ap, K, gp, N)      # deterministic: fixed-order reduce
    assert torch.equal(dW, dW2)


@pytest.mark.parametrize("bk", [32, 64])
def test_tc_many_tiles_per_cta(bk):
    """More output tiles than SMs: every CTA walks several tiles while the producer already streams
    the next tile's k-blocks into the pipeline stages the epilogue of the previous one has freed;
    rows 39936.. exercise the partially valid last row block.  Both k-block widths (pipeline depths)."""
    ops = _ops()
    ops.tc_debug(4, bk)
    g_ = torch.Generator().manual_seed(77)
    M, K, N = 40003, 400, 64
    x = torch.randn(M, N, generator=g_)
    W = torch.randn(N, K, generator=g_) / N ** 0.5
    b = torch.randn(K, generator=g_) * 0.1
    a = ops.raw_tc_split(x.to(DEV))
    _, WTp = ops.raw_tc_prep_weight(W.to(DEV), want_w=False)
    y, yp = ops.raw_tc_linear_fwd(a, N, WTp, K, b.to(DEV), True, True, True, ones_col=True)
    want = (x.double() @ W.double() + b.double()).clamp_min(0)
    assert _err(y, want) < 5e-5 and _err(_join(yp, K), want) < 5e-5
    # backward of the same layer, vector epilogue with the ReLU mask (no column sums)
    gy = torch.randn(M, K, generator=g_)
    W2 = torch.randn(N, K, generator=g_) / K ** 0.5          # dx [M,N] = g [M,K] @ W2^T
    gp, _ = ops.raw_tc_split_bwd(gy.to(DEV), yp)             # top split masked by relu(y)
    # the mask is what the kernel emitted (hi plane > 0): a logit within rounding of 0 may round
    # to either side of the fp64 value's sign, that is not an error of the backward kernel
    wantg = gy.double() * (yp[:, :K].double().cpu() > 0)
    assert _err(_join(gp, K), wantg) < 5e-5
    act = torch.randn(M, N, generator=g_).clamp_min(0)
    ap = ops.raw_tc_split(act.to(DEV), ones_col=True)
    Wp, _ = ops.raw_tc_prep_weight(W2.to(DEV), want_wt=False)
    dx, dxp, _ = ops.raw_tc_linear_bwd_dx(gp, K, Wp, N, ap, True, True, False)
    torch.cuda.synchronize()
    wantdx = (wantg @ W2.double().t()) * (act.double() > 0)
    assert _err(dx, wantdx) < 5e-5 and _err(_join(dxp, N), wantdx) < 5e-5
    ops.tc_debug(4, 64)
    # element-wise on the tail rows (a max-norm bound would hide one bad row)
    assert _err(dx[-80:], wantdx[-80:]) < 5e-5


def test_tc_cross_fwd():
    """CrossNetV2 layer (dcn_v2/net.py:222-226): x0 * (xl @ W + b) + xl in the GEMM epilogue."""
    ops = _ops()
    g = torch.Generator().manual_seed(5)
    M, C = 777, 1560
    x0 = torch.randn(M, C, generator=g)
    xl = torch.randn(M, C, generator=g)
    W = torch.randn(C, C, generator=g) / C ** 0.5
    b = torch.randn(C, generator=g) * 0.1
    xlp = ops.raw_tc_split(xl.to(DEV))
    _, WTp = ops.raw_tc_prep_weight(W.to(DEV), want_w=False)
    out, outp, u = ops.raw_tc_cross_fwd(xlp, WTp, b.to(DEV), x0.to(DEV), xl.to(DEV), True,
                                        want_u=True)
    torch.cuda.synchronize()
    wantu = xl.double() @ W.double() + b.double()
    want = x0.double() * wantu + xl.double()
    assert _err(u, wantu) < 5e-5
    assert _err(out, want) < 5e-5
    assert _err(_join(outp, C), want) < 5e-5


def test_cross_v2_layer_chain_autograd():
    """Two chained CrossNetV2 layers through ops.cross_v2 on the wgmma back end (the second
    consumes the planes the first one's epilogue emitted): output and every gradient vs fp64."""
    from paddlerec_b200 import nn as bnn
    from tests.util import rel_err
    ops = _ops()
    g = torch.Generator().manual_seed(9)
    M, C = 300, 200
    x0 = torch.randn(M, C, generator=g)
    Ws = [torch.randn(C, C, generator=g) / C ** 0.5 for _ in range(2)]
    bs = [torch.randn(C, generator=g) * 0.1 for _ in range(2)]
    gy = torch.randn(M, C, generator=g)
    x0d = x0.double().requires_grad_(True)
    Wd = [w.double().requires_grad_(True) for w in Ws]
    bd = [b.double().requires_grad_(True) for b in bs]
    xi = x0d
    for W, b in zip(Wd, bd):
        xi = xi + x0d * (xi @ W + b)
    (xi * gy.double()).sum().backward()
    x0c = x0.to(DEV).requires_grad_(True)
    Wc = [w.to(DEV).requires_grad_(True) for w in Ws]
    bc = [b.to(DEV).requires_grad_(True) for b in bs]
    xc, planes = x0c, None
    for W, b in zip(Wc, bc):
        xc, planes = ops.cross_v2(x0c, xc, W, b, bnn.mm, "bf16x3", xl_planes=planes)
    (xc * gy.to(DEV)).sum().backward()
    torch.cuda.synchronize()
    assert rel_err(xc, xi) < 1e-4 and rel_err(x0c.grad, x0d.grad) < 1e-4
    for a, b in zip(Wc + bc, Wd + bd):
        assert rel_err(a.grad, b.grad) < 1e-4


def test_tc_linear_autograd_small_and_odd_shapes():
    """nn.Linear in bf16x3 precision = ops.tc_linear: shapes the models actually use (13 -> 13*D,
    K = 13, N = 1, 3-D inputs)."""
    from tests.util import rel_err
    ops = _ops()
    g = torch.Generator().manual_seed(21)
    for lead, K, N in [((70,), 13, 208), ((33,), 256, 1), ((4, 25), 128, 80), ((129,), 40, 7)]:
        x = torch.randn(*lead, K, generator=g)
        W = torch.randn(K, N, generator=g) / K ** 0.5
        b = torch.randn(N, generator=g) * 0.1
        gy = torch.randn(*lead, N, generator=g)
        xd, Wd, bd = (t.double().requires_grad_(True) for t in (x, W, b))
        ((xd @ Wd + bd) * gy.double()).sum().backward()
        xc, Wc, bc = (t.to(DEV).requires_grad_(True) for t in (x, W, b))
        y = ops.tc_linear(xc, Wc, bc)
        (y * gy.to(DEV)).sum().backward()
        torch.cuda.synchronize()
        assert rel_err(y, x.double() @ W.double() + b.double()) < 5e-5
        for a, r in ((xc, xd), (Wc, Wd), (bc, bd)):
            assert rel_err(a.grad, r.grad) < 5e-5, (lead, K, N)


@pytest.mark.parametrize("sizes", [[624, 400, 400, 400, 1], [429, 512, 256, 128, 32]])
@pytest.mark.parametrize("last_act", [False, True])
@pytest.mark.parametrize("backend", ["tcgen05", "tcgen05+overlap", "cublas"])
def test_tower_backends_match_fp64(backend, last_act, sizes):
    """The whole tower (forward + every gradient) on both back ends, headline shape."""
    from paddlerec_b200 import tower
    from tests.util import rel_err
    g = torch.Generator().manual_seed(11)
    M = 1100
    L = len(sizes) - 1
    x = torch.randn(M, sizes[0], generator=g)
    Ws = [torch.randn(sizes[i], sizes[i + 1], generator=g) / sizes[i] ** 0.5 for i in range(L)]
    bs = [torch.randn(sizes[i + 1], generator=g) * 0.1 for i in range(L)]
    # ReLU is not differentiable at 0: a pre-activation within rounding of 0 may land on either
    # side in fp32 and flip that unit's whole gradient path, which is not an error of either
    # implementation.  Drop the (few) samples that have any pre-activation that close to 0.
    keep = torch.ones(M, dtype=torch.bool)
    h = x.double()
    for i in range(L):
        z = h @ Ws[i].double() + bs[i].double()
        if i < L - 1 or last_act:
            keep &= (z.abs() > 1e-4).all(1)
            h = torch.relu(z)
    x = x[keep].contiguous()
    M = x.shape[0]
    assert 700 < M < 1100
    xd = x.double().requires_grad_(True)
    Wd = [w.double().requires_grad_(True) for w in Ws]
    bd = [b.double().requires_grad_(True) for b in bs]
    h = xd
    for i in range(L):
        h = h @ Wd[i] + bd[i]
        if i < L - 1 or last_act:
            h = torch.relu(h)
    gy = torch.randn(M, sizes[-1], generator=g)
    (h * gy.double()).sum().backward()
    xc = x.to(DEV).requires_grad_(True)
    Wc = [w.to(DEV).requires_grad_(True) for w in Ws]
    bc = [b.to(DEV).requires_grad_(True) for b in bs]
    prev = tower.BACKEND
    tower.set_backend(backend.split("+")[0])
    tower.set_overlap_dw(backend.endswith("overlap"))   # dW GEMMs on the side stream
    try:
        y = tower.mlp(xc, Wc, bc, last_act=last_act)
        (y * gy.to(DEV)).sum().backward()
        assert bool(tower._PENDING) == backend.endswith("overlap")
        tower.wait_pending()        # what the optimizers do before they touch the gradients
        torch.cuda.current_stream().synchronize()
    finally:
        tower.set_backend(prev)
        tower.set_overlap_dw(False)
    assert rel_err(y, h) < 1e-4
    assert rel_err(xc.grad, xd.grad) < 1e-4
    for a, b in zip(Wc + bc, Wd + bd):
        assert rel_err(a.grad, b.grad) < 1e-4


@pytest.mark.parametrize("M,K", [(1000, 400), (257, 8), (5000, 2048), (70, 520)])
def test_tc_head_width1_layer(M, K):
    """The streaming kernels of the width-1 head (forward GEMV, backward outer product + mask +
    split + dW/db) vs fp64."""
    ops = _ops()
    g_ = torch.Generator().manual_seed(M + K)
    act = torch.randn(M, K, generator=g_).clamp_min(0)
    w = torch.randn(K, 1, generator=g_) / K ** 0.5
    b = torch.randn(1, generator=g_)
    dy = torch.randn(M, 1, generator=g_)
    ap = ops.raw_tc_split(act.to(DEV))
    a64 = _join(ap, K).cpu()                      # what the kernel actually reads (hi + lo)
    y = ops.raw_tc_head_fwd(ap, K, w.to(DEV), b.to(DEV))
    assert _err(y, a64 @ w.double() + b.double()) < 1e-5
    gp, dW, db = ops.raw_tc_head_bwd(ap, K, w.to(DEV), dy.to(DEV))
    torch.cuda.synchronize()
    want_g = (dy.double() @ w.double().t()) * (ap[:, :K].double().cpu() > 0)
    assert _err(_join(gp, K), want_g) < 2e-5
    assert _err(dW, a64.t() @ dy.double()) < 1e-5
    assert abs(float(db) - float(dy.double().sum())) < 1e-5 * float(dy.abs().sum())
    gp2, dW2, db2 = ops.raw_tc_head_bwd(ap, K, w.to(DEV), dy.to(DEV))
    assert torch.equal(dW, dW2) and torch.equal(db, db2)        # deterministic


@pytest.mark.parametrize("M,N,K", [(20000, 400, 624), (4099, 624, 400), (8192, 40, 1560)])
def test_tc_large_m_every_output_kind(M, N, K):
    """Tower-sized row counts with several tiles per CTA: forward with every output kind, masked
    dX, odd tile counts."""
    ops = _ops()
    g = torch.Generator().manual_seed(M + N)
    x = torch.randn(M, K, generator=g)
    W = torch.randn(K, N, generator=g) / K ** 0.5
    b = torch.randn(N, generator=g) * 0.1
    a = ops.raw_tc_split(x.to(DEV))
    Wp, WTp = ops.raw_tc_prep_weight(W.to(DEV))
    want = (x.double() @ W.double() + b.double()).clamp_min(0)
    y, _ = ops.raw_tc_linear_fwd(a, K, WTp, N, b.to(DEV), True, True, False)
    _, yp = ops.raw_tc_linear_fwd(a, K, WTp, N, b.to(DEV), True, False, True, ones_col=True)
    gy = torch.randn(M, N, generator=g)
    gp, _ = ops.raw_tc_split_bwd(gy.to(DEV), None)
    dx, _, _ = ops.raw_tc_linear_bwd_dx(gp, N, Wp, K, None, True, False, False)
    _, dxp, _ = ops.raw_tc_linear_bwd_dx(gp, N, Wp, K, a, False, True, False)
    torch.cuda.synchronize()
    assert _err(y, want) < 5e-5 and _err(_join(yp, N), want) < 5e-5
    wdx = gy.double() @ W.double().t()
    assert _err(dx, wdx) < 5e-5
    assert _err(_join(dxp, K), wdx * (a[:, :K].double().cpu() > 0)) < 5e-5


def test_ctr_head_fused_ops():
    """sum_sigmoid and log_loss_mean (one kernel each way) vs the torch composition in fp64, float
    and int64 labels, gradients through both."""
    ops = _ops()
    g = torch.Generator().manual_seed(3)
    n = 70001
    parts = [torch.randn(n, 1, generator=g) for _ in range(3)]
    label_f = (torch.rand(n, 1, generator=g) < 0.3).float()
    for label in (label_f, label_f.long()):
        pd = [t.double().requires_grad_(True) for t in parts]
        pr = torch.sigmoid(pd[0] + pd[1] + pd[2])
        y = label.double()
        lr = (-y * torch.log(pr + 1e-4) - (1 - y) * torch.log(1 - pr + 1e-4)).mean()
        lr.backward()
        pc = [t.to(DEV).requires_grad_(True) for t in parts]
        pred = ops.sum_sigmoid(*pc)
        loss = ops.log_loss_mean(pred, label.to(DEV))
        loss.backward()
        torch.cuda.synchronize()
        assert pred.shape == (n, 1) and _err(pred, pr.detach()) < 1e-6
        assert abs(float(loss) - float(lr)) < 1e-6 * abs(float(lr))
        for a, b in zip(pc, pd):
            assert _err(a.grad, b.grad) < 1e-5
        loss2 = ops.log_loss_mean(pred.detach(), label.to(DEV))
        assert float(loss2) == float(loss)           # deterministic reduction
    two = ops.sum_sigmoid(parts[0].to(DEV), parts[1].to(DEV))
    assert _err(two, torch.sigmoid(parts[0].double() + parts[1].double())) < 1e-6
