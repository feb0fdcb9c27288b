"""ESMM on the H100: the head kernels against fp64 (at a batch where every CTA loops, K in {8, 64,
200}, saturated logits of both signs, the gradient of each output alone and of all six), the pooled
lookup with padding and out-of-range ids, the model against both goldens in both tower precisions,
one step at the config shape (B = 65536, V = 737946) against an fp64 torch step from the same state,
and the trainer / infer loop on the model directory's config.yaml."""
import os

import numpy as np
import pytest
import torch

from tests import esmm_oracle
from tests.util import load_golden, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"
OUTS = ("ctr_out", "ctr_one", "cvr_out", "cvr_one", "ctcvr_prop", "ctcvr_one")
F, L, D = 23, 3, 12


@pytest.fixture(autouse=True)
def _reset_oob():
    """The out-of-range counter is process-wide: leave it at zero for the modules that follow."""
    yield
    from paddlerec_b200 import ops
    ops.raw_oob_count(reset=True)


# ---- the head kernels against fp64 ---------------------------------------------------------------
def _head_problem(B, K, seed):
    """h >= 0 (ReLU'd), W and b fp32; in every fifth row the logit gap is 25..60 in size, with both
    signs, in both towers."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    hs, Ws, bs = [], [], []
    for _ in range(2):
        h = torch.relu(torch.randn(B, K, device=DEV, generator=g))
        W = torch.randn(K, 2, device=DEV, generator=g) / K ** 0.5
        b = torch.randn(2, device=DEV, generator=g) * 0.1
        # a saturated row has one nonzero activation, at the column of W1 - W0's largest (even
        # rows) or smallest (odd rows) entry: its logit gap is large without cancelling terms
        dW = W[:, 1] - W[:, 0]
        rows = torch.arange(0, B, 5, device=DEV)
        col = torch.where(rows % 2 == 0, dW.argmax(), dW.argmin())
        want = 25 + 35 * torch.rand(rows.numel(), device=DEV, generator=g)
        h[rows] = 0
        h[rows, col] = want / dW[col].abs()
        hs.append(h.contiguous())
        Ws.append(W)
        bs.append(b)
    return hs, Ws, bs


def _ref_forward(h, W, b):
    """fp64 logits, both classes computed on their own, and the per-row magnitude sum |h||W| + |b|."""
    z = h.double() @ W.double() + b.double()
    mag = (h.double().abs() @ W.double().abs()).sum(1) + b.double().abs().sum()
    d = z[:, 0] - z[:, 1]
    p1 = 1 / (1 + torch.exp(d))
    p0 = 1 / (1 + torch.exp(-d))
    return p0, p1, mag


@pytest.mark.parametrize("K", [8, 64, 200])
def test_esmm_head_kernels_vs_fp64(K):
    from paddlerec_b200 import ops
    B = 3 * 65536 + 17
    (hc, hv), (Wc, Wv), (bc, bv) = _head_problem(B, K, K)
    outs = ops.raw_esmm_head_fwd(hc, hv, Wc, bc, Wv, bv)
    pc0, pc1, mc = _ref_forward(hc, Wc, bc)
    pv0, pv1, mv = _ref_forward(hv, Wv, bv)
    # each class against fp64, relative to itself: the small class of a saturated row included
    for got, p0, p1, mag in ((outs[0], pc0, pc1, mc), (outs[2], pv0, pv1, mv)):
        for c, p in ((0, p0), (1, p1)):
            bound = 2e-6 * (p0 * p1 * mag + p) + 1e-300
            assert float(((got[:, c].double() - p).abs() / bound).max()) <= 1.0, (K, c)
    sat_c = (pc0 < 1e-10) | (pc1 < 1e-10)
    sat_v = (pv0 < 1e-10) | (pv1 < 1e-10)
    for p0, p1 in ((pc0, pc1), (pv0, pv1)):          # both signs of saturation occur in both towers
        assert bool((p0 < 1e-10).any()) and bool((p1 < 1e-10).any())
    assert bool((outs[0][sat_c].min(1).values > 0).all()) and bool((outs[2][sat_v].min(1).values > 0).all())
    assert torch.equal(outs[1][:, 0], outs[0][:, 1]) and torch.equal(outs[3][:, 0], outs[2][:, 1])
    one = pc1 * pv1
    # + half the spacing of fp32's subnormals: the product of two saturated classes can be one
    e_one = 2e-6 * (pc0 * pc1 * mc * pv1 + pv0 * pv1 * mv * pc1 + 2 * one) + 2.0 ** -150
    assert float(((outs[5][:, 0].double() - one).abs() / e_one).max()) <= 1.0
    assert torch.equal(outs[4][:, 1], outs[5][:, 0])
    assert float(((outs[4][:, 0].double() - (1 - one)).abs() - e_one).max()) <= 1.2e-7

    # the backward: each output's gradient alone, then all six
    gen = torch.Generator(device=DEV).manual_seed(100 + K)
    gs = [torch.randn(B, 2 if i % 2 == 0 else 1, device=DEV, generator=gen) for i in range(6)]
    p_ctr, p_cvr = outs[0], outs[2]
    P = [p_ctr.double(), p_cvr.double()]
    for pick in [[i] for i in range(6)] + [list(range(6))]:
        grads = [gs[i] if i in pick else None for i in range(6)]
        got = ops.raw_esmm_head_bwd(grads, p_ctr, p_cvr, hc, hv, Wc, Wv)
        z = torch.zeros(B, 2, device=DEV, dtype=torch.float64)
        G = [z if t is None else t.double() if t.shape[1] == 2 else torch.cat([torch.zeros_like(t), t], 1).double()
             for t in grads]
        Gc = G[4][:, 1] - G[4][:, 0] + G[5][:, 1]
        Gm = G[4].abs().sum(1) + G[5][:, 1].abs()
        Gt = [G[0] + G[1], G[2] + G[3]]
        Gt[0][:, 1] += Gc * P[1][:, 1]
        Gt[1][:, 1] += Gc * P[0][:, 1]
        mags = [(G[0] + G[1]).abs().sum(1) + Gm * P[1][:, 1], (G[2] + G[3]).abs().sum(1) + Gm * P[0][:, 1]]
        for t, (h, W) in enumerate(((hc, Wc), (hv, Wv))):
            p = P[t]
            s = p[:, 0] * p[:, 1] * (Gt[t][:, 1] - Gt[t][:, 0])
            ms = p[:, 0] * p[:, 1] * mags[t]
            dz = torch.stack([-s, s], 1)
            W64 = W.double()
            dh_ref = dz @ W64.t()
            # + a few subnormal spacings: s of a row saturated in both towers can be subnormal
            tiny = 2.0 ** -146
            dh_bound = (2e-6 * ms[:, None] + tiny) * W64.abs().sum(1)[None, :] + tiny
            assert float(((got[t].double() - dh_ref).abs() - dh_bound).max()) <= 0, (K, pick, t)
            dW_ref = h.double().t() @ dz
            dW_bound = 2e-6 * (h.double().abs().t() @ (ms + tiny))[:, None] + 1e-300
            assert float(((got[2 + 2 * t].double() - dW_ref).abs() - dW_bound).max()) <= 0, (K, pick, t)
            db_bound = 2e-6 * float((ms + tiny).sum()) + 1e-300
            assert float((got[3 + 2 * t].double() - dz.sum(0)).abs().max()) <= db_bound, (K, pick, t)
    again = ops.raw_esmm_head_bwd(grads, p_ctr, p_cvr, hc, hv, Wc, Wv)
    assert all(torch.equal(a, b) for a, b in zip(got, again))       # fixed-order sums: bit-identical


def test_esmm_head_formulas_are_the_softmax_product_backward():
    """The kernel's gradient formulas equal fp64 autograd through the reference's head."""
    from paddlerec_b200 import ops
    from paddlerec_b200.multitask.esmm import net
    B, K = 1000, 64
    (hc, hv), (Wc, Wv), (bc, bv) = _head_problem(B, K, 3)
    gen = torch.Generator(device=DEV).manual_seed(4)
    gs = [torch.randn(B, 2 if i % 2 == 0 else 1, device=DEV, generator=gen) for i in range(6)]
    leaves = [t.double().requires_grad_(True) for t in (hc, hv, Wc, bc, Wv, bv)]
    ref = net.torch_head(*leaves)
    sum((r * g.double()).sum() for r, g in zip(ref, gs)).backward()
    hc1, hv1, Wc1, bc1, Wv1, bv1 = [t.detach().clone().requires_grad_(True) for t in (hc, hv, Wc, bc, Wv, bv)]
    got = ops.esmm_head(hc1, hv1, Wc1, bc1, Wv1, bv1)
    sum((o * g).sum() for o, g in zip(got, gs)).backward()
    for a, b in zip((hc1, hv1, Wc1, bc1, Wv1, bv1), leaves):
        assert rel_err(a.grad, b.grad) <= 1e-5


def test_esmm_head_rejects_unsupported_shapes():
    from paddlerec_b200 import _lib, ops
    B = 64
    for K in (6, 260):
        h = torch.rand(B, K, device=DEV)
        W, b = torch.rand(K, 2, device=DEV), torch.rand(2, device=DEV)
        with pytest.raises(_lib.B200RecError, match="K="):
            ops.raw_esmm_head_fwd(h, h, W, b, W, b)
        with pytest.raises(_lib.B200RecError, match="K="):
            ops.raw_esmm_head_bwd([None] * 6, torch.rand(B, 2, device=DEV), torch.rand(B, 2, device=DEV),
                                  h, h, W, W)
    K = 64
    buf = torch.rand(B * K + 1, device=DEV)
    h_bad = buf[1:].view(B, K)                       # contiguous, 4 bytes past a 16-byte boundary
    h = torch.rand(B, K, device=DEV)
    W, b = torch.rand(K, 2, device=DEV), torch.rand(2, device=DEV)
    with pytest.raises(_lib.B200RecError, match="aligned"):
        ops.raw_esmm_head_fwd(h_bad, h, W, b, W, b)
    p = torch.rand(B, 2, device=DEV)
    with pytest.raises(_lib.B200RecError, match="aligned"):
        ops.raw_esmm_head_bwd([None] * 6, p, p, h, h_bad, W, W)


# ---- the pooled lookup -------------------------------------------------------------------------
def test_pooled_lookup_with_padding_and_out_of_range_ids():
    from paddlerec_b200 import ops
    from paddlerec_b200.multitask.esmm import net
    V, B = 5000, 4099
    torch.manual_seed(1)
    layer = net.ESMMLayer(V, D, F, [32, 16], [32, 16], device=DEV)
    g = torch.Generator(device=DEV).manual_seed(2)
    ids = torch.randint(0, V, (B, F, L), device=DEV, generator=g)
    ids[:, :, 2][torch.rand(B, F, device=DEV, generator=g) < 0.3] = 0       # padded bags
    ids[7] = 0                                                               # an all-padding sample
    ids[11, 4, 1] = ids[11, 4, 0]                                            # a repeated id in a bag
    ids[3, 0, 0], ids[5, 6, 2], ids[9, 22, 1] = -1, V, V + 5                 # out of range
    ops.raw_oob_count(reset=True)
    x = layer.pooled_input(ids)
    assert ops.raw_oob_count(reset=True) == 3
    W = layer.embedding.weight.double()
    ok = (ids > 0) & (ids < V)
    ref = (W[ids.clamp(0, V - 1)] * ok[..., None]).sum(2).reshape(B, F * D)
    assert float((x.double() - ref).abs().max()) <= 1e-6
    assert not x[7].any()
    dx = torch.randn(B, F * D, device=DEV, generator=g)
    (x * dx).sum().backward()
    assert ops.raw_oob_count(reset=True) == 3        # the id grouping counts them again, as for gather
    dW = layer.embedding.grad_rows.to_dense().double()
    flat = ids.reshape(-1)
    keep = (flat > 0) & (flat < V)
    rows = dx.double().reshape(B, F, 1, D).expand(B, F, L, D).reshape(-1, D)
    want = torch.zeros(V, D, device=DEV, dtype=torch.float64).index_add_(0, flat[keep], rows[keep])
    assert float((dW - want).abs().max()) <= 1e-5 * float(want.abs().max())
    assert not dW[0].any()


# ---- the model against the goldens -------------------------------------------------------------
def _run_golden(name, precision):
    from paddlerec_b200 import nn as bnn
    from paddlerec_b200.multitask.esmm import dygraph_model, net
    gold = load_golden(name)
    n_ctr, n_cvr = esmm_oracle.tower_sizes(gold["param"])
    ctr = [gold["param"]["linear_%d.weight" % i].shape[1] for i in range(n_ctr - 1)]
    cvr = [gold["param"]["linear_%d.weight" % (n_ctr + i)].shape[1] for i in range(n_cvr - 1)]
    V = gold["param"]["embedding.weight"].shape[0]
    layer = net.ESMMLayer(V, D, F, ctr, cvr, device=DEV)
    layer.load_state_dict({k: torch.tensor(v, dtype=torch.float32) for k, v in gold["param"].items()})
    dm = dygraph_model.DygraphModel()
    ids, clk, buy = dm.create_feeds([torch.tensor(gold["in"][k]) for k in ("ids", "clk", "buy")],
                                    {"hyper_parameters.max_len": L})
    prev = bnn.get_matmul_precision()
    bnn.set_matmul_precision(precision)
    try:
        x = layer.pooled_input(ids)
        z = [layer._hidden(x, lin) @ lin[-1].weight + lin[-1].bias
             for lin in (layer._ctr_linears, layer._cvr_linears)]
        outs = layer(ids)
        loss = dm.create_loss(outs[1], clk, outs[5], buy)
        loss.backward()
    finally:
        bnn.set_matmul_precision(prev)
    return gold, layer, z, outs, loss


@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
@pytest.mark.parametrize("name", ["esmm_init", "esmm_saturated"])
def test_esmm_layer_matches_golden(name, precision):
    gold, layer, z, outs, loss = _run_golden(name, precision)
    for k, v in zip(("z_ctr", "z_cvr"), z):
        assert rel_err(v, gold["out"][k]) <= 1e-4, k
    for k, o in zip(OUTS, outs):
        assert float(np.abs(o.detach().cpu().numpy() - gold["out"][k]).max()) <= 1e-4, k
    assert abs(float(loss.detach()) - float(gold["out"]["loss"])) <= 1e-4 * abs(float(gold["out"]["loss"]))
    named = dict(layer.named_parameters())
    # bf16x3's towers carry the logits with ~1e-5 absolute error; through a saturated softmax the
    # gradient scales with p0 p1 = O(exp(-|z1 - z0|)), so that error becomes a relative one
    tol = 5e-4 if (precision == "bf16x3" and name == "esmm_saturated") else 1e-4
    for k, want in gold["grad"].items():
        got = layer.embedding.grad_rows.to_dense() if k == "embedding.weight" else named[k].grad
        assert rel_err(got, want) <= tol, (k, rel_err(got, want))


# ---- one step at the config shape -----------------------------------------------------------------
def test_esmm_config_shape_step_vs_fp64():
    from paddlerec_b200 import functional as BF
    from paddlerec_b200 import nn as bnn
    from paddlerec_b200 import optim, tower
    from paddlerec_b200.multitask.esmm import dygraph_model, net
    B, V, fc, lr = 65536, 737946, [256, 64], 1e-3
    torch.manual_seed(3)
    layer = net.ESMMLayer(V, D, F, fc, fc, device=DEV)
    g = torch.Generator(device=DEV).manual_seed(4)
    ids = torch.randint(1, V, (B, F, L), device=DEV, generator=g)
    ids[torch.rand(B, F, L, device=DEV, generator=g) < 0.2] = 0
    clk = (torch.rand(B, 1, device=DEV, generator=g) < 0.3).to(torch.int64)
    buy = clk * (torch.rand(B, 1, device=DEV, generator=g) < 0.2).to(torch.int64)
    p64 = {k: v.detach().double().clone().requires_grad_(True) for k, v in layer.state_dict().items()}
    W0 = layer.embedding.weight.detach().clone()
    dm = dygraph_model.DygraphModel()
    opt = optim.Adam(learning_rate=lr, parameters=layer.parameters(), lazy_mode=True)
    prev = bnn.get_matmul_precision()
    bnn.set_matmul_precision("bf16x3")
    try:
        outs = layer(ids)
        loss = dm.create_loss(outs[1], clk, outs[5], buy)
        metrics, _ = dm.create_metrics()
        metrics[0].update(outs[0].detach(), clk)
        metrics[1].update(outs[4].detach(), buy)
        loss.backward()
        grad_rows = layer.embedding.grad_rows.to_dense().double()
        opt.step()
        torch.cuda.synchronize()
    finally:
        bnn.set_matmul_precision(prev)

    # fp64 torch step from the same state: the reference's op sequence, then Adam on touched rows
    inputs = [ids[:, f, :] for f in range(F)]
    ref = esmm_oracle.esmm_forward(p64, inputs, 3, 3)
    ref_loss = esmm_oracle.esmm_loss(ref[1], clk, ref[5], buy)
    ref_loss.backward()
    assert abs(float(loss.detach()) - float(ref_loss.detach())) <= 1e-4 * float(ref_loss.detach())
    for o, r in zip(outs, ref):
        assert float((o.detach().double() - r.detach()).abs().max()) <= 1e-4
    # the AUC histograms: a sample may change bucket only where fp64 puts it within 1e-5 of an edge
    for m, r, lab in ((metrics[0], ref[0], clk), (metrics[1], ref[4], buy)):
        ref_m = BF.Auc("ROC")
        ref_m.update(r.detach().float(), lab)
        p = r.detach()[:, 1] * 4095
        n_edge = int(((p - p.round()).abs() < 1e-5 * 4095).sum())
        diff = int((m.stats()[0] - ref_m.stats()[0]).abs().sum() + (m.stats()[1] - ref_m.stats()[1]).abs().sum())
        assert diff <= 2 * n_edge, (diff, n_edge)
        assert int(m.stats()[0].sum() + m.stats()[1].sum()) == B
    gW = p64["embedding.weight"].grad
    tower.wait_pending()
    # The heads' parameters element-wise.  Below them, norm-wise: among 65536 x 2 x 320 hidden units
    # a few pre-activations lie within bf16x3's error of 0, their ReLU mask differs from fp64's, and
    # each flip moves one sample's input gradient by about one of its 256 terms (the embedding rows,
    # sums over ~6 samples, inherit that); the dW sums over 65536 samples cancel to ~1/256 of their
    # terms' magnitude.
    named = dict(layer.named_parameters())
    for k in ("linear_2.weight", "linear_2.bias", "linear_5.weight", "linear_5.bias"):
        assert rel_err(named[k].grad, p64[k].grad) <= 1e-4, k

    def l2(a, b):
        return float((a.double() - b).norm() / b.norm())

    errs = {k: l2(v.grad, p64[k].grad) for k, v in named.items() if v.grad is not None}
    emb = l2(grad_rows, gW)
    assert max(errs.values()) <= 1e-3 and emb <= 5e-3, (errs, emb)
    # lazy Adam, first step: only the touched rows move, by lr_t * m / (sqrt(v) + eps * sqrt(1 - b2))
    touched = torch.zeros(V, dtype=torch.bool, device=DEV)
    touched[ids[ids > 0]] = True
    W1 = layer.embedding.weight.detach()
    assert torch.equal(W1[~touched], W0[~touched]) and not W1[0].any()
    b1, b2, eps = 0.9, 0.999, 1e-8
    lr_t = lr * (1 - b2) ** 0.5 / (1 - b1)
    gt = grad_rows[touched]          # the update applied to the gradient it was given
    step = lr_t * (1 - b1) * gt / ((1 - b2) ** 0.5 * gt.abs() + eps * (1 - b2) ** 0.5)
    got = (W1[touched].double() - W0[touched].double())
    # W is stored in fp32 (|W| <= 1: half an ulp is 6e-8), the update is computed in fp32
    assert float(((got + step).abs() - 1.5e-7 - 1e-5 * step.abs()).max()) <= 0


# ---- trainer and infer on config.yaml -----------------------------------------------------------
def test_esmm_trainer_and_infer_on_config(tmp_path):
    from paddlerec_b200 import checkpoint, runner
    from paddlerec_b200.multitask.esmm import dygraph_model
    d = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "paddlerec_b200",
                     "multitask", "esmm")
    cfg = runner.load_yaml(os.path.join(d, "config.yaml"))
    cfg["config_abs_dir"] = d
    cfg["runner.model_save_path"] = str(tmp_path / "out")
    cfg["runner.infer_load_path"] = str(tmp_path / "out")
    losses, metrics, net_ = runner.train(cfg)
    assert len(losses) == 15 and np.all(np.isfinite(losses))
    assert sorted(metrics) == ["auc_ctcvr", "auc_ctr"] and all(0.0 <= v <= 1.0 for v in metrics.values())
    results = runner.infer(cfg)
    assert sorted(results) == [0, 1, 2]
    assert all(0.0 <= v <= 1.0 for r in results.values() for v in r.values())
    fresh = dygraph_model.DygraphModel().create_model(cfg)
    runner.load_model(str(tmp_path / "out" / "2"), fresh)
    saved = checkpoint.load_pdparams(str(tmp_path / "out" / "2" / "rec.pdparams"))
    assert sorted(saved) == sorted(["embedding.weight"] + ["linear_%d.%s" % (i, k) for i in range(6)
                                                           for k in ("weight", "bias")])
    for k, v in fresh.state_dict().items():
        assert torch.equal(v, net_.state_dict()[k]), k
