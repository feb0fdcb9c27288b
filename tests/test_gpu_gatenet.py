"""GateNet on the H100: the embedding-gate kernels and the gated wgmma tower against fp64 (at sizes
where every CTA of the gate kernels loops, with a hot id, out-of-range ids and saturated gates), the
model against every golden in both tower precisions, one B=65536, V=1e6 step checked on a slice, and
the trainer / infer loop on the model directory's config.yaml."""
import os

import numpy as np
import pytest
import torch

from tests import gatenet_oracle
from tests.util import elementwise_excess, load_golden, rel_err, slots

pytestmark = pytest.mark.gpu
DEV = "cuda"
NS = 512


@pytest.fixture(autouse=True)
def _reset_oob():
    """The out-of-range counter is process-wide: leave it at zero for the modules that follow."""
    yield
    from paddlerec_b200 import ops
    ops.raw_oob_count(reset=True)


def gated_tol(n_gated):
    """bf16x3's 1e-4 bar, doubled per hidden gate: z = y * tanh(y @ G) is about quadratic in y, so each
    gated layer doubles the relative error it receives (the fp32 path keeps 1e-4)."""
    return 1e-4 * 2 ** n_gated
kThreads = 256            # kGateEmbedThreads, csrc/gate_embed.cuh
kCtasPerSm = 8            # gate_embed_grid(), csrc/gate_embed.cuh


def _sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _zipf_ids(g, n, V, hot_id, hot_count):
    u = torch.rand(n, generator=g, device=DEV, dtype=torch.float64)
    ids = ((V ** (1 - 1.05) - 1) * u + 1) ** (1 / (1 - 1.05))            # inverse CDF, s = 1.05
    ids = (ids.long() - 1).clamp(0, V - 1)
    ids[ids == hot_id] = (hot_id + 1) % V
    ids[torch.randperm(n, generator=g, device=DEV)[:hot_count]] = hot_id
    return ids


def _gate_ref(W, ids, gate_w, D):
    V = W.shape[0]
    ok = ((ids >= 0) & (ids < V)).unsqueeze(2).double()
    e = W[ids.clamp(0, V - 1), :D].double() * ok
    ew = e * gate_w.double().reshape(1, -1, 1)
    g = torch.sigmoid(ew.sum(2, keepdim=True))
    return e, g, ew.abs().sum(2, keepdim=True), ok


# ---- embedding-gate kernels --------------------------------------------------------------------
@pytest.mark.parametrize("Dn", [0, 13])
@pytest.mark.parametrize("F", [1, 26])
@pytest.mark.parametrize("D", [1, 4, 9, 16, 64])
def test_gate_embed_kernels_vs_fp64(D, F, Dn):
    from paddlerec_b200 import ops
    spb = kThreads // F
    grid = kCtasPerSm * _sm()
    B = 3 * grid * spb                       # every CTA walks 3 sample groups
    assert (B + spb - 1) // spb >= 3 * grid
    V = 200_000
    g = torch.Generator(device=DEV).manual_seed(D * 100 + F + Dn)
    W = torch.empty(V, D, device=DEV).uniform_(-1, 1, generator=g)
    ids = _zipf_ids(g, B * F, V, 12345, 3000).reshape(B, F)
    ids[5, 0], ids[7, F - 1], ids[B - 1, F // 2] = -3, V, V + 1000        # out of range
    gate_w = torch.randn(F, device=DEV, generator=g) * 2
    gate_w[0] = 60.0                          # saturates g to 1 (or 0 for negative row sums)
    if F > 2:
        gate_w[1] = -60.0
    dense = torch.rand(B, Dn, device=DEV, generator=g) if Dn else None
    ops.raw_oob_count(reset=True)
    out = ops.raw_gate_embed_fwd(W, ids, gate_w, dense, D)
    assert ops.raw_oob_count(reset=True) == 3
    e, gg, ewabs, ok = _gate_ref(W, ids, gate_w, D)
    assert float(gg.min()) < 1e-20 and float(gg.max()) == 1.0
    ref = (e * gg).reshape(B, -1)
    got = out[:, :F * D]
    assert torch.isfinite(out).all()
    bound = 2e-6 * (e.abs() * (gg + ewabs)).reshape(B, -1) + 1e-30
    assert bool(((got.double() - ref).abs() <= bound).all())
    if Dn:
        assert torch.equal(out[:, F * D:], dense)
    # backward
    dout = torch.randn(B, F * D + Dn, device=DEV, generator=g)
    drow, dgate = ops.raw_gate_embed_bwd(W, ids, gate_w, dout, D)
    do = dout[:, :F * D].double().reshape(B, F, D)
    q = (do * e).sum(2, keepdim=True)
    qabs = (do * e).abs().sum(2, keepdim=True)
    c = q * gg * (1 - gg)
    w = gate_w.double().reshape(1, -1, 1)
    ref_row = (do * gg + c * w) * ok
    mag = (do.abs() * gg + qabs * w.abs() * (1 + ewabs)) * ok
    assert bool(((drow.double().reshape(B, F, D) - ref_row).abs() <= 2e-6 * mag + 1e-30).all())
    assert bool((drow.reshape(B, F, D)[~ok.bool().squeeze(2)] == 0).all())
    se = e.sum(2, keepdim=True)
    ref_dg = (c * se).sum((0, 2))
    mag_dg = (qabs * (1 + ewabs) * e.abs().sum(2, keepdim=True)).sum((0, 2))
    assert bool(((dgate.double() - ref_dg).abs() <= 2e-6 * mag_dg + 1e-30).all())
    # the SelectedRows the autograd node builds: group_ids + segment_reduce of the rows
    groups = ops.raw_group_ids(ids, V, -1)
    assert ops.raw_oob_count(reset=True) == 3          # the grouping counts them too, as for gather
    rows = ops.raw_segment_reduce(drow, groups.seg_offsets, groups.sorted_pos, groups.num, groups.n)
    U = int(groups.num[0])
    flat = ids.reshape(-1)
    keep = (flat >= 0) & (flat < V)
    dense_ref = torch.zeros(V, D, device=DEV, dtype=torch.float64).index_add_(
        0, flat[keep], ref_row.reshape(-1, D)[keep])
    dense_mag = torch.zeros(V, D, device=DEV, dtype=torch.float64).index_add_(
        0, flat[keep], mag.reshape(-1, D)[keep])
    u = groups.unique_ids[:U]
    assert int((flat == 12345).sum()) >= 3000
    assert bool(((rows[:U].double() - dense_ref[u]).abs() <= 2e-6 * dense_mag[u] + 1e-30).all())
    # a second run is bit-identical
    out2 = ops.raw_gate_embed_fwd(W, ids, gate_w, dense, D)
    drow2, dgate2 = ops.raw_gate_embed_bwd(W, ids, gate_w, dout, D)
    assert ops.raw_oob_count(reset=True) == 3          # by the forward only, not the backward
    assert torch.equal(out, out2) and torch.equal(drow, drow2) and torch.equal(dgate, dgate2)


# ---- gated tower ---------------------------------------------------------------------------------
def _tower_ref(x, Ws, bs, Gs):
    y = x
    us, zs = [], []
    for i in range(len(Gs)):
        u = y @ Ws[i] + bs[i]
        us.append(u)
        r = torch.relu(u)
        y = r * torch.tanh(r @ Gs[i])
        zs.append(y)
    return y @ Ws[-1] + bs[-1], us, zs


@pytest.mark.parametrize("K", [247, 512])
@pytest.mark.parametrize("N", [32, 128, 256, 512])
def test_gated_tower_vs_fp64(N, K):
    from paddlerec_b200 import tower
    M = 1000
    g = torch.Generator(device=DEV).manual_seed(N + K)
    sizes = [K, N, 32, 1]
    x = torch.randn(M, K, device=DEV, generator=g)
    Ws = [(torch.randn(sizes[i], sizes[i + 1], device=DEV, generator=g) / sizes[i] ** 0.5)
          .requires_grad_(True) for i in range(3)]
    bs = [(0.1 * torch.randn(sizes[i + 1], device=DEV, generator=g)).requires_grad_(True)
          for i in range(3)]
    Gs = [(3 * torch.randn(n, n, device=DEV, generator=g) / n ** 0.5).requires_grad_(True)
          for n in (N, 32)]
    xg = x.clone().requires_grad_(True)
    out = tower.mlp(xg, Ws, bs, gates=Gs)
    # fp64 reference; samples with a ReLU near-tie anywhere are excluded (DESIGN §2)
    p64 = [t.detach().double().requires_grad_(True) for t in [x] + Ws + bs + Gs]
    ref, us, zs = _tower_ref(p64[0], p64[1:4], p64[4:7], p64[7:9])
    tie = torch.zeros(M, dtype=torch.bool, device=DEV)
    for u in us:
        tie |= (u.abs() < 1e-3 * u.square().mean().sqrt()).any(1)
    keep = ~tie
    assert int(keep.sum()) > M // 2
    dy = torch.randn(M, 1, device=DEV, generator=g) * keep.unsqueeze(1)
    out.backward(dy)
    grads = torch.autograd.grad(ref, p64 + [us[0]], dy.double())
    du0 = grads[-1]
    # gate outputs are negative somewhere and feed the width-1 top layer: their gradient is not
    # masked away (a ReLU mask on z would zero it)
    z_last = zs[-1].detach()
    assert bool((z_last[keep] < 0).any())
    dz = dy.double() @ p64[3].detach().t()
    assert bool((dz[keep][z_last[keep] < 0] != 0).all())
    tol = gated_tol(len(Gs))
    assert elementwise_excess(out[keep], ref[keep], tol, tol) <= 0
    # dx0 = du0 @ W0^T sums K-wide rows of mixed sign: held to tol of the summed magnitude
    mag = du0.abs() @ p64[1].detach().abs().t()
    err = (xg.grad.double() - grads[0])[keep].abs()
    assert bool((err <= tol * mag[keep] + tol * float(grads[0][keep].square().mean().sqrt())).all())
    names = ["W0", "W1", "W2", "b0", "b1", "b2", "G0", "G1"]
    for name, got, want in zip(names, [t.grad for t in Ws + bs + Gs], grads[1:]):
        assert elementwise_excess(got, want, tol, tol) <= 0, name


# ---- the model against the goldens -------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
@pytest.mark.parametrize("name", ["gatenet_init", "gatenet_scaled", "gatenet_embed", "gatenet_hidden"])
def test_gatenet_layer_matches_golden(name, precision):
    from paddlerec_b200 import functional as BF
    from paddlerec_b200 import nn as bnn
    from paddlerec_b200.rank.gatenet import net
    gold = load_golden(name)
    n_fc, eg, hg = gatenet_oracle.flags(gold["param"])
    fc = [gold["param"]["linear_%d.weight" % i].shape[1] for i in range(n_fc)]
    V = gold["param"]["embedding.weight"].shape[0]
    layer = net.GateDNNLayer(V, 9, 13, 26, fc, eg, hg, device=DEV)
    layer.load_state_dict({k: torch.tensor(v, dtype=torch.float32) for k, v in gold["param"].items()})
    ids = torch.tensor(gold["in"]["ids"], device=DEV)
    dense = torch.tensor(gold["in"]["dense"], dtype=torch.float32, device=DEV)
    label = torch.tensor(gold["in"]["label"], dtype=torch.float32, device=DEV)
    prev = bnn.get_matmul_precision()
    bnn.set_matmul_precision(precision)
    try:
        logit = layer.logit(ids, dense)
        pred = torch.sigmoid(logit) if precision == "fp32" else layer(ids, dense)
        BF.log_loss_mean(pred, label).backward()
    finally:
        bnn.set_matmul_precision(prev)
    # logits relative to their own scale: ~1e-10 at the reference's init survives the bf16 planes
    tol = gated_tol(n_fc if hg else 0) if precision == "bf16x3" else 1e-4
    assert rel_err(logit, gold["out"]["logit"]) <= tol
    named = dict(layer.named_parameters())
    for k, want in gold["grad"].items():
        if k.startswith("embedding_gate_weight_"):
            continue
        got = layer.embedding.grad_rows.to_dense() if k == "embedding.weight" else named[k].grad
        assert rel_err(got, want) <= tol, k
    if eg:     # the 26 [1] gate weights are one [F] vector on the device: compared as one tensor
        got = torch.cat([named["embedding_gate_weight_%d" % f].grad for f in range(26)])
        want = np.concatenate([gold["grad"]["embedding_gate_weight_%d" % f] for f in range(26)])
        assert rel_err(got, want) <= tol


# ---- one B = 65536 step -----------------------------------------------------------------------
def test_gatenet_full_size_step_on_a_slice_vs_oracle():
    from paddlerec_b200 import functional as BF
    from paddlerec_b200 import nn as bnn
    from paddlerec_b200 import optim
    from paddlerec_b200.rank.gatenet import net
    B, V, D, F, Dn = 65536, 1_000_000, 9, 26, 13
    fc = [512, 256, 128, 32]
    torch.manual_seed(2)
    layer = net.GateDNNLayer(V, D, Dn, F, fc, True, True, device=DEV)
    with torch.no_grad():      # the reference's init makes the logit vanish (SURVEY Q18)
        for G, s in zip(layer._hidden_gate_weight, (5.0, 20.0, 100.0, 100.0)):
            G.mul_(s)
    g = torch.Generator(device=DEV).manual_seed(9)
    ids = torch.randint(0, V, (B, F), device=DEV, generator=g)
    dense = torch.rand(B, Dn, device=DEV, generator=g)
    label = (torch.rand(B, 1, device=DEV, generator=g) < 0.3).float()
    opt = optim.Adam(learning_rate=1e-3, parameters=layer.parameters(), lazy_mode=True)
    prev = bnn.get_matmul_precision()
    bnn.set_matmul_precision("bf16x3")
    try:
        logit = layer.logit(ids, dense)
        BF.log_loss_mean(torch.sigmoid(logit), label).backward()
    finally:
        bnn.set_matmul_precision(prev)
    s = slice(0, NS)
    uniq = torch.unique(ids[s])
    remap = torch.searchsorted(uniq, ids[s])
    p = {k: v.detach().double() for k, v in layer.state_dict().items() if k != "embedding.weight"}
    p["embedding.weight"] = layer.embedding.weight.detach()[uniq].double()
    ref = gatenet_oracle.gatenet_logit(p, [remap[:, i:i + 1] for i in range(F)], dense[s].double(),
                                       len(fc), True, True)
    assert rel_err(logit[s], ref) <= gated_tol(len(fc))
    for k in ["embedding_gate_weight_0", "linear_0.weight", "hidden_gate_weight_0",
              "hidden_gate_weight_3", "last_layer.weight"]:
        assert torch.isfinite(dict(layer.named_parameters())[k].grad).all(), k
    assert layer.embedding.grad_rows.count() > 100_000
    opt.step()
    torch.cuda.synchronize()


# ---- trainer and infer on config.yaml -----------------------------------------------------------
def test_gatenet_trainer_and_infer_on_config(tmp_path):
    from paddlerec_b200 import runner
    d = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "paddlerec_b200",
                     "rank", "gatenet")
    cfg = runner.load_yaml(os.path.join(d, "config.yaml"))
    cfg["config_abs_dir"] = d
    cfg["runner.model_save_path"] = str(tmp_path / "out")
    cfg["runner.infer_load_path"] = str(tmp_path / "out")
    losses, metrics, _ = runner.train(cfg)
    assert len(losses) > 0 and np.all(np.isfinite(losses)) and "auc" in metrics
    results = runner.infer(cfg)
    assert sorted(results) == [2] and all(0.0 <= r["auc"] <= 1.0 for r in results.values())
