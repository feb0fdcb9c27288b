"""GateNet on the CPU: the oracle against the goldens minted from the reference's gatenet/net.py, the
reference's checkpoint names, the vanishing signal its hidden gates cause at initialisation (SURVEY
Q18), and the train -> infer -> checkpoint loop of the gatenet model directory (with torch stand-ins
for the two embedding-gate kernels, installed next to tests/cpu_kernels.py's)."""
import math
import os

import numpy as np
import pytest
import torch

from tests import cpu_kernels, gatenet_oracle
from tests.util import load_golden, slots, to_params

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "paddlerec_b200")
F, Dn, D = 26, 13, 9
GOLDENS = ["gatenet_init", "gatenet_scaled", "gatenet_embed", "gatenet_hidden"]


def _oracle(g, dtype=torch.float64):
    p = to_params(g["param"], dtype)
    logit = gatenet_oracle.gatenet_logit(p, slots(g["in"]["ids"]), torch.tensor(g["in"]["dense"], dtype=dtype),
                                         *gatenet_oracle.flags(p))
    return p, logit


# ---- oracle vs goldens -----------------------------------------------------------------------------
@pytest.mark.parametrize("name", GOLDENS)
def test_oracle_matches_gatenet_golden(name):
    from oracle import nets
    g = load_golden(name)
    p, logit = _oracle(g)
    pred = torch.sigmoid(logit)
    loss = nets.log_loss(pred, torch.tensor(g["in"]["label"], dtype=torch.float64)).mean()
    grads = dict(zip(p, torch.autograd.grad(loss, list(p.values()))))
    # the logit is compared relative to its own scale: at the reference's init it is ~1e-10
    scale = float(np.abs(g["out"]["logit"]).max())
    np.testing.assert_allclose(logit.detach().numpy(), g["out"]["logit"], rtol=0, atol=1e-12 * scale)
    np.testing.assert_allclose(pred.detach().numpy(), g["out"]["pred"], rtol=0, atol=1e-12)
    np.testing.assert_allclose(loss.detach().numpy(), g["out"]["loss"], rtol=0, atol=1e-12)
    assert set(grads) == set(g["grad"])
    for k, v in grads.items():
        ref = g["grad"][k]
        np.testing.assert_allclose(v.numpy(), ref, rtol=0, atol=1e-12 * max(np.abs(ref).max(), 1e-300),
                                   err_msg=k)


def test_gatenet_goldens_cover_the_cases():
    init, scaled = load_golden("gatenet_init"), load_golden("gatenet_scaled")
    embed, hidden = load_golden("gatenet_embed"), load_golden("gatenet_hidden")
    assert gatenet_oracle.flags(init["param"])[1:] == (True, True)
    assert gatenet_oracle.flags(embed["param"])[1:] == (True, False)
    assert gatenet_oracle.flags(hidden["param"])[1:] == (False, True)
    ids = init["in"]["ids"]
    assert (ids == 0).any() and ids[2, 5] == ids[2, 4] and len(set(ids[3:, 0])) == 1
    # no padding_idx: id 0 is a real row and receives gradient
    assert init["grad"]["embedding.weight"][0].any()
    # the embedding-gate weights take both signs, and their gradients are nonzero
    w = np.concatenate([scaled["param"]["embedding_gate_weight_%d" % f] for f in range(F)])
    assert (w > 0).any() and (w < 0).any()
    assert all(np.abs(scaled["grad"]["embedding_gate_weight_%d" % f]).max() > 0 for f in range(F))
    # scaled hidden gates give an O(0.01..1) logit, the reference's init a vanishing one
    assert 1e-2 < np.sqrt(np.mean(scaled["out"]["logit"] ** 2)) < 10
    assert np.abs(init["out"]["logit"]).max() < 1e-8


def test_state_dict_names_and_shapes_match_the_reference():
    from paddlerec_b200.rank.gatenet import net
    for name in GOLDENS:
        g = load_golden(name)
        n_fc, eg, hg = gatenet_oracle.flags(g["param"])
        fc = [g["param"]["linear_%d.weight" % i].shape[1] for i in range(n_fc)]
        layer = net.GateDNNLayer(53, D, Dn, F, fc, eg, hg, device="cpu")
        got = {k: tuple(v.shape) for k, v in layer.state_dict().items()}
        assert got == {k: tuple(v.shape) for k, v in g["param"].items()}, name


def test_reference_initialisation_makes_the_signal_vanish():
    """SURVEY Q18: y = relu(.) >= 0 is small, so y * tanh(y @ G) ~ y^2 @ G and every gated layer
    squares the scale down.  At config.yaml's shape (V 1000001 -> a small V here; D 9, fc
    [512, 256, 128, 32]) in fp64 the logit is ~1e-12 with both gates, ~1e-9 with the hidden gates
    only, ~0.1 with the embedding gate only; in fp32 the prediction is exactly 0.5."""
    from paddlerec_b200.rank.gatenet import net
    fc = [512, 256, 128, 32]
    g = torch.Generator().manual_seed(3)
    ids = torch.randint(0, 1000, (256, F), generator=g)
    dense = torch.rand(256, Dn, generator=g, dtype=torch.float64)
    rms = {}
    for eg, hg in [(True, True), (False, True), (True, False)]:
        torch.manual_seed(11)
        layer = net.GateDNNLayer(1000, D, Dn, F, fc, eg, hg, device="cpu")
        p = {k: v.detach().double().requires_grad_(True) for k, v in layer.state_dict().items()}
        logit = gatenet_oracle.gatenet_logit(p, slots(ids), dense, len(fc), eg, hg)
        rms[(eg, hg)] = float(logit.detach().square().mean().sqrt())
        if eg and hg:
            # every gradient but the last bias's passes through the vanished signal
            inner = [v for k, v in p.items() if k != "last_layer.bias"]
            gs = torch.autograd.grad(torch.sigmoid(logit).mean(), inner)
            assert max(float(x.abs().max()) for x in gs) < 1e-6
            pred32 = torch.sigmoid(gatenet_oracle.gatenet_logit(
                {k: v.detach().float() for k, v in p.items()}, slots(ids), dense.float(), len(fc), eg, hg))
            assert bool((pred32 == 0.5).all())
    assert 1e-14 < rms[(True, True)] < 1e-10
    assert 1e-11 < rms[(False, True)] < 1e-7
    assert 1e-2 < rms[(True, False)] < 1.0


# ---- torch stand-ins for the two embedding-gate kernels (TEST DOUBLES, host-logic tests only) ----
def _gated_rows(W, ids, gate_w, D):
    V = W.shape[0]
    ok = ((ids >= 0) & (ids < V)).unsqueeze(2).to(W.dtype)
    e = W[ids.clamp(0, V - 1), :D] * ok
    g = torch.sigmoid((e * gate_w.reshape(1, -1, 1)).sum(2, keepdim=True))
    return e, g


def raw_gate_embed_fwd(W, ids, gate_w, dense, D=None):
    D = W.shape[1] if D is None else D
    e, g = _gated_rows(W, ids, gate_w.detach().reshape(-1), D)
    out = (e * g).reshape(ids.shape[0], -1)
    return torch.cat([out, dense], 1) if dense is not None else out


def raw_gate_embed_bwd(W, ids, gate_w, dout, D=None):
    D = W.shape[1] if D is None else D
    B, F_ = ids.shape
    with torch.enable_grad():
        e = W[ids.clamp(0, W.shape[0] - 1), :D].detach().requires_grad_(True)
        ok = ((ids >= 0) & (ids < W.shape[0])).unsqueeze(2).to(W.dtype)
        w = gate_w.detach().reshape(-1).clone().requires_grad_(True)
        x = e * ok
        out = (x * torch.sigmoid((x * w.reshape(1, -1, 1)).sum(2, keepdim=True))).reshape(B, -1)
        de, dw = torch.autograd.grad((out * dout[:, :F_ * D]).sum(), [e, w])
    return (de * ok).reshape(B * F_, D), dw


@pytest.fixture
def cpu_engine(monkeypatch):
    from paddlerec_b200 import ops, runner
    from paddlerec_b200.rank.deepfm import dygraph_model as criteo_base

    cpu_kernels.install(monkeypatch, ops)
    monkeypatch.setattr(ops, "raw_gate_embed_fwd", raw_gate_embed_fwd)
    monkeypatch.setattr(ops, "raw_gate_embed_bwd", raw_gate_embed_bwd)
    monkeypatch.setattr(runner, "_require_cuda", lambda: None)
    monkeypatch.setattr(criteo_base.DygraphModel, "device", "cpu")
    return runner


def test_stand_ins_match_the_golden_gradients(cpu_engine):
    """The stand-ins (through ops.gate_embed and the fp32 op sequence of net.GateDNNLayer) are checked
    against the reference's gradients before the loop test relies on them."""
    from oracle import nets
    from paddlerec_b200.rank.gatenet import net
    g = load_golden("gatenet_scaled")
    n_fc, eg, hg = gatenet_oracle.flags(g["param"])
    fc = [g["param"]["linear_%d.weight" % i].shape[1] for i in range(n_fc)]
    layer = net.GateDNNLayer(53, D, Dn, F, fc, eg, hg, device="cpu")
    layer.load_state_dict({k: torch.tensor(v, dtype=torch.float32) for k, v in g["param"].items()})
    ids, dense = torch.tensor(g["in"]["ids"]), torch.tensor(g["in"]["dense"], dtype=torch.float32)
    logit = layer.logit(ids, dense)
    loss = nets.log_loss(torch.sigmoid(logit), torch.tensor(g["in"]["label"], dtype=torch.float32)).mean()
    loss.backward()
    ref = g["out"]["logit"]
    assert np.abs(logit.detach().numpy() - ref).max() <= 1e-4 * np.abs(ref).max()
    named = dict(layer.named_parameters())
    for k in ["embedding_gate_weight_0", "embedding_gate_weight_25", "linear_0.weight",
              "hidden_gate_weight_0", "hidden_gate_weight_%d" % (n_fc - 1), "last_layer.bias"]:
        got, want = named[k].grad.numpy(), g["grad"][k]
        assert np.abs(got - want).max() <= 1e-4 * np.abs(want).max(), k
    dW = layer.embedding.grad_rows.to_dense().numpy()
    want = g["grad"]["embedding.weight"]
    assert np.abs(dW - want).max() <= 1e-4 * np.abs(want).max()


def _config(runner, tmp_path, **over):
    d = os.path.join(PKG, "rank", "gatenet")
    cfg = runner.load_yaml(os.path.join(d, "config.yaml"))
    cfg["config_abs_dir"] = d
    cfg["runner.model_save_path"] = str(tmp_path / "out")
    cfg["runner.infer_load_path"] = str(tmp_path / "out")
    cfg.update(over)
    return cfg


def test_gatenet_train_infer_checkpoint_round_trip(cpu_engine, tmp_path):
    runner = cpu_engine
    V = 2003
    cfg = _config(runner, tmp_path, **{"runner.train_batch_size": 16, "runner.infer_batch_size": 16,
                                       "runner.epochs": 2, "runner.infer_start_epoch": 0,
                                       "runner.infer_end_epoch": 2,
                                       "hyper_parameters.sparse_feature_number": V,
                                       "runner.reader_type": "PackedReader"})
    losses, metric_values, net = runner.train(cfg)
    assert len(losses) == 10 and np.all(np.isfinite(losses)) and "auc" in metric_values
    for e in range(2):
        assert sorted(os.listdir(tmp_path / "out" / str(e))) == ["rec.pdopt", "rec.pdparams"]
    results = runner.infer(cfg)
    assert sorted(results) == [0, 1] and all(0.0 <= r["auc"] <= 1.0 for r in results.values())

    from paddlerec_b200 import checkpoint
    saved = checkpoint.load_pdparams(str(tmp_path / "out" / "1" / "rec.pdparams"))
    fc = [512, 256, 128, 32]
    sizes = [F * D + Dn] + fc
    want = {"embedding.weight": (V, D), "last_layer.weight": (fc[-1], 1), "last_layer.bias": (1,)}
    want.update({"embedding_gate_weight_%d" % f: (1,) for f in range(F)})
    for i in range(len(fc)):
        want["linear_%d.weight" % i] = (sizes[i], sizes[i + 1])
        want["linear_%d.bias" % i] = (sizes[i + 1],)
        want["hidden_gate_weight_%d" % i] = (sizes[i + 1], sizes[i + 1])
    assert {k: tuple(v.shape) for k, v in saved.items()} == want
    for k, v in net.state_dict().items():
        assert np.array_equal(saved[k], v.numpy()), k
    # the vanishing quirk, reproduced: the embedding-gate weights barely move in two epochs
    assert math.isfinite(float(saved["embedding_gate_weight_0"][0]))
