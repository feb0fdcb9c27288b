"""ESMM on the CPU: the oracle against the goldens minted from the reference's esmm/net.py, the
restated reader against the reference reader's output, the reference's checkpoint names, and the
train -> infer -> checkpoint loop of the multitask/esmm model directory.  Torch stand-ins for the
two head kernels are defined here; the pooled lookup runs on tests/cpu_kernels.py's stand-in."""
import os

import numpy as np
import pytest
import torch

from tests import cpu_kernels, esmm_oracle
from tests.util import GOLDEN_DIR, load_golden, to_params

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "paddlerec_b200")
GOLDENS = ["esmm_init", "esmm_saturated"]
OUTS = ("ctr_out", "ctr_one", "cvr_out", "cvr_one", "ctcvr_prop", "ctcvr_one")
V, D, F, L = 61, 12, 23, 3


def _inputs(g):
    ids = torch.as_tensor(g["in"]["ids"])
    return [ids[:, f, :] for f in range(ids.shape[1])]


def _fc(params):
    n_ctr, n_cvr = esmm_oracle.tower_sizes(params)
    ctr = [params["linear_%d.weight" % i].shape[1] for i in range(n_ctr - 1)]
    cvr = [params["linear_%d.weight" % (n_ctr + i)].shape[1] for i in range(n_cvr - 1)]
    return ctr, cvr


# ---- oracle vs goldens -----------------------------------------------------------------------------
@pytest.mark.parametrize("name", GOLDENS)
def test_oracle_matches_esmm_golden(name):
    g = load_golden(name)
    p = to_params(g["param"])
    n_ctr, n_cvr = esmm_oracle.tower_sizes(p)
    inputs = _inputs(g)
    z_ctr, z_cvr = esmm_oracle.esmm_logits(p, inputs, n_ctr, n_cvr)
    outs = esmm_oracle.esmm_forward(p, inputs, n_ctr, n_cvr)
    loss = esmm_oracle.esmm_loss(outs[1], torch.as_tensor(g["in"]["clk"]), outs[5],
                                 torch.as_tensor(g["in"]["buy"]))
    grads = dict(zip(p, torch.autograd.grad(loss, list(p.values()))))
    for k, v in (("z_ctr", z_ctr), ("z_cvr", z_cvr)):
        ref = g["out"][k]
        np.testing.assert_allclose(v.detach().numpy(), ref, rtol=0, atol=1e-12 * np.abs(ref).max())
    for k, v in zip(OUTS, outs):
        np.testing.assert_allclose(v.detach().numpy(), g["out"][k], rtol=0, atol=1e-12, err_msg=k)
    np.testing.assert_allclose(loss.detach().numpy(), g["out"]["loss"], rtol=0, atol=1e-12)
    assert set(grads) == set(g["grad"])
    for k, v in grads.items():
        ref = g["grad"][k]
        np.testing.assert_allclose(v.numpy(), ref, rtol=0, atol=1e-12 * max(np.abs(ref).max(), 1e-300),
                                   err_msg=k)


def test_esmm_goldens_cover_the_cases():
    for name in GOLDENS:
        g = load_golden(name)
        ids, clk, buy = g["in"]["ids"], g["in"]["clk"], g["in"]["buy"]
        assert ids.shape[1:] == (F, L)
        assert (ids[1] == 0).all()                                   # every bag of a sample padding
        assert (ids[0, 7] == 0).all()                                # one all-padding bag
        assert ids[0, 2, 0] == ids[0, 2, 1] != 0                     # the same id twice in one bag
        shared = ids[3, 0, 0]
        assert (ids[3:, 0, 0] == shared).all() and ids[4, 5, 1] == shared
        assert (buy <= clk).all() and buy.any() and (clk - buy).any()
        # the padding row takes no gradient; the CVR tower's last layer does (through the product)
        assert not g["grad"]["embedding.weight"][0].any()
        assert np.abs(g["grad"]["linear_5.weight"]).max() > 0
    sat = load_golden("esmm_saturated")
    for k in ("z_ctr", "z_cvr"):
        gap = sat["out"][k][:, 1] - sat["out"][k][:, 0]
        assert gap.max() > 20 and gap.min() < -20
    # the small class keeps its relative accuracy: far below fp32's epsilon, still nonzero
    assert 0 < sat["out"]["ctr_out"].min() < 1e-8 and 0 < sat["out"]["cvr_out"].min() < 1e-8


# ---- the reader -----------------------------------------------------------------------------------
def test_reader_matches_the_reference_reader():
    from paddlerec_b200.multitask.esmm import esmm_reader
    ref = np.load(os.path.join(GOLDEN_DIR, "esmm_reader_batches.npz"))
    for split in ("train", "test"):
        path = os.path.join(GOLDEN_DIR, "esmm_sample", split, "small.txt")
        samples = list(esmm_reader.RecDataset([path], {"hyper_parameters.max_len": 3}))
        assert len(samples) == 10
        ids = np.stack([np.stack(s[:F]) for s in samples])
        assert ids.dtype == np.int64 and np.array_equal(ids, ref[split + "/ids"])
        assert np.array_equal(np.stack([s[F] for s in samples]), ref[split + "/clk"])
        assert np.array_equal(np.stack([s[F + 1] for s in samples]), ref[split + "/buy"])
    # the two files differ, and truncation and padding both occur in the sample
    assert not np.array_equal(ref["train/clk"], ref["test/clk"])
    assert (ref["train/ids"] == 0).any() and (ref["train/ids"] != 0).all(axis=2).any()


def test_reader_skips_the_fourth_column_and_unknown_fields():
    from paddlerec_b200.multitask.esmm import esmm_reader
    s = esmm_reader.parse_line("7,1,0,101:9,101:1,999:5,101:2,101:3,101:4,301:8\n", 3)
    assert s[0].tolist() == [1, 2, 3] and s[22].tolist() == [8, 0, 0]
    assert all(not x.any() for x in s[1:22])
    assert s[23].tolist() == [1] and s[24].tolist() == [0]


# ---- checkpoint names ------------------------------------------------------------------------------
def test_state_dict_names_and_shapes_match_the_reference():
    from paddlerec_b200.multitask.esmm import net
    for name in GOLDENS:
        g = load_golden(name)
        ctr, cvr = _fc(g["param"])
        layer = net.ESMMLayer(V, D, F, ctr, cvr, device="cpu")
        got = {k: tuple(v.shape) for k, v in layer.state_dict().items()}
        assert got == {k: tuple(v.shape) for k, v in g["param"].items()}, name
        assert list(layer.state_dict()) == list(g["param"])
        assert not layer.embedding.weight[0].any()                  # padding row zeroed at init


# ---- torch stand-ins for the two head kernels (TEST DOUBLES, host-logic tests only) --------------
def raw_esmm_head_fwd(h_ctr, h_cvr, W_ctr, b_ctr, W_cvr, b_cvr):
    from paddlerec_b200.multitask.esmm import net
    with torch.no_grad():
        return tuple(o.contiguous() for o in net.torch_head(h_ctr, h_cvr, W_ctr, b_ctr, W_cvr, b_cvr))


def raw_esmm_head_bwd(grads, p_ctr, p_cvr, h_ctr, h_cvr, W_ctr, W_cvr):
    """The kernel's formulas, restated: fold the CTCVR gradient into the two towers' class-1
    gradients, then the softmax backward s = p0 p1 (G1 - G0) per tower."""
    z = torch.zeros(h_ctr.shape[0], 2)
    g = [z if t is None else t.reshape(-1, 2) if t.shape[-1] == 2 else
         torch.cat([torch.zeros_like(t), t], 1) for t in grads]
    Gc = g[4][:, 1] - g[4][:, 0] + g[5][:, 1]
    G_ctr = g[0] + g[1]
    G_cvr = g[2] + g[3]
    G_ctr[:, 1] += Gc * p_cvr[:, 1]
    G_cvr[:, 1] += Gc * p_ctr[:, 1]
    out = []
    for p, G, h, W in ((p_ctr, G_ctr, h_ctr, W_ctr), (p_cvr, G_cvr, h_cvr, W_cvr)):
        s = p[:, 0] * p[:, 1] * (G[:, 1] - G[:, 0])
        dz = torch.stack([-s, s], 1)
        out.append((dz @ W.detach().t(), h.t() @ dz, dz.sum(0)))
    (dh_c, dW_c, db_c), (dh_v, dW_v, db_v) = out
    return dh_c, dh_v, dW_c, db_c, dW_v, db_v


@pytest.fixture
def cpu_engine(monkeypatch):
    from paddlerec_b200 import ops, runner
    from paddlerec_b200.multitask.esmm import dygraph_model

    cpu_kernels.install(monkeypatch, ops)
    monkeypatch.setattr(ops, "raw_esmm_head_fwd", raw_esmm_head_fwd)
    monkeypatch.setattr(ops, "raw_esmm_head_bwd", raw_esmm_head_bwd)
    monkeypatch.setattr(runner, "_require_cuda", lambda: None)
    monkeypatch.setattr(dygraph_model.DygraphModel, "device", "cpu")
    return runner


def _model_from_golden(g):
    from paddlerec_b200.multitask.esmm import net
    ctr, cvr = _fc(g["param"])
    layer = net.ESMMLayer(V, D, F, ctr, cvr, device="cpu")
    layer.load_state_dict({k: torch.tensor(v, dtype=torch.float32) for k, v in g["param"].items()})
    return layer


@pytest.mark.parametrize("name", GOLDENS)
def test_model_and_head_node_match_the_golden(cpu_engine, name):
    """The model's CPU path (the pooled-lookup stand-in and the reference's torch head) against the
    golden, then ops.esmm_head on the stand-ins: the autograd node's gradient plumbing, with the
    gradient of each output alone (the others reach the backward as None) and all together."""
    from paddlerec_b200 import ops
    from paddlerec_b200.multitask.esmm import dygraph_model
    g = load_golden(name)
    layer = _model_from_golden(g)
    dm = dygraph_model.DygraphModel()
    cfg = {"hyper_parameters.max_len": L}
    ids, clk, buy = dm.create_feeds([torch.as_tensor(g["in"]["ids"]), torch.as_tensor(g["in"]["clk"]),
                                     torch.as_tensor(g["in"]["buy"])], cfg)
    outs = layer(ids)
    loss = dm.create_loss(outs[1], clk, outs[5], buy)
    loss.backward()
    for k, o in zip(OUTS, outs):
        assert np.abs(o.detach().numpy() - g["out"][k]).max() <= 1e-5, k
    assert abs(float(loss.detach()) - float(g["out"]["loss"])) <= 1e-4 * abs(float(g["out"]["loss"]))
    named = dict(layer.named_parameters())
    checked = ["linear_0.weight", "linear_2.weight", "linear_2.bias"]
    if name == "esmm_init":
        # saturated, torch's fp32 softmax backward p * (G - sum(p G)) cancels in the large class and
        # loses the CVR tower's tiny gradients; the fused kernel's p0 p1 (G1 - G0) does not (GPU test)
        checked += ["linear_3.weight", "linear_5.bias"]
    for k in checked:
        got, want = named[k].grad.numpy(), g["grad"][k]
        assert np.abs(got - want).max() <= 1e-4 * np.abs(want).max(), k
    dW = layer.embedding.grad_rows.to_dense().numpy()
    want = g["grad"]["embedding.weight"]
    assert np.abs(dW - want).max() <= 1e-4 * np.abs(want).max()

    # the autograd node against torch autograd through the reference's head
    gen = torch.Generator().manual_seed(5)
    h = [torch.rand(7, 16, generator=gen) for _ in range(2)]
    Wb = [torch.randn(16, 2, generator=gen), torch.randn(2, generator=gen),
          torch.randn(16, 2, generator=gen), torch.randn(2, generator=gen)]
    weights = [torch.randn(7, 2 if i % 2 == 0 else 1, generator=gen) for i in range(6)]
    from paddlerec_b200.multitask.esmm import net
    for pick in [[i] for i in range(6)] + [list(range(6))]:
        leaves = [t.clone().requires_grad_(True) for t in h + Wb]
        got = ops.esmm_head(*leaves[:2], *leaves[2:])
        sum(((got[i] * weights[i]).sum() for i in pick), torch.zeros(())).backward()
        ref_leaves = [t.clone().double().requires_grad_(True) for t in h + Wb]
        ref = net.torch_head(*ref_leaves[:2], *ref_leaves[2:])
        sum(((ref[i] * weights[i].double()).sum() for i in pick), torch.zeros((), dtype=torch.float64)).backward()
        for a, b in zip(leaves, ref_leaves):
            want = torch.zeros_like(b) if b.grad is None else b.grad     # untouched tower: zeros
            assert torch.allclose(a.grad.double(), want, rtol=1e-5, atol=1e-6), pick


def _config(runner, tmp_path, **over):
    d = os.path.join(PKG, "multitask", "esmm")
    cfg = runner.load_yaml(os.path.join(d, "config.yaml"))
    cfg["config_abs_dir"] = d
    cfg["runner.model_save_path"] = str(tmp_path / "out")
    cfg["runner.infer_load_path"] = str(tmp_path / "out")
    cfg.update(over)
    return cfg


def test_esmm_train_infer_checkpoint_round_trip(cpu_engine, tmp_path):
    runner = cpu_engine
    Vs = 1009
    cfg = _config(runner, tmp_path, **{"hyper_parameters.sparse_feature_number": Vs})
    losses, metric_values, net_ = runner.train(cfg)
    assert len(losses) == 15 and np.all(np.isfinite(losses))
    assert sorted(metric_values) == ["auc_ctcvr", "auc_ctr"]
    assert all(0.0 <= v <= 1.0 for v in metric_values.values())
    for e in range(3):
        assert sorted(os.listdir(tmp_path / "out" / str(e))) == ["rec.pdopt", "rec.pdparams"]
    results = runner.infer(cfg)
    assert sorted(results) == [0, 1, 2]
    assert all(sorted(r) == ["auc_ctcvr", "auc_ctr"] and all(0.0 <= v <= 1.0 for v in r.values())
               for r in results.values())

    from paddlerec_b200 import checkpoint
    saved = checkpoint.load_pdparams(str(tmp_path / "out" / "2" / "rec.pdparams"))
    sizes = [F * D, 256, 64, 2]
    want = {"embedding.weight": (Vs, D)}
    for t in range(2):
        for i in range(3):
            want["linear_%d.weight" % (3 * t + i)] = (sizes[i], sizes[i + 1])
            want["linear_%d.bias" % (3 * t + i)] = (sizes[i + 1],)
    assert {k: tuple(v.shape) for k, v in saved.items()} == want
    for k, v in net_.state_dict().items():
        assert np.array_equal(saved[k], v.numpy()), k
    # lazy Adam never touches the padding row
    assert not saved["embedding.weight"][0].any()
