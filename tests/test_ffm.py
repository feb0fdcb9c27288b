"""FFM on the CPU: the oracle against the goldens minted from the reference's ffm/net.py, the
train -> infer -> checkpoint loop of the ffm model directory (with torch stand-ins for the two FFM
kernels, installed next to tests/cpu_kernels.py's), the reference's checkpoint names, and the
saturation the reference's constant dense initialisers cause on the sample data."""
import os

import numpy as np
import pytest
import torch

from tests import cpu_kernels, ffm_oracle
from tests.util import load_golden, slots, to_params

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "paddlerec_b200")
F, Dn = 26, 13


# ---- oracle vs goldens -----------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["ffm_d9", "ffm_d16"])
def test_oracle_matches_ffm_golden(name):
    from oracle import nets
    g = load_golden(name)
    p = to_params(g["param"])
    i = g["in"]
    pred = ffm_oracle.ffm_forward(p, slots(i["ids"]), torch.tensor(i["dense"]), F + Dn)
    loss = nets.log_loss(pred, torch.tensor(i["label"], dtype=torch.float64)).mean()
    grads = dict(zip(p, torch.autograd.grad(loss, list(p.values()))))
    np.testing.assert_allclose(pred.detach().numpy(), g["out"]["pred"], rtol=0, atol=1e-12)
    np.testing.assert_allclose(loss.detach().numpy(), g["out"]["loss"], rtol=0, atol=1e-12)
    assert set(grads) == set(g["grad"])
    for k, v in grads.items():
        np.testing.assert_allclose(v.numpy(), g["grad"][k], rtol=0, atol=1e-12, err_msg=k)


def test_ffm_golden_covers_edge_cases():
    g = load_golden("ffm_d9")
    ids = g["in"]["ids"]
    assert (ids == 0).any() and ids[2, 5] == ids[2, 4] and len(set(ids[3:, 0])) == 1
    # no padding_idx: id 0 is a real row and receives gradient
    assert g["grad"]["ffm.embedding.weight"][0].any() and g["grad"]["ffm.embedding_one.weight"][0].any()
    # the dense parameters were overridden, so the prediction is not saturated and they learn
    assert 0.01 < g["out"]["pred"].min() and g["out"]["pred"].max() < 0.99
    assert np.abs(g["grad"]["ffm.dense_w"]).max() > 0 and np.abs(g["grad"]["bias"]).max() > 0


def test_reference_initialisation_saturates_on_the_sample_data(tmp_path):
    """SURVEY.md Appendix C: with dense_w_one = dense_w = 1 the dense-only logit is
    sum_k x_k + D * sum_{k<k'} x_k x_k'; on the reference's 80 sample rows (ffm/data/sample_data,
    the same file as deepfm's) it runs from 0.02 to 278 and a third of the rows exceed 17, where
    fp32 sigmoid is exactly 1.0."""
    import gzip

    from paddlerec_b200.rank.deepfm.criteo_reader import RecDataset
    path = tmp_path / "sample_train.txt"
    with gzip.open(os.path.join(os.path.dirname(__file__), "golden", "ref_deepfm_sample_train.txt.gz"),
                   "rt") as fh:
        path.write_text(fh.read())
    x = torch.tensor(np.stack([s[-1] for s in RecDataset([str(path)])]), dtype=torch.float64)
    assert x.shape == (80, Dn)
    D = 9
    logit = x.sum(1) + D * (x.sum(1).square() - x.square().sum(1)) / 2
    assert 0.01 < float(logit.min()) < 0.03 and 277 < float(logit.max()) < 279
    sat = float((logit > 17).double().mean())
    assert 0.3 < sat < 0.4
    assert bool((torch.sigmoid(logit[logit > 17].float()) == 1.0).all())


# ---- torch stand-ins for the two FFM kernels (TEST DOUBLES, host-logic tests only) ------------------
def _ffm_terms(rows, ids, dense, dense_w, dense_w1, bias, D):
    B = ids.shape[0]
    NF = F + dense.shape[1]
    R = NF * D
    e = torch.cat([rows[:, :, :R], dense.unsqueeze(2) * dense_w.reshape(1, -1, R)], 1)
    e = e.reshape(B, NF, NF, D)
    iu = torch.triu_indices(NF, NF, 1)
    y2 = (e[:, iu[0], iu[1]] * e[:, iu[1], iu[0]]).sum((1, 2))
    y1 = rows[:, :, R].sum(1) + (dense * dense_w1.reshape(1, -1)).sum(1)
    if bias is not None:
        y1 = y1 + bias.reshape(())
    return y1, y2


def _rows(W, ids, pad):
    V = W.shape[0]
    ok = (ids >= 0) & (ids < V) & (ids != pad)
    return W[ids.clamp(0, V - 1)], ok.unsqueeze(2).to(W.dtype)


def raw_ffm_fwd(W, ids, dense, dense_w, dense_w1, bias, pad, D):
    raw, ok = _rows(W, ids, pad)
    return _ffm_terms(raw * ok, ids, dense, dense_w, dense_w1, bias, D)


def raw_ffm_bwd(W, ids, dense, dense_w, gy1, gy2, groups, pad, D):
    from paddlerec_b200 import ops
    raw, ok = _rows(W, ids, pad)
    with torch.enable_grad():
        leaf = raw.detach().requires_grad_(True)
        dw = dense_w.detach().clone().requires_grad_(True)
        dw1 = torch.zeros(dense.shape[1], requires_grad=True)    # y1 is linear in dense_w1
        b = torch.zeros(1, requires_grad=True)
        y1, y2 = _ffm_terms(leaf * ok, ids, dense, dw, dw1, b, D)
        gr, gdw, gdw1, gb = torch.autograd.grad((y1 * gy1 + y2 * gy2).sum(), [leaf, dw, dw1, b])
    G = ops.fused_grad_cols((F + dense.shape[1]) * D)
    flat = gr.reshape(-1, W.shape[1])[:, :G].contiguous()
    rows = cpu_kernels.raw_segment_reduce(flat, groups.seg_offsets, groups.sorted_pos, groups.num,
                                          groups.n)
    return rows, gdw, gdw1, gb


@pytest.fixture
def cpu_engine(monkeypatch):
    from paddlerec_b200 import ops, runner
    from paddlerec_b200.rank.deepfm import dygraph_model as criteo_base

    cpu_kernels.install(monkeypatch, ops)
    monkeypatch.setattr(ops, "raw_ffm_fwd", raw_ffm_fwd)
    monkeypatch.setattr(ops, "raw_ffm_bwd", raw_ffm_bwd)
    monkeypatch.setattr(runner, "_require_cuda", lambda: None)
    monkeypatch.setattr(criteo_base.DygraphModel, "device", "cpu")
    return runner


def test_stand_ins_match_the_oracle(cpu_engine):
    """The stand-ins are checked before the loop test relies on them."""
    from paddlerec_b200 import ops
    g = load_golden("ffm_d9")
    D, V = 9, g["param"]["ffm.embedding.weight"].shape[0]
    R = (F + Dn) * D
    W = torch.zeros(V, ops.fused_slot(R))
    W[:, :R] = torch.tensor(g["param"]["ffm.embedding.weight"], dtype=torch.float32)
    W[:, R] = torch.tensor(g["param"]["ffm.embedding_one.weight"][:, 0], dtype=torch.float32)
    p = to_params(g["param"], torch.float32, requires_grad=False)
    ids, dense = torch.tensor(g["in"]["ids"]), torch.tensor(g["in"]["dense"], dtype=torch.float32)
    y1, y2 = raw_ffm_fwd(W, ids, dense, p["ffm.dense_w"], p["ffm.dense_w_one"], None, -1, D)
    r1, r2 = ffm_oracle.ffm_terms(to_params(g["param"], requires_grad=False), slots(ids),
                            torch.tensor(g["in"]["dense"]), F + Dn)
    assert torch.allclose(y1.double(), r1.reshape(-1), atol=1e-5)
    assert torch.allclose(y2.double(), r2.reshape(-1), atol=1e-5)


def _config(runner, tmp_path, **over):
    d = os.path.join(PKG, "rank", "ffm")
    cfg = runner.load_yaml(os.path.join(d, "config.yaml"))
    cfg["config_abs_dir"] = d
    cfg["runner.model_save_path"] = str(tmp_path / "out")
    cfg["runner.infer_load_path"] = str(tmp_path / "out")
    cfg.update(over)
    return cfg


def test_ffm_train_infer_checkpoint_round_trip(cpu_engine, tmp_path):
    runner = cpu_engine
    V = 2003
    cfg = _config(runner, tmp_path, **{"runner.train_batch_size": 16, "runner.infer_batch_size": 16,
                                       "runner.epochs": 2, "runner.infer_end_epoch": 2,
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
    # the reference's five state_dict names and shapes (as minted from its net.py)
    R = (F + Dn) * 9
    want = {k: tuple(v.shape) for k, v in load_golden("ffm_d9")["param"].items()}
    want["ffm.embedding.weight"] = (V, R)
    want["ffm.embedding_one.weight"] = (V, 1)
    assert {k: tuple(v.shape) for k, v in saved.items()} == want
    for k, v in net.state_dict().items():
        assert np.array_equal(saved[k], v.numpy()), k
    # the saturation quirk, reproduced: every row of the bundled sample has a dense-only logit above
    # 17 under the reference's constant initialisers, p(1-p) is 0 in fp32, and nothing learns
    assert np.all(saved["ffm.dense_w"] == 1.0) and saved["bias"][0] == 0.0
