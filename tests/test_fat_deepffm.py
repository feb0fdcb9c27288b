"""FAT-DeepFFM on the CPU: the oracle against the goldens minted from the reference's
fat_deepffm/net.py, the reference's state_dict names and shapes, and the train -> infer ->
checkpoint loop of the fat_deepffm model directory (with torch stand-ins for the four FAT-DeepFFM
kernels, installed next to tests/cpu_kernels.py's)."""
import os

import numpy as np
import pytest
import torch

from tests import cpu_kernels, fat_deepffm_oracle
from tests.util import load_golden, slots, to_params

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "paddlerec_b200")
GF, GDn, GD = 8, 4, 10          # the goldens' fields and D (tests/golden/make_fat_deepffm_golden.py)


# ---- oracle vs goldens -----------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["fat_deepffm_d10", "fat_deepffm_d10_init"])
def test_oracle_matches_fat_deepffm_golden(name):
    from oracle import nets
    g = load_golden(name)
    p = to_params(g["param"])
    i = g["in"]
    pred = fat_deepffm_oracle.fat_deepffm_forward(p, slots(i["ids"]), torch.tensor(i["dense"]),
                                                  GF + GDn)
    loss = nets.log_loss(pred, torch.tensor(i["label"], dtype=torch.float64)).mean()
    grads = dict(zip(p, torch.autograd.grad(loss, list(p.values()))))
    np.testing.assert_allclose(pred.detach().numpy(), g["out"]["pred"], rtol=0, atol=1e-12)
    np.testing.assert_allclose(loss.detach().numpy(), g["out"]["loss"], rtol=0, atol=1e-12)
    assert set(grads) == set(g["grad"])
    for k, v in grads.items():
        np.testing.assert_allclose(v.numpy(), g["grad"][k], rtol=0, atol=1e-12, err_msg=k)


def test_fat_deepffm_goldens_cover_edge_cases():
    g = load_golden("fat_deepffm_d10")
    ids = g["in"]["ids"]
    assert (ids == 0).any() and ids[2, 5] == ids[2, 4] and len(set(ids[3:, 0])) == 1
    # no padding_idx: id 0 is a real row and receives gradient
    assert g["grad"]["cen.embedding.weight"][0].any()
    assert 0.01 < g["out"]["pred"].min() and g["out"]["pred"].max() < 0.99
    assert np.abs(g["grad"]["cen.dense_w"]).max() > 0 and np.abs(g["grad"]["bias"]).max() > 0
    init = load_golden("fat_deepffm_d10_init")
    assert np.all(init["param"]["cen.dense_w"] == 1.0) and (init["in"]["dense"] == 0).any()


def _pool_part_of_ddense_w(p, ids, dense, num_fields):
    """ddense_w of sum(pool) alone: where the max pool sends its gradient in the dense rows."""
    dw = p["cen.dense_w"].detach().clone().requires_grad_(True)
    q = dict(p, **{"cen.dense_w": dw})
    ids = torch.cat(list(ids), 1)
    feat = torch.cat([q["cen.embedding.weight"][ids], dense.unsqueeze(2) * dw], 1)
    D = feat.shape[2] // num_fields
    pooled = fat_deepffm_oracle.adaptive_max_pool1d_to_1(feat.reshape(-1, num_fields ** 2, D))
    return torch.autograd.grad(pooled.sum(), dw)[0]


def test_oracle_tie_rule_at_the_reference_initialisation():
    """dense_w = 1.0 makes every dense block an exact tie: the pool's gradient reaches only column 0
    of each block (the first maximum), for any dense value."""
    g = load_golden("fat_deepffm_d10_init")
    p = to_params(g["param"], requires_grad=False)
    gd = _pool_part_of_ddense_w(p, slots(g["in"]["ids"]), torch.tensor(g["in"]["dense"]), GF + GDn)
    blocks = gd.reshape(GDn, GF + GDn, GD)
    assert blocks[:, :, 0].abs().sum() > 0 and not blocks[:, :, 1:].any()


# ---- torch stand-ins for the four kernels (TEST DOUBLES, host-logic tests only) --------------------
def _e(W, ids, dense, dense_w, pad, D):
    V = W.shape[0]
    NF = ids.shape[1] + dense.shape[1]
    R = NF * D
    ok = ((ids >= 0) & (ids < V) & (ids != pad)).unsqueeze(2).to(W.dtype)
    return torch.cat([W[ids.clamp(0, V - 1), :R] * ok, dense.unsqueeze(2) * dense_w.reshape(1, -1, R)], 1)


def _pool(e, D):
    B = e.shape[0]
    return fat_deepffm_oracle.adaptive_max_pool1d_to_1(e.reshape(B, -1, D)).reshape(B, -1)


def _interact(e, attn, bias, D):
    B, NF = e.shape[0], e.shape[1]
    s = e.reshape(B, NF * NF, D) * attn.unsqueeze(2)
    y1 = s.sum((1, 2))
    if bias is not None:
        y1 = y1 + bias.reshape(())
    fa = s.reshape(B, NF, NF, D)
    iu = torch.triu_indices(NF, NF, 1)
    return y1, (fa[:, iu[0], iu[1]] * fa[:, iu[1], iu[0]]).reshape(B, -1)


def raw_fat_ffm_pool_fwd(W, ids, dense, dense_w, pad, D):
    return _pool(_e(W, ids, dense, dense_w, pad, D), D)


def raw_fat_ffm_fwd(W, ids, dense, dense_w, attn, bias, pad, D):
    return _interact(_e(W, ids, dense, dense_w, pad, D), attn, bias, D)


def raw_fat_ffm_bwd_attn(W, ids, dense, dense_w, attn, gy1, dh, pad, D):
    with torch.enable_grad():
        a = attn.detach().requires_grad_(True)
        y1, h = _interact(_e(W, ids, dense, dense_w, pad, D), a, None, D)
        return torch.autograd.grad((y1 * gy1).sum() + (h * dh).sum(), a)[0]


def raw_fat_ffm_bwd(W, ids, dense, dense_w, attn, gy1, dh, dpool, groups, pad, D):
    from paddlerec_b200 import ops
    with torch.enable_grad():
        leaf = W.detach().clone().requires_grad_(True)
        dw = dense_w.detach().clone().requires_grad_(True)
        e = _e(leaf, ids, dense, dw, pad, D)
        y1, h = _interact(e, attn, None, D)
        l = (y1 * gy1).sum() + (h * dh).sum() + (_pool(e, D) * dpool).sum()
        gW, gdw = torch.autograd.grad(l, [leaf, dw])
    R = e.shape[1] * D
    G = ops.fused_grad_cols(R)
    # per-position rows, then the segment reduce: what the kernel sums per id
    V = W.shape[0]
    ok = ((ids >= 0) & (ids < V) & (ids != pad)).reshape(-1)
    per_pos = torch.zeros(ids.numel(), G)
    with torch.enable_grad():
        leaf_rows = W[ids.clamp(0, V - 1)].detach().requires_grad_(True)
        e = torch.cat([leaf_rows[:, :, :R] * ok.reshape(ids.shape).unsqueeze(2).to(W.dtype),
                       dense.unsqueeze(2) * dense_w.reshape(1, -1, R)], 1)
        y1, h = _interact(e, attn, None, D)
        l = (y1 * gy1).sum() + (h * dh).sum() + (_pool(e, D) * dpool).sum()
        gr = torch.autograd.grad(l, leaf_rows)[0]
    per_pos[:, :R] = gr.reshape(-1, W.shape[1])[:, :R]
    rows = cpu_kernels.raw_segment_reduce(per_pos, groups.seg_offsets, groups.sorted_pos, groups.num,
                                          groups.n)
    del gW
    return rows, gdw.reshape(dense_w.shape), gy1.sum().reshape(1)


@pytest.fixture
def cpu_engine(monkeypatch):
    from paddlerec_b200 import ops, runner
    from paddlerec_b200.rank.deepfm import dygraph_model as criteo_base

    cpu_kernels.install(monkeypatch, ops)
    for f in (raw_fat_ffm_pool_fwd, raw_fat_ffm_fwd, raw_fat_ffm_bwd_attn, raw_fat_ffm_bwd):
        monkeypatch.setattr(ops, f.__name__, f)
    monkeypatch.setattr(runner, "_require_cuda", lambda: None)
    monkeypatch.setattr(criteo_base.DygraphModel, "device", "cpu")
    return runner


def _layer_on_golden(name):
    from paddlerec_b200.rank.fat_deepffm import net
    g = load_golden(name)
    V = g["param"]["cen.embedding.weight"].shape[0]
    layer = net.FAT_DeepFFMLayer(V, GD, GDn, GF, [32, 16], device="cpu")
    layer.load_state_dict({k: torch.tensor(v, dtype=torch.float32) for k, v in g["param"].items()})
    layer.eval()
    return g, layer


@pytest.mark.parametrize("name", ["fat_deepffm_d10", "fat_deepffm_d10_init"])
def test_stand_ins_through_the_layer_match_the_golden(cpu_engine, name):
    """The stand-ins, driven by the layer's autograd glue (one table pass), against the golden;
    checked before the loop test relies on them."""
    from oracle import nets
    g, layer = _layer_on_golden(name)
    ids = torch.tensor(g["in"]["ids"])
    pred = layer(ids, torch.tensor(g["in"]["dense"], dtype=torch.float32))
    loss = nets.log_loss(pred, torch.tensor(g["in"]["label"], dtype=torch.float32)).mean()
    loss.backward()
    np.testing.assert_allclose(pred.detach().numpy(), g["out"]["pred"], rtol=0, atol=1e-5)
    got = {"cen.embedding.weight": layer.cen.table_grad_dense(), "bias": layer.bias.grad}
    got.update({k: v.grad for k, v in layer.named_parameters() if v.grad is not None})
    assert set(got) == set(g["grad"])
    for k, v in got.items():
        want = g["grad"][k]
        np.testing.assert_allclose(v.detach().numpy(), want, rtol=1e-3,
                                   atol=1e-5 * max(np.abs(want).max(), 1e-3), err_msg=k)


def test_state_dict_names_and_shapes():
    from paddlerec_b200.rank.fat_deepffm import net
    V, D, F, Dn = 31, 10, 26, 13
    layer = net.FAT_DeepFFMLayer(V, D, Dn, F, [1600, 1600], device="cpu")
    NF = F + Dn
    R, NN, PD = NF * D, NF * NF, NF * (NF - 1) // 2 * D
    want = {"cen.embedding.weight": (V, R), "cen.dense_w": (1, Dn, R),
            "cen.fc.ReductionLinear.weight": (NN, NN), "cen.fc.ReductionLinear.bias": (NN,),
            "cen.fc.AdditionLinear.weight": (NN, NN), "cen.fc.AdditionLinear.bias": (NN,),
            "dnn.linear_0.weight": (PD, 1600), "dnn.linear_0.bias": (1600,),
            "dnn.linear_1.weight": (1600, 1600), "dnn.linear_1.bias": (1600,),
            "dnn.linear_2.weight": (1600, 1), "dnn.linear_2.bias": (1,), "bias": (1,)}
    assert {k: tuple(v.shape) for k, v in layer.state_dict().items()} == want
    assert PD == 7410
    # the same names the reference's net registers (as minted into the goldens)
    assert set(load_golden("fat_deepffm_d10")["param"]) == set(want)
    # the one-name fused table: the w1 column exists in the slot but stays zero and unexposed
    W = layer.cen._fused.weight
    assert not W[:, R].any() and len(layer.cen._fused.views()) == 1
    assert bool((layer.cen.dense_w.detach() == 1.0).all())
    assert layer.dnn.linear_0.weight.l2_decay == 1e-7


def _config(runner, tmp_path, **over):
    d = os.path.join(PKG, "rank", "fat_deepffm")
    cfg = runner.load_yaml(os.path.join(d, "config.yaml"))
    cfg["config_abs_dir"] = d
    cfg["runner.model_save_path"] = str(tmp_path / "out")
    cfg["runner.infer_load_path"] = str(tmp_path / "out")
    cfg.update(over)
    return cfg


def test_fat_deepffm_train_infer_checkpoint_round_trip(cpu_engine, tmp_path):
    runner = cpu_engine
    V = 2003
    cfg = _config(runner, tmp_path, **{"runner.train_batch_size": 16, "runner.infer_batch_size": 16,
                                       "runner.epochs": 2, "runner.infer_end_epoch": 2,
                                       "hyper_parameters.sparse_feature_number": V,
                                       "hyper_parameters.layer_sizes_dnn": [64, 32],
                                       "runner.reader_type": "PackedReader"})
    losses, metric_values, net = runner.train(cfg)
    assert len(losses) == 10 and np.all(np.isfinite(losses)) and "auc" in metric_values
    for e in range(2):
        assert sorted(os.listdir(tmp_path / "out" / str(e))) == ["rec.pdopt", "rec.pdparams"]
    results = runner.infer(cfg)
    assert sorted(results) == [0, 1] and all(0.0 <= r["auc"] <= 1.0 for r in results.values())

    from paddlerec_b200 import checkpoint
    saved = checkpoint.load_pdparams(str(tmp_path / "out" / "1" / "rec.pdparams"))
    R = 39 * 10
    assert saved["cen.embedding.weight"].shape == (V, R)
    assert saved["dnn.linear_0.weight"].shape == (741 * 10, 64)
    for k, v in net.state_dict().items():
        assert np.array_equal(saved[k], v.numpy()), k
    # the fused table's hidden w1 column stayed zero through two epochs of lazy Adam
    assert not net.cen._fused.weight[:, R].any()
    # SURVEY.md Q17: with dense_w = 1.0 the Criteo dense values drive every sample's logit far past
    # fp32 sigmoid saturation, so each loss is a multiple of -log(1e-4) / 16 and nothing learns
    unit = -np.log(1e-4) / 16
    assert np.allclose(np.array(losses) / unit, np.round(np.array(losses) / unit), atol=1e-3)
    assert np.all(saved["cen.dense_w"] == 1.0)
