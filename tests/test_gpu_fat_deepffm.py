"""FAT-DeepFFM on the GPU: the four b200rec_fat_ffm_* kernels against an fp64 oracle (autograd over
tests/fat_deepffm_oracle.py's operations), the layer against the goldens minted from the reference's
fat_deepffm/net.py, the first-maximum tie rule at the reference's initialisation, determinism with
a hot id, padding / out-of-range ids, rejected shapes, one B=65536 step, and the trainer."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from tests.util import elementwise_excess, load_golden

pytestmark = pytest.mark.gpu
DEV = "cuda"
U32 = 2.0 ** -24          # unit roundoff of fp32


@pytest.fixture(autouse=True)
def _reset_oob():
    yield
    from paddlerec_b200 import ops
    ops.raw_oob_count(reset=True)


def _problem(B, F, Dn, D, V, seed, zipf=None, scale=0.1):
    from paddlerec_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(seed)
    NF = F + Dn
    R = NF * D
    W = torch.zeros(V, ops.fused_slot(R), device=DEV)
    W[:, :R] = torch.randn(V, R, device=DEV, generator=g) * scale
    W[:, R] = 7.0                       # the unused w1 column: must not leak into anything
    if zipf is None:
        ids = torch.randint(0, V, (B, F), device=DEV, generator=g)
    else:
        rng = np.random.default_rng(seed)
        ids = torch.tensor((rng.zipf(zipf, size=(B, F)) - 1) % V, device=DEV)
    dense = torch.rand(B, Dn, device=DEV, generator=g) * 2 - 0.5     # both signs
    dense_w = torch.randn(Dn, R, device=DEV, generator=g) * scale
    attn = torch.relu(torch.randn(B, NF * NF, device=DEV, generator=g) + 0.3)   # ReLU zeros too
    gy1 = torch.randn(B, device=DEV, generator=g)
    dh = torch.randn(B, NF * (NF - 1) // 2 * D, device=DEV, generator=g)
    dpool = torch.randn(B, NF * NF, device=DEV, generator=g)
    return W, ids, dense, dense_w, attn, gy1, dh, dpool


def _oracle(W, ids, dense, dense_w, attn, bias, gy1, dh, dpool, D, pad=-1, absolute=False):
    """fp64 pool, y1, h and the gradients of sum(gy1*y1 + dh*h + dpool*pool) w.r.t. the table,
    dense_w and attn.  The argmax is taken on the fp32 rows as the kernels form them (first
    maximum); absolute=True replaces every input by its magnitude, turning each output into the
    sum of |terms| it adds."""
    B, F = ids.shape
    Dn = dense.shape[1]
    NF, R, NN = F + Dn, (F + Dn) * D, (F + Dn) ** 2
    V = W.shape[0]
    f = (lambda t: t.double().abs()) if absolute else (lambda t: t.double())
    ok = ((ids >= 0) & (ids < V) & (ids != pad)).unsqueeze(2)
    idc = ids.clamp(0, V - 1)
    e32 = torch.cat([W[idc, :R] * ok, dense.unsqueeze(2) * dense_w.unsqueeze(0)], 1)
    idx = (e32.reshape(B, NN, D) == e32.reshape(B, NN, D).max(-1, keepdim=True).values
           ).to(torch.int8).argmax(-1, keepdim=True)
    tw = f(W[:, :R]).requires_grad_(True)
    dw = f(dense_w).requires_grad_(True)
    at = f(attn).requires_grad_(True)
    e = torch.cat([tw[idc] * ok.double(), f(dense).unsqueeze(2) * dw.unsqueeze(0)], 1)
    pool = torch.gather(e.reshape(B, NN, D), -1, idx).reshape(B, NN)
    s = e.reshape(B, NN, D) * at.unsqueeze(2)
    y1 = s.sum((1, 2)) + (0.0 if bias is None else f(bias))
    fa = s.reshape(B, NF, NF, D)
    iu = torch.triu_indices(NF, NF, 1, device=W.device)
    h = (fa[:, iu[0], iu[1]] * fa[:, iu[1], iu[0]]).reshape(B, -1)
    l = (f(gy1) * y1).sum() + (f(dh) * h).sum() + (f(dpool) * pool).sum()
    gw, gdw, gat = torch.autograd.grad(l, [tw, dw, at])
    return {"pool": pool.detach(), "y1": y1.detach(), "h": h.detach(), "dW": gw, "ddw": gdw,
            "dattn": gat}


def _run(W, ids, dense, dense_w, attn, bias, gy1, dh, dpool, D, pad=-1):
    from paddlerec_b200 import ops
    pool = ops.raw_fat_ffm_pool_fwd(W, ids, dense, dense_w, pad, D)
    y1, h = ops.raw_fat_ffm_fwd(W, ids, dense, dense_w, attn, bias, pad, D)
    dattn = ops.raw_fat_ffm_bwd_attn(W, ids, dense, dense_w, attn, gy1, dh, pad, D)
    groups = ops.raw_group_ids(ids, W.shape[0], pad)
    rows, ddw, db = ops.raw_fat_ffm_bwd(W, ids, dense, dense_w, attn, gy1, dh, dpool, groups, pad, D)
    return {"pool": pool, "y1": y1, "h": h, "dattn": dattn, "groups": groups, "rows": rows,
            "ddw": ddw, "dbias": db}


def _dense_rows(groups, rows, V):
    U = int(groups.num[0])
    out = torch.zeros(V, rows.shape[1], dtype=torch.float64, device=DEV)
    out[groups.unique_ids[:U]] = rows[:U].double()
    return out


def _within(got, want, mag, k, what=""):
    """|got - want| <= k * (sum of |terms|): k is gamma_n = n*u/(1-n*u) for the longest chain of
    fp32 roundings that forms the output (Higham, Accuracy and Stability, 3.1), times 1.01."""
    excess = (got.double() - want).abs() - k * 1.01 * mag - 1e-30
    assert float(excess.max()) <= 0, "%s: worst excess %.3e" % (what, float(excess.max()))


def _gamma(n):
    return n * U32 / (1 - n * U32)


def _check_all(out, W, ids, dense, dense_w, attn, bias, gy1, dh, dpool, D, pad=-1):
    B, F = ids.shape
    Dn = dense.shape[1]
    NF, R, NN = F + Dn, (F + Dn) * D, (F + Dn) ** 2
    V = W.shape[0]
    r = _oracle(W, ids, dense, dense_w, attn, bias, gy1, dh, dpool, D, pad)
    m = _oracle(W, ids, dense, dense_w, attn, bias, gy1, dh, dpool, D, pad, absolute=True)
    # a maximum is exact: the kernel's pool is the oracle's rounded to fp32, bit for bit (an fp64
    # product of fp32 values is exact, so its rounding is the kernel's fp32 product)
    assert torch.equal(out["pool"], r["pool"].float())
    # y1: per thread ceil(NN/256) blocks of D adds and one fma each, 5 shuffles, 8 warp sums, bias
    _within(out["y1"], r["y1"], m["y1"], _gamma(math.ceil(NN / 256) * (D + 1) + 14), "y1")
    # h: two dense products (x * dense_w), two attention products, one final product
    _within(out["h"], r["h"], m["h"], _gamma(5), "h")
    # dattn: a chain of D fmas of e * (gy1 + dh * attn * e), each term with 4 roundings of its own
    _within(out["dattn"], r["dattn"], m["dattn"], _gamma(D + 5), "dattn")
    # a table row: ~5 roundings per position, then the segment's positions in a fixed chain (light
    # warps walk up to 64 in a row; hot CTAs 1024/8 + 8, then the chunks)
    counts = torch.bincount(ids[(ids >= 0) & (ids < V) & (ids != pad)], minlength=V)
    n_pos = int(counts.max())
    chain = min(n_pos, 64) if n_pos <= 64 else 128 + 8 + math.ceil(n_pos / 1024)
    full = _dense_rows(out["groups"], out["rows"], V)
    _within(full[:, :R], r["dW"], m["dW"], _gamma(chain + 6), "dW")
    assert not full[:, R:].any()                       # w1 and padding columns are exactly 0
    slices = max(1, min(256, (B + 255) // 256))
    per_slice = math.ceil(B / slices)
    if Dn:
        _within(out["ddw"], r["ddw"], m["ddw"], _gamma(per_slice + slices + 6), "ddw")
    _within(out["dbias"], gy1.double().sum().reshape(1), gy1.double().abs().sum().reshape(1),
            _gamma(per_slice + slices), "dbias")


def _fat_smem(F, Dn, D, nbuf):
    """FatSmem (csrc/fat_ffm.cuh): dense_w | pairs | attention row | reduction | nbuf buffers."""
    NF = F + Dn
    R, P = NF * D, NF * (NF - 1) // 2
    up = lambda x: (x + 15) // 16 * 16                                     # noqa: E731
    off_buf = up(up(up(Dn * R * 4) + P * 4) + NF * NF * 4) + 16 * (256 // 32 + 4)
    return off_buf + nbuf * F * ((R + 1 + 3) // 4 * 4) * 4


def _smem_limit():
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin


def _largest_d(F=26, Dn=13):
    D = 1
    while _fat_smem(F, Dn, D + 1, 1) <= _smem_limit():
        D += 1
    return D


@pytest.mark.parametrize("F,Dn,D,B", [(26, 13, 1, 300), (26, 13, 4, 300), (26, 13, 10, 300),
                                      (26, 13, 16, 300), (26, 13, "max", 200), (3, 2, 10, 300),
                                      (5, 0, 16, 300), (1, 1, 3, 300), (2, 0, 7, 300),
                                      (26, 13, 10, 1)])
def test_fat_kernels_vs_fp64_oracle(F, Dn, D, B):
    if D == "max":
        D = _largest_d(F, Dn)
        assert _fat_smem(F, Dn, D, 2) > _smem_limit()      # the single-buffered path
    V = 97
    W, ids, dense, dense_w, attn, gy1, dh, dpool = _problem(B, F, Dn, D, V, seed=F * 100 + D)
    ids[0, 0] = ids[0, -1]                       # the same row at two fields of one sample
    bias = torch.tensor([0.3], device=DEV)
    out = _run(W, ids, dense, dense_w, attn, bias, gy1, dh, dpool, D)
    _check_all(out, W, ids, dense, dense_w, attn, bias, gy1, dh, dpool, D)


def _layer_from_golden(name):
    from paddlerec_b200.rank.fat_deepffm import net
    g = load_golden(name)
    V = g["param"]["cen.embedding.weight"].shape[0]
    layer = net.FAT_DeepFFMLayer(V, 10, 4, 8, [32, 16], device=DEV)
    layer.load_state_dict({k: torch.tensor(v, dtype=torch.float32) for k, v in g["param"].items()})
    layer.eval()                                          # the goldens are eval mode (dropout off)
    return g, layer


@pytest.mark.parametrize("name", ["fat_deepffm_d10", "fat_deepffm_d10_init"])
@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
def test_fat_deepffm_layer_matches_golden(name, precision):
    """FAT_DeepFFMLayer end to end (fused table, both autograd halves, the attention MLP, the DNN,
    sum_sigmoid, the log-loss kernels) on the golden's parameters: pred, loss and every gradient.

    Tolerance: element-wise 1e-4 in fp32.  Under 'bf16x3' the attention MLP and the DNN run on the
    split-bf16 wgmma GEMMs, whose dropped lo*lo products leave ~2^-16 relative error per dot
    product; where a ReLU's input is within that of zero the unit's gradient switches on or off,
    and the attention MLP's 144 outputs all feed every table gradient, so that mode is held to
    2e-3."""
    from paddlerec_b200 import functional as BF
    from paddlerec_b200 import nn as bnn
    bnn.set_matmul_precision(precision)
    try:
        g, layer = _layer_from_golden(name)
        ids = torch.tensor(g["in"]["ids"], device=DEV)
        dense = torch.tensor(g["in"]["dense"], dtype=torch.float32, device=DEV)
        label = torch.tensor(g["in"]["label"], device=DEV)
        pred = layer([ids[:, i:i + 1] for i in range(8)], dense)
        loss = BF.log_loss_mean(pred, label)
        loss.backward()
        tol = 1e-4 if precision == "fp32" else 2e-3
        assert elementwise_excess(pred, g["out"]["pred"], tol, tol) <= 0
        assert elementwise_excess(loss, g["out"]["loss"], tol, tol) <= 0
        got = {"cen.embedding.weight": layer.cen.table_grad_dense()}
        got.update({k: v.grad for k, v in layer.named_parameters() if v.grad is not None})
        assert set(got) == set(g["grad"])
        for k, v in got.items():
            assert elementwise_excess(v, g["grad"][k], tol, tol) <= 0, k
    finally:
        bnn.set_matmul_precision("fp32")


def test_fat_tie_rule_at_the_reference_initialisation():
    """dense_w = 1.0 (the reference's Constant(1.0)): every dense block is an exact tie, so the pool
    part of ddense_w is nonzero only in column 0 of each block, for positive, negative and zero
    dense values alike."""
    from paddlerec_b200 import ops
    B, F, Dn, D, V = 256, 26, 13, 10, 500
    W, ids, dense, _, attn, gy1, dh, dpool = _problem(B, F, Dn, D, V, seed=31)
    dense_w = torch.ones(Dn, (F + Dn) * D, device=DEV)
    dense[::7] = 0.0
    zero = torch.zeros_like
    groups = ops.raw_group_ids(ids, V, -1)
    _, ddw, _ = ops.raw_fat_ffm_bwd(W, ids, dense, dense_w, attn, zero(gy1), zero(dh), dpool, groups,
                                    -1, D)
    blocks = ddw.reshape(Dn, F + Dn, D)
    assert bool((blocks[:, :, 0] != 0).all()) and not blocks[:, :, 1:].any()
    # and the whole gradient against fp64 at that initialisation
    out = _run(W, ids, dense, dense_w, attn, None, gy1, dh, dpool, D)
    _check_all(out, W, ids, dense, dense_w, attn, None, gy1, dh, dpool, D)


def test_fat_deterministic_with_a_hot_id():
    """Zipf ids plus one id at 3000 positions (three hot chunks and a combine): a second run is bit
    identical, and the result matches the fp64 oracle."""
    B, F, Dn, D, V = 4096, 26, 13, 10, 5000
    W, ids, dense, dense_w, attn, gy1, dh, dpool = _problem(B, F, Dn, D, V, seed=11, zipf=1.05)
    ids[:3000, 7] = 4242
    a = _run(W, ids, dense, dense_w, attn, None, gy1, dh, dpool, D)
    b = _run(W, ids, dense, dense_w, attn, None, gy1, dh, dpool, D)
    assert int(torch.bincount(ids.reshape(-1), minlength=V).max()) > 2048
    U = int(a["groups"].num[0])
    for k in ("pool", "y1", "h", "dattn", "ddw", "dbias"):
        assert torch.equal(a[k], b[k]), k
    assert torch.equal(a["rows"][:U], b["rows"][:U])
    _check_all(a, W, ids, dense, dense_w, attn, None, gy1, dh, dpool, D)


def test_fat_padding_and_out_of_range_ids():
    from paddlerec_b200 import ops
    B, F, Dn, D, V, pad = 64, 26, 13, 4, 50, 3
    W, ids, dense, dense_w, attn, gy1, dh, dpool = _problem(B, F, Dn, D, V, seed=2)
    ids[0, 0], ids[1, 5], ids[2, :] = V + 5, -7, pad
    ids[3, 1] = pad
    ops.raw_oob_count(reset=True)
    ops.raw_fat_ffm_pool_fwd(W, ids, dense, dense_w, pad, D)
    assert ops.raw_oob_count(reset=True) == 2          # counted once per position, by the pool
    ops.raw_fat_ffm_fwd(W, ids, dense, dense_w, attn, None, pad, D)
    ops.raw_fat_ffm_bwd_attn(W, ids, dense, dense_w, attn, gy1, dh, pad, D)
    assert ops.raw_oob_count(reset=True) == 0          # and by no later kernel of the step
    out = _run(W, ids, dense, dense_w, attn, None, gy1, dh, dpool, D, pad=pad)
    rows = out["groups"].unique_ids[:int(out["groups"].num[0])]
    assert not bool(((rows == pad) | (rows < 0) | (rows >= V)).any())
    _check_all(out, W, ids, dense, dense_w, attn, None, gy1, dh, dpool, D, pad=pad)


def test_fat_rejects_what_it_cannot_hold():
    from paddlerec_b200 import _lib
    lib = _lib.load()
    W = torch.zeros(10, 4096, device=DEV)
    ids = torch.zeros(4, 40, dtype=torch.int64, device=DEV)
    buf = torch.zeros(1 << 20, device=DEV)
    P = ctypes.c_void_p
    w, x = P(W.data_ptr()), P(buf.data_ptr())

    def fwd(F, Dn, D, ldw, w_off=0):
        return lib.b200rec_fat_ffm_fwd(P(W.data_ptr() + w_off), ldw, P(ids.data_ptr()), x, x, x, None,
                                       x, x, 4, F, Dn, D, 10, -1, None)

    def attn_bwd(F, Dn, D, ldw):
        return lib.b200rec_fat_ffm_bwd_attn(w, ldw, P(ids.data_ptr()), x, x, x, x, x, x, 4, F, Dn, D,
                                            10, -1, None)

    def pool(F, Dn, D, ldw):
        return lib.b200rec_fat_ffm_pool_fwd(w, ldw, P(ids.data_ptr()), x, x, x, 4, F, Dn, D, 10, -1,
                                            None)
    assert fwd(26, 13, 10, 392) == 0 and attn_bwd(26, 13, 10, 392) == 0 and pool(26, 13, 10, 392) == 0
    torch.cuda.synchronize()
    for call in (fwd, attn_bwd, pool):
        assert call(26, 13, 10, 390) == -1 and b"ldw" in lib.b200rec_last_error()   # no room for w1
        assert call(26, 13, 10, 394) == -1                                           # ldw % 4
        assert call(40, 30, 1, 4096) == -1 and b"F+Dn" in lib.b200rec_last_error()  # > 64 fields
        assert call(0, 13, 10, 4096) == -1
        assert call(26, 13, 0, 4096) == -1
    assert fwd(26, 13, 10, 392, w_off=4) == -1                        # W not 16-byte aligned
    Dmax = _largest_d()
    ldw = ((39 * (Dmax + 1) + 1) + 3) // 4 * 4
    assert fwd(26, 13, Dmax + 1, ldw) == -1 and b"shared memory" in lib.b200rec_last_error()
    assert attn_bwd(26, 13, Dmax + 1, ldw) == -1 and b"shared memory" in lib.b200rec_last_error()
    n = ctypes.c_size_t(0)
    assert lib.b200rec_fat_ffm_bwd_workspace_bytes(4, 26, 13, 10, ctypes.byref(n)) == 0 and n.value > 0
    assert lib.b200rec_fat_ffm_bwd_workspace_bytes(4, 40, 30, 10, ctypes.byref(n)) == -1
    rc = lib.b200rec_fat_ffm_bwd(w, 392, P(ids.data_ptr()), x, x, x, x, x, x, x, x, x, x, 392, x, x,
                                 4, 26, 13, 10, 10, -1, x, n.value - 1, None)
    assert rc != 0 and b"workspace" in lib.b200rec_last_error()


# ---- one training step at the benchmark's size -----------------------------------------------------
NS = 512


def test_fat_full_size_step_on_a_slice_vs_oracle():
    """B=65536, V=1e6, D=10: the prediction of a 512-sample slice whose ids appear nowhere else in
    the batch, and the gradient rows of every id of that slice (so only these samples contribute),
    against fp64; then one lazy Adam step changes exactly the touched rows.  Eval mode: the DNN's
    dropout would make the step random."""
    from oracle import nets
    from paddlerec_b200 import functional as BF
    from paddlerec_b200 import optim
    from paddlerec_b200.rank.fat_deepffm import net
    from tests import fat_deepffm_oracle
    torch.cuda.empty_cache()
    if torch.cuda.mem_get_info()[0] < 30e9:
        pytest.skip("needs ~20 GB of free HBM")
    B, V, D, F, Dn = 65536, 1_000_000, 10, 26, 13
    NF = F + Dn
    torch.manual_seed(1)
    layer = net.FAT_DeepFFMLayer(V, D, Dn, F, [1600, 1600], device=DEV)
    layer.eval()
    with torch.no_grad():      # the reference's constant 1.0 saturates the sigmoid (SURVEY.md Q17)
        layer.cen.dense_w.normal_(0, 0.05)
    g = torch.Generator(device=DEV).manual_seed(9)
    ids = torch.randint(0, V - 100_000, (B, F), device=DEV, generator=g)
    ids[:NS] = torch.randint(V - 100_000, V, (NS, F), device=DEV, generator=g)
    ids[:NS:5, 2] = V - 77
    dense = torch.rand(B, Dn, device=DEV, generator=g)
    label = (torch.rand(B, 1, device=DEV, generator=g) < 0.3).float()
    opt = optim.Adam(learning_rate=1e-4, parameters=layer.parameters())
    pred = layer(ids, dense)
    BF.log_loss_mean(pred, label).backward()
    s = slice(0, NS)
    W = layer.cen._fused.weight.detach()
    uniq = torch.unique(ids[s])
    remap = torch.searchsorted(uniq, ids[s])
    R = NF * D
    p = {k: v.detach().double() for k, v in layer.state_dict().items() if k != "cen.embedding.weight"}
    p["cen.embedding.weight"] = W[uniq, :R].double()
    p = {k: v.requires_grad_(True) for k, v in p.items()}
    ref = fat_deepffm_oracle.fat_deepffm_forward(p, [remap[:, i:i + 1] for i in range(F)],
                                                 dense[s].double(), NF)
    assert elementwise_excess(pred[s], ref) <= 0
    l = nets.log_loss(ref, label[s].double()).sum() / B
    gw = torch.autograd.grad(l, [p["cen.embedding.weight"]])[0]
    sr = layer.cen._fused.grad_rows
    U = int(sr.num[0])
    where = torch.searchsorted(sr.rows[:U].contiguous(), uniq)
    assert torch.equal(sr.rows[where], uniq)
    assert elementwise_excess(sr.value[where, :R], gw) <= 0
    assert not sr.value[:U, R:].any()
    before = W[V - 100_000:].clone()
    opt.step()
    touched = torch.zeros(V, dtype=torch.bool, device=DEV)
    touched[sr.rows[:U]] = True
    changed = (W[V - 100_000:] != before).any(1)
    assert torch.equal(changed, touched[V - 100_000:])
    assert not W[:, R].any()


def test_fat_deepffm_trainer_runs_the_sample_config(tmp_path):
    """tools/trainer.py's loop on the model directory's config (B=1, V=1e6+1, D=10) for the 80
    bundled sample rows; loss and AUC are finite, and the saved model infers."""
    from paddlerec_b200 import runner
    d = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "paddlerec_b200",
                     "rank", "fat_deepffm")
    cfg = runner.load_yaml(os.path.join(d, "config.yaml"))
    cfg["config_abs_dir"] = d
    cfg["runner.model_save_path"] = str(tmp_path / "out")
    cfg["runner.infer_load_path"] = str(tmp_path / "out")
    losses, metric_values, _ = runner.train(cfg)
    assert len(losses) > 0 and np.all(np.isfinite(losses))
    assert np.isfinite(metric_values["auc"])
    results = runner.infer(cfg)
    assert all(np.isfinite(r["auc"]) for r in results.values())
