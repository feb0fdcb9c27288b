"""FFM on the GPU: b200rec_ffm_fwd / _bwd against the fp64 oracle (tests/ffm_oracle.py and its
autograd) and against the goldens minted from the reference's ffm/net.py; determinism with a hot id;
padding / out-of-range ids; rejected shapes; the wide-row optimizers; and one B=65536, V=1e6 step."""
import ctypes

import numpy as np
import pytest
import torch

from tests.util import elementwise_excess, load_golden

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(autouse=True)
def _reset_oob():
    yield
    from paddlerec_b200 import ops
    ops.raw_oob_count(reset=True)


def _problem(B, F, Dn, D, V, seed, pad=-1, zipf=None, scale=0.1):
    from paddlerec_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(seed)
    R = (F + Dn) * D
    W = torch.zeros(V, ops.fused_slot(R), device=DEV)
    W[:, :R + 1] = torch.randn(V, R + 1, device=DEV, generator=g) * scale
    if zipf is None:
        ids = torch.randint(0, V, (B, F), device=DEV, generator=g)
    else:
        rng = np.random.default_rng(seed)
        ids = torch.tensor((rng.zipf(zipf, size=(B, F)) - 1) % V, device=DEV)
    dense = torch.rand(B, Dn, device=DEV, generator=g)
    dense_w = torch.randn(Dn, R, device=DEV, generator=g) * scale
    dense_w1 = torch.randn(Dn, device=DEV, generator=g) * scale
    return W, ids, dense, dense_w, dense_w1


def _oracle(W, ids, dense, dense_w, dense_w1, bias, gy1, gy2, D, pad=-1, absolute=False):
    """fp64 (on the GPU) y1, y2 and the gradients of sum(gy1*y1 + gy2*y2); with absolute=True every
    input is replaced by its magnitude, which turns each output into the sum of |terms| it adds."""
    F, Dn = ids.shape[1], dense.shape[1]
    NF, R = F + Dn, (F + Dn) * D
    f = (lambda t: t.double().abs()) if absolute else (lambda t: t.double())
    V = W.shape[0]
    ok = ((ids >= 0) & (ids < V) & (ids != pad)).double().unsqueeze(2)
    idc = ids.clamp(0, V - 1)
    p = {"ffm.embedding.weight": f(W[:, :R]).requires_grad_(True),
         "ffm.embedding_one.weight": f(W[:, R:R + 1]).requires_grad_(True),
         "ffm.dense_w": f(dense_w).reshape(1, Dn, R).requires_grad_(True),
         "ffm.dense_w_one": f(dense_w1).requires_grad_(True)}
    emb = p["ffm.embedding.weight"][idc] * ok
    emb1 = p["ffm.embedding_one.weight"][idc] * ok
    # ffm_oracle.ffm_terms over pre-gathered rows, so that padding / out-of-range ids read zeros
    dx = f(dense)
    y1 = emb1.sum(1) + (dx * p["ffm.dense_w_one"]).unsqueeze(2).sum(1)
    feat = torch.cat([emb, dx.unsqueeze(2) * p["ffm.dense_w"]], 1).reshape(-1, NF, NF, D)
    iu = torch.triu_indices(NF, NF, 1, device=W.device)
    y2 = (feat[:, iu[0], iu[1]] * feat[:, iu[1], iu[0]]).sum((1, 2)).unsqueeze(1)
    if bias is not None:
        y1 = y1 + f(bias)
    l = (f(gy1) * y1.reshape(-1)).sum() + (f(gy2) * y2.reshape(-1)).sum()
    grads = dict(zip(p, torch.autograd.grad(l, list(p.values()))))
    return y1.detach().reshape(-1), y2.detach().reshape(-1), grads


def _run(W, ids, dense, dense_w, dense_w1, bias, gy1, gy2, D, pad=-1):
    from paddlerec_b200 import ops
    y1, y2 = ops.raw_ffm_fwd(W, ids, dense, dense_w, dense_w1, bias, pad, D)
    groups = ops.raw_group_ids(ids, W.shape[0], pad)
    dW, ddw, ddw1, db = ops.raw_ffm_bwd(W, ids, dense, dense_w, gy1, gy2, groups, pad, D)
    return y1, y2, groups, dW, ddw, ddw1, db


def _dense_rows(groups, dW, V):
    U = int(groups.num[0])
    out = torch.zeros(V, dW.shape[1], dtype=torch.float64, device=DEV)
    out[groups.unique_ids[:U]] = dW[:U].double()
    return out


def _within(got, want, mag, k=2e-6, what=""):
    excess = (got.double() - want).abs() - k * mag - 1e-30
    assert float(excess.max()) <= 0, "%s: worst excess %.3e" % (what, float(excess.max()))


@pytest.mark.parametrize("F,Dn,D", [(26, 13, 1), (26, 13, 4), (26, 13, 9), (26, 13, 16),
                                    (26, 13, 32), (3, 2, 9), (5, 0, 16), (1, 1, 3), (2, 0, 7)])
def test_ffm_kernels_vs_fp64_oracle(F, Dn, D):
    B, V = 300, 97
    W, ids, dense, dense_w, dense_w1 = _problem(B, F, Dn, D, V, seed=F * 100 + D)
    ids[0, 0] = ids[0, -1]                       # the same row at two fields of one sample
    bias = torch.tensor([0.3], device=DEV)
    g = torch.Generator(device=DEV).manual_seed(5)
    gy1, gy2 = torch.randn(B, device=DEV, generator=g), torch.randn(B, device=DEV, generator=g)
    y1, y2, groups, dW, ddw, ddw1, db = _run(W, ids, dense, dense_w, dense_w1, bias, gy1, gy2, D)
    r1, r2, rg = _oracle(W, ids, dense, dense_w, dense_w1, bias, gy1, gy2, D)
    m1, m2, mg = _oracle(W, ids, dense, dense_w, dense_w1, bias, gy1, gy2, D, absolute=True)
    _within(y1, r1, m1, what="y1")
    _within(y2, r2, m2, what="y2")
    R = (F + Dn) * D
    full = _dense_rows(groups, dW, V)
    _within(full[:, :R], rg["ffm.embedding.weight"], mg["ffm.embedding.weight"], what="dW")
    _within(full[:, R:R + 1], rg["ffm.embedding_one.weight"], mg["ffm.embedding_one.weight"],
            what="dW1")
    assert not full[:, R + 1:].any()
    if Dn:
        _within(ddw, rg["ffm.dense_w"].reshape(Dn, R), mg["ffm.dense_w"].reshape(Dn, R), what="ddw")
        _within(ddw1, rg["ffm.dense_w_one"], mg["ffm.dense_w_one"], what="ddw1")
    _within(db, gy1.double().sum().reshape(1), gy1.double().abs().sum().reshape(1), what="dbias")


@pytest.mark.parametrize("name,D", [("ffm_d9", 9), ("ffm_d16", 16)])
def test_ffm_layer_matches_golden(name, D):
    """FFMLayer end to end (fused table, autograd, sum_sigmoid, log-loss kernels) on the golden's
    parameters: pred, loss and every gradient element-wise within 1e-4."""
    from paddlerec_b200 import functional as BF
    from paddlerec_b200.rank.ffm import net
    g = load_golden(name)
    V = g["param"]["ffm.embedding.weight"].shape[0]
    layer = net.FFMLayer(V, D, 13, 39, device=DEV)
    layer.load_state_dict({k: torch.tensor(v, dtype=torch.float32) for k, v in g["param"].items()})
    ids = torch.tensor(g["in"]["ids"], device=DEV)
    dense = torch.tensor(g["in"]["dense"], dtype=torch.float32, device=DEV)
    label = torch.tensor(g["in"]["label"], device=DEV)
    pred = layer([ids[:, i:i + 1] for i in range(26)], dense)
    loss = BF.log_loss_mean(pred, label)
    loss.backward()
    assert elementwise_excess(pred, g["out"]["pred"]) <= 0
    assert elementwise_excess(loss, g["out"]["loss"]) <= 0
    dW, dW1 = layer.ffm.table_grad_dense()
    got = {"ffm.embedding.weight": dW, "ffm.embedding_one.weight": dW1,
           "ffm.dense_w": layer.ffm.dense_w.grad, "ffm.dense_w_one": layer.ffm.dense_w_one.grad,
           "bias": layer.bias.grad}
    assert set(got) == set(g["grad"])
    for k, v in got.items():
        assert elementwise_excess(v, g["grad"][k]) <= 0, k


def test_ffm_deterministic_with_a_hot_id():
    """Zipf ids plus one id at 3000 positions (two hot chunks and a combine): a second run is bit
    identical, and the result matches the fp64 oracle."""
    B, F, Dn, D, V = 4096, 26, 13, 9, 5000
    W, ids, dense, dense_w, dense_w1 = _problem(B, F, Dn, D, V, seed=11, zipf=1.05)
    ids[:3000, 7] = 4242
    g = torch.Generator(device=DEV).manual_seed(3)
    gy1, gy2 = torch.randn(B, device=DEV, generator=g), torch.randn(B, device=DEV, generator=g)
    a = _run(W, ids, dense, dense_w, dense_w1, None, gy1, gy2, D)
    b = _run(W, ids, dense, dense_w, dense_w1, None, gy1, gy2, D)
    U = int(a[2].num[0])
    counts = torch.bincount(ids.reshape(-1), minlength=V)
    assert int(counts.max()) > 2048
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert torch.equal(a[3][:U], b[3][:U])
    for x, y in zip(a[4:], b[4:]):
        assert torch.equal(x, y)
    _, _, rg = _oracle(W, ids, dense, dense_w, dense_w1, None, gy1, gy2, D)
    _, _, mg = _oracle(W, ids, dense, dense_w, dense_w1, None, gy1, gy2, D, absolute=True)
    R = (F + Dn) * D
    full = _dense_rows(a[2], a[3], V)
    _within(full[:, :R], rg["ffm.embedding.weight"], mg["ffm.embedding.weight"], k=4e-6, what="dW")
    _within(full[:, R:R + 1], rg["ffm.embedding_one.weight"], mg["ffm.embedding_one.weight"],
            k=4e-6, what="dW1")
    _within(a[4], rg["ffm.dense_w"].reshape(Dn, R), mg["ffm.dense_w"].reshape(Dn, R), k=4e-6,
            what="ddw")


def test_ffm_padding_and_out_of_range_ids():
    from paddlerec_b200 import ops
    B, F, Dn, D, V, pad = 64, 26, 13, 4, 50, 3
    W, ids, dense, dense_w, dense_w1 = _problem(B, F, Dn, D, V, seed=2)
    ids[0, 0], ids[1, 5], ids[2, :] = V + 5, -7, pad
    ids[3, 1] = pad
    ops.raw_oob_count(reset=True)
    ops.raw_ffm_fwd(W, ids, dense, dense_w, dense_w1, None, pad, D)
    assert ops.raw_oob_count(reset=True) == 2          # counted once per position by the forward
    gy1, gy2 = torch.ones(B, device=DEV), torch.ones(B, device=DEV)
    y1, y2, groups, dW, *_ = _run(W, ids, dense, dense_w, dense_w1, None, gy1, gy2, D, pad=pad)
    U = int(groups.num[0])
    rows = groups.unique_ids[:U]
    assert not bool(((rows == pad) | (rows < 0) | (rows >= V)).any())
    r1, r2, _ = _oracle(W, ids, dense, dense_w, dense_w1, None, gy1, gy2, D, pad=pad)
    m1, m2, _ = _oracle(W, ids, dense, dense_w, dense_w1, None, gy1, gy2, D, pad=pad, absolute=True)
    _within(y1, r1, m1, what="y1")
    _within(y2, r2, m2, what="y2")


def test_ffm_rejects_what_it_cannot_hold():
    from paddlerec_b200 import _lib
    lib = _lib.load()
    W = torch.zeros(10, 2048, device=DEV)
    ids = torch.zeros(4, 40, dtype=torch.int64, device=DEV)
    dense = torch.zeros(4, 30, device=DEV)
    y = torch.zeros(4, device=DEV)
    P = ctypes.c_void_p

    def fwd(F, Dn, D, ldw, w_off=0):
        return lib.b200rec_ffm_fwd(P(W.data_ptr() + w_off), ldw, P(ids.data_ptr()), P(dense.data_ptr()),
                                   P(W.data_ptr()), P(W.data_ptr()), None, P(y.data_ptr()),
                                   P(y.data_ptr()), 4, F, Dn, D, 10, -1, None)
    assert fwd(26, 13, 9, 352) == 0
    torch.cuda.synchronize()
    assert fwd(26, 13, 9, 351) == -1 and b"ldw" in lib.b200rec_last_error()     # no room for w1
    assert fwd(26, 13, 9, 354) == -1                                             # ldw % 4
    assert fwd(26, 13, 9, 352, w_off=4) == -1                                    # W not 16-byte aligned
    assert fwd(40, 30, 1, 2048) == -1 and b"F+Dn" in lib.b200rec_last_error()    # more than 64 fields
    assert fwd(0, 13, 9, 2048) == -1
    assert fwd(26, 13, 0, 2048) == -1
    assert fwd(26, 13, 48, 2048) == -1 and b"shared memory" in lib.b200rec_last_error()
    n = ctypes.c_size_t(0)
    assert lib.b200rec_ffm_bwd_workspace_bytes(4, 26, 13, 9, ctypes.byref(n)) == 0 and n.value > 0
    assert lib.b200rec_ffm_bwd_workspace_bytes(4, 40, 30, 9, ctypes.byref(n)) == -1


# ---- wide rows in the row-wise optimizers -----------------------------------------------------------
@pytest.mark.parametrize("D", [352, 628, 1000])
@pytest.mark.parametrize("opt", ["adam", "sgd"])
def test_wide_row_optimizers_vs_oracle(D, opt):
    from oracle import optim as oopt
    from paddlerec_b200 import ops
    V, n, ldw = 300, 500, D + 12
    g = torch.Generator(device=DEV).manual_seed(D)
    W = torch.randn(V, ldw, device=DEV, generator=g)
    ids = torch.randint(0, V // 2, (n,), device=DEV, generator=g)
    groups = ops.raw_group_ids(ids, V, -1)
    U = int(groups.num[0])
    rows = torch.randn(n, D, device=DEV, generator=g)
    sr = ops.SelectedRows(groups.unique_ids, rows, groups.num, V)
    uniq = groups.unique_ids[:U].cpu().numpy()
    W0 = W.double().cpu().numpy()
    gr = rows[:U].double().cpu().numpy()
    if opt == "adam":
        m = torch.rand(V, ldw, device=DEV, generator=g) * 0.1
        v = torch.rand(V, ldw, device=DEV, generator=g) * 0.1
        m0, v0 = m.double().cpu().numpy(), v.double().cpu().numpy()
        t = 3
        ops.raw_sparse_adam(W, m, v, sr, 1e-2, 0.9, 0.999, 1e-8, 0.9 ** t, 0.999 ** t)
        want, wm, wv = oopt.adam_lazy(W0[:, :D], m0[:, :D], v0[:, :D], uniq, gr, 1e-2, 0.9, 0.999,
                                      1e-8, t)
        np.testing.assert_allclose(m[:, :D].cpu().numpy(), wm, rtol=1e-5, atol=1e-7)
        np.testing.assert_allclose(v[:, :D].cpu().numpy(), wv, rtol=1e-5, atol=1e-7)
        assert torch.equal(m[:, D:], torch.tensor(m0[:, D:], dtype=torch.float32, device=DEV))
    else:
        ops.raw_sparse_sgd(W, sr, 0.05)
        want = oopt.sgd(W0[:, :D], uniq, gr, 0.05)
    np.testing.assert_allclose(W[:, :D].cpu().numpy(), want, rtol=1e-5, atol=1e-6)
    untouched = np.setdiff1d(np.arange(V), uniq)
    assert np.array_equal(W[untouched].cpu().numpy(), W0[untouched].astype(np.float32))
    assert np.array_equal(W[:, D:].cpu().numpy(), W0[:, D:].astype(np.float32))


# ---- one step at the benchmark's size ---------------------------------------------------------------
NS = 512


def test_ffm_full_size_step_on_a_slice_vs_oracle():
    """B=65536, V=1e6, D=16: pred of 512 samples and the gradient rows of every table row only those
    samples touch, against the fp64 oracle; then one lazy Adam step changes only touched rows."""
    from paddlerec_b200 import functional as BF
    from paddlerec_b200 import optim
    from paddlerec_b200.rank.ffm import net
    torch.cuda.empty_cache()
    if torch.cuda.mem_get_info()[0] < 20e9:
        pytest.skip("needs ~12 GB of free HBM")
    B, V, D, F, Dn = 65536, 1_000_000, 16, 26, 13
    torch.manual_seed(1)
    layer = net.FFMLayer(V, D, Dn, F + Dn, device=DEV)
    with torch.no_grad():      # the reference's constant 1.0 saturates the sigmoid (SURVEY.md C)
        layer.ffm.dense_w.normal_(0, 0.05)
        layer.ffm.dense_w_one.normal_(0, 0.05)
    g = torch.Generator(device=DEV).manual_seed(9)
    ids = torch.randint(0, V, (B, F), device=DEV, generator=g)
    ids[:NS:5, 2] = 77
    dense = torch.rand(B, Dn, device=DEV, generator=g)
    label = (torch.rand(B, 1, device=DEV, generator=g) < 0.3).float()
    opt = optim.Adam(learning_rate=1e-3, parameters=layer.parameters())
    pred = layer(ids, dense)
    BF.log_loss_mean(pred, label).backward()
    s = slice(0, NS)
    W = layer.ffm._fused.weight.detach()
    uniq = torch.unique(ids[s])
    remap = torch.searchsorted(uniq, ids[s])
    p = {k: v.detach().double() for k, v in layer.state_dict().items() if not k.startswith("ffm.emb")}
    R = (F + Dn) * D
    p["ffm.embedding.weight"] = W[uniq, :R].double()
    p["ffm.embedding_one.weight"] = W[uniq, R:R + 1].double()
    p = {k: v.requires_grad_(True) for k, v in p.items()}
    from oracle import nets
    from tests import ffm_oracle
    ref = ffm_oracle.ffm_forward(p, [remap[:, i:i + 1] for i in range(F)], dense[s].double(), F + Dn)
    assert elementwise_excess(pred[s], ref) <= 0
    l = nets.log_loss(ref, label[s].double()).sum() / B
    gw = torch.autograd.grad(l, [p["ffm.embedding.weight"]])[0]
    sr = layer.ffm._fused.grad_rows
    U = int(sr.num[0])
    only = ~torch.isin(uniq, ids[NS:])
    assert int(only.sum()) > 1000          # at V=1e6 most of the slice's ids also occur elsewhere
    where = torch.searchsorted(sr.rows[:U].contiguous(), uniq[only])
    assert torch.equal(sr.rows[where], uniq[only])
    assert elementwise_excess(sr.value[where, :R], gw[only]) <= 0
    before = W[:200_000].clone()
    opt.step()
    touched = torch.zeros(200_000, dtype=torch.bool, device=DEV)
    sel = sr.rows[:U]
    touched[sel[sel < 200_000]] = True
    changed = (W[:200_000] != before).any(1)
    assert not bool((changed & ~touched).any()) and float(changed[touched].float().mean()) > 0.99
