"""Parity of every CUDA entry point (called through the C ABI via paddlerec_b200.ops.raw_*) against
the CPU oracle on seeded inputs.  Tolerances: gathers are bit-exact; fp32 reductions are compared
with a float64 oracle at 2e-6 relative to the tensor's max magnitude (fp32 rounding of <=39-term
sums), optimizers at 1e-6."""
import numpy as np
import pytest
import torch

from oracle import nets
from oracle import optim as ooptim
from tests.util import rel_err

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _ops():
    from paddlerec_b200 import ops
    return ops


def make_fm_inputs(B, F, Dn, D, V, seed, pad_frac=0.05, zipf=False):
    g = torch.Generator().manual_seed(seed)
    if zipf:
        r = torch.rand(B, F, generator=g, dtype=torch.float64)
        ids = (V ** r).to(torch.int64).clamp_(1, V - 1)  # heavy duplication on small ids
    else:
        ids = torch.randint(1, V, (B, F), generator=g)
    ids[torch.rand(B, F, generator=g) < pad_frac] = 0
    if B > 1:
        ids[1, :] = 0
    dense = torch.rand(B, Dn, generator=g)
    dense[torch.rand(B, Dn, generator=g) < 0.3] = 0
    W = torch.randn(V, D, generator=g) * 0.1
    W1 = torch.randn(V, 1, generator=g) * 0.1
    dense_w = torch.randn(1, Dn, D, generator=g) * 0.1
    dense_w1 = torch.randn(Dn, generator=g) * 0.1
    return ids, dense, W, W1, dense_w, dense_w1


def oracle_fm(ids, dense, W, W1, dense_w, dense_w1, dtype=torch.float64, pad=0):
    p = {"fm.embedding.weight": W.to(dtype).clone().requires_grad_(True),
         "fm.embedding_one.weight": W1.to(dtype).clone().requires_grad_(True),
         "fm.dense_w": dense_w.to(dtype).clone().requires_grad_(True),
         "fm.dense_w_one": dense_w1.to(dtype).clone().requires_grad_(True)}
    if pad != 0:  # oracle helper hard-codes padding_idx=0 like the reference; remap for other pads
        raise NotImplementedError
    y1, y2, feat = nets.deepfm_fm(p, [ids[:, i:i + 1] for i in range(ids.shape[1])], dense.to(dtype))
    return p, y1, y2, feat


@pytest.mark.parametrize("D", [1, 4, 8, 9, 10, 16, 40, 64, 128])
@pytest.mark.parametrize("B", [1, 7, 300])
def test_embed_fm_fwd(D, B):
    ops = _ops()
    F, Dn, V = 26, 13, 1000
    ids, dense, W, W1, dense_w, dense_w1 = make_fm_inputs(B, F, Dn, D, V, seed=100 + D + B)
    _, y1, y2, feat = oracle_fm(ids, dense, W, W1, dense_w, dense_w1)
    gfeat, gy1, gy2, gS = ops.raw_embed_fm_fwd(W.to(DEV), W1.to(DEV), ids.to(DEV), dense.to(DEV),
                                                dense_w.reshape(Dn, D).to(DEV), dense_w1.to(DEV), 0)
    # gathered rows: bit-exact copies; dense rows: one fp32 multiply, identical to fp32 oracle
    f32 = torch.cat([W[ids] * (ids != 0).unsqueeze(-1), dense.unsqueeze(2) * dense_w], 1)
    assert torch.equal(gfeat.cpu(), f32)
    # fp32 reductions: error bound is relative to the magnitude of the summed terms (a single
    # sample's y2 = 0.5*sum(S^2 - Q) can cancel to ~0)
    scale1 = float((W1[ids].abs().sum((1, 2)) + (dense * dense_w1).abs().sum(1)).max())
    scale2 = float(0.5 * (feat.sum(1).square() + feat.square().sum(1)).sum(1).max())
    assert float((gy1.cpu().double() - y1.reshape(-1)).abs().max()) <= 2e-6 * scale1 + 1e-12
    assert float((gy2.cpu().double() - y2.reshape(-1)).abs().max()) <= 2e-6 * scale2 + 1e-12
    assert rel_err(gS.cpu(), feat.sum(1)) < 2e-6
    assert ops.raw_oob_count() == 0


def test_embed_fm_fwd_odd_fields_and_oob():
    ops = _ops()
    B, F, Dn, D, V = 33, 5, 3, 16, 50
    ids, dense, W, W1, dense_w, dense_w1 = make_fm_inputs(B, F, Dn, D, V, seed=5)
    ids[0, 0] = V + 7      # out of range -> treated as padding, counted
    ids[2, 1] = -3
    ops.raw_oob_count()
    gfeat, gy1, gy2, _ = ops.raw_embed_fm_fwd(W.to(DEV), W1.to(DEV), ids.to(DEV), dense.to(DEV),
                                               dense_w.reshape(Dn, D).to(DEV), dense_w1.to(DEV), 0)
    ids_ok = ids.clone()
    ids_ok[0, 0] = 0
    ids_ok[2, 1] = 0
    _, y1, y2, feat = oracle_fm(ids_ok, dense, W, W1, dense_w, dense_w1)
    assert rel_err(gfeat.cpu(), feat) < 1e-7
    assert rel_err(gy2.cpu(), y2.reshape(-1)) < 2e-6
    assert ops.raw_oob_count() == 2


def test_embed_fm_fwd_empty_batch():
    ops = _ops()
    W = torch.zeros(10, 16, device=DEV)
    W1 = torch.zeros(10, 1, device=DEV)
    feat, y1, y2, S = ops.raw_embed_fm_fwd(W, W1, torch.zeros(0, 26, dtype=torch.int64, device=DEV),
                                           torch.zeros(0, 13, device=DEV),
                                           torch.zeros(13, 16, device=DEV),
                                           torch.zeros(13, device=DEV), 0)
    assert feat.shape == (0, 39, 16) and y1.numel() == 0


@pytest.mark.parametrize("V,n", [(50, 1), (1000, 5000), (100000000, 4096), (5_000_000_000, 3000)])
def test_group_ids(V, n):
    ops = _ops()
    g = torch.Generator().manual_seed(V % 1000 + n)
    ids = torch.randint(0, min(V, 2 ** 62), (n,), generator=g)
    if n > 10:
        ids[::7] = ids[3]          # many duplicates
        ids[5] = 0                  # padding
        ids[6] = V                  # out of range
        ids[8] = -1
    ops.raw_oob_count()
    gr = ops.raw_group_ids(ids.to(DEV), V, 0)
    U, kept = gr.num.cpu().tolist()
    valid = (ids != 0) & (ids >= 0) & (ids < V)
    uniq = torch.unique(ids[valid])
    assert U == uniq.numel() and kept == int(valid.sum())
    assert torch.equal(gr.unique_ids[:U].cpu(), uniq)
    seg = gr.seg_offsets[:U + 1].cpu()
    pos = gr.sorted_pos[:kept].cpu().long()
    assert seg[0] == 0 and seg[-1] == kept
    for u in range(min(U, 200)):
        ps = pos[seg[u]:seg[u + 1]]
        assert (ids[ps] == uniq[u]).all()
        assert (ps[1:] > ps[:-1]).all()  # stable: ascending positions inside a segment
    assert sorted(pos.tolist()) == torch.nonzero(valid).reshape(-1).tolist()


def test_group_ids_all_padding_and_empty():
    ops = _ops()
    gr = ops.raw_group_ids(torch.zeros(17, dtype=torch.int64, device=DEV), 100, 0)
    assert gr.num.cpu().tolist() == [0, 0]
    gr = ops.raw_group_ids(torch.zeros(0, dtype=torch.int64, device=DEV), 100, 0)
    assert gr.num.cpu().tolist() == [0, 0]


@pytest.mark.parametrize("D", [1, 4, 9, 10, 16, 40, 64, 128])
@pytest.mark.parametrize("zipf", [False, True])
def test_embed_fm_bwd(D, zipf):
    ops = _ops()
    B, F, Dn, V = 97, 26, 13, 400
    ids, dense, W, W1, dense_w, dense_w1 = make_fm_inputs(B, F, Dn, D, V, seed=7 + D, zipf=zipf)
    g = torch.Generator().manual_seed(D)
    A = torch.randn(B, F + Dn, D, generator=g)
    g1 = torch.randn(B, generator=g)
    g2 = torch.randn(B, generator=g)
    p, y1, y2, feat = oracle_fm(ids, dense, W, W1, dense_w, dense_w1)
    L = (feat * A.double()).sum() + (y1.reshape(-1) * g1.double()).sum() + \
        (y2.reshape(-1) * g2.double()).sum()
    L.backward()
    gfeat, _, _, gS = ops.raw_embed_fm_fwd(W.to(DEV), W1.to(DEV), ids.to(DEV), dense.to(DEV),
                                           dense_w.reshape(Dn, D).to(DEV), dense_w1.to(DEV), 0)
    gr = ops.raw_group_ids(ids.to(DEV), V, 0)
    dW_rows, dW1_rows, ddw, ddw1 = ops.raw_embed_fm_bwd(gfeat, gS, A.to(DEV), g1.to(DEV),
                                                        g2.to(DEV), dense.to(DEV), gr.seg_offsets,
                                                        gr.sorted_pos, gr.num, F)
    dW = ops.SelectedRows(gr.unique_ids, dW_rows, gr.num, V).to_dense().cpu()
    dW1 = ops.SelectedRows(gr.unique_ids, dW1_rows.unsqueeze(1), gr.num, V).to_dense().cpu()
    assert rel_err(dW, p["fm.embedding.weight"].grad) < 3e-6
    assert rel_err(dW1, p["fm.embedding_one.weight"].grad) < 3e-6
    assert rel_err(ddw.cpu(), p["fm.dense_w"].grad[0]) < 3e-6
    assert rel_err(ddw1.cpu(), p["fm.dense_w_one"].grad) < 3e-6
    assert not dW[0].any() and not dW1[0].any()      # padding row: no gradient
    # deterministic: a second run is bit-identical
    dW_rows2, dW1_rows2, ddw2, _ = ops.raw_embed_fm_bwd(gfeat, gS, A.to(DEV), g1.to(DEV),
                                                        g2.to(DEV), dense.to(DEV), gr.seg_offsets,
                                                        gr.sorted_pos, gr.num, F)
    U = int(gr.num[0])
    assert torch.equal(dW_rows[:U], dW_rows2[:U]) and torch.equal(ddw, ddw2)


@pytest.mark.parametrize("D", [1, 2, 4, 9, 16, 64, 128])
def test_gather_and_segment_reduce(D):
    ops = _ops()
    V, n = 300, 2000
    g = torch.Generator().manual_seed(D)
    W = torch.randn(V, D, generator=g)
    ids = torch.randint(0, V, (n,), generator=g)
    ids[::11] = 3
    out = ops.raw_gather(W.to(DEV), ids.reshape(40, 50).to(DEV), 3)
    ref = W[ids] * (ids != 3).unsqueeze(1)
    assert torch.equal(out.cpu().reshape(n, D), ref)
    out_nopad = ops.raw_gather(W.to(DEV), ids.to(DEV), -1)
    assert torch.equal(out_nopad.cpu(), W[ids])
    dOut = torch.randn(n, D, generator=g)
    gr = ops.raw_group_ids(ids.to(DEV), V, 3)
    rows = ops.raw_segment_reduce(dOut.to(DEV), gr.seg_offsets, gr.sorted_pos, gr.num, n)
    dense = ops.SelectedRows(gr.unique_ids, rows, gr.num, V).to_dense().cpu()
    uniq, merged = ooptim.merge_rows(ids.numpy(), dOut.numpy(), padding_idx=3)
    ref_dense = np.zeros((V, D))
    ref_dense[uniq] = merged
    assert rel_err(dense, ref_dense) < 2e-6


@pytest.mark.parametrize("D", [1, 9, 16, 64])
def test_sparse_optimizers(D):
    ops = _ops()
    V, n = 500, 700
    g = torch.Generator().manual_seed(3 * D)
    W = torch.randn(V, D, generator=g)
    ids = torch.randint(1, V, (n,), generator=g)
    dOut = torch.randn(n, D, generator=g)
    uniq, merged = ooptim.merge_rows(ids.numpy(), dOut.numpy())

    def selected():
        gr = ops.raw_group_ids(ids.to(DEV), V, -1)
        rows = ops.raw_segment_reduce(dOut.to(DEV), gr.seg_offsets, gr.sorted_pos, gr.num, n)
        return ops.SelectedRows(gr.unique_ids, rows, gr.num, V)

    # SGD
    Wd = W.to(DEV).clone()
    ops.raw_sparse_sgd(Wd, selected(), 0.1)
    assert rel_err(Wd.cpu(), ooptim.sgd(W.double().numpy(), uniq, merged, 0.1)) < 1e-6
    # lazy Adam, two steps
    Wd = W.to(DEV).clone()
    m = torch.zeros_like(Wd)
    v = torch.zeros_like(Wd)
    Wr, mr, vr = W.double().numpy(), np.zeros((V, D)), np.zeros((V, D))
    for t in (1, 2):
        ops.raw_sparse_adam(Wd, m, v, selected(), 1e-3, 0.9, 0.999, 1e-8, 0.9 ** t, 0.999 ** t)
        Wr, mr, vr = ooptim.adam_lazy(Wr, mr, vr, uniq, merged, 1e-3, 0.9, 0.999, 1e-8, t)
    assert rel_err(Wd.cpu(), Wr) < 1e-6 and rel_err(m.cpu(), mr) < 1e-6 and rel_err(v.cpu(), vr) < 1e-6
    untouched = np.setdiff1d(np.arange(V), uniq)
    assert torch.equal(Wd.cpu()[untouched], W[untouched])   # lazy: other rows untouched
    # row-wise AdaGrad
    Wd = W.to(DEV).clone()
    g2 = torch.zeros(V, device=DEV)
    Wr, g2r = W.double().numpy(), np.zeros(V)
    for _ in range(2):
        ops.raw_sparse_adagrad(Wd, g2, selected(), 0.05, 3.0, -10.0, 10.0)
        Wr, g2r = ooptim.adagrad_row(Wr, g2r, uniq, merged, 0.05, 3.0, -10.0, 10.0)
    assert rel_err(Wd.cpu(), Wr) < 1e-6 and rel_err(g2.cpu(), g2r) < 1e-6


@pytest.mark.parametrize("C", [156, 351, 1560])
def test_cross_v2(C):
    ops = _ops()
    B = 77
    g = torch.Generator().manual_seed(C)
    x0, xl, xw, dout = (torch.randn(B, C, generator=g) for _ in range(4))
    bias = torch.randn(C, generator=g)
    out = ops.raw_cross_v2_fwd(x0.to(DEV), xl.to(DEV), xw.to(DEV), bias.to(DEV))
    assert rel_err(out.cpu(), xl.double() + x0.double() * (xw.double() + bias.double())) < 1e-6
    dxw, dx0, dbias = ops.raw_cross_v2_bwd(dout.to(DEV), x0.to(DEV), xw.to(DEV), bias.to(DEV))
    assert rel_err(dxw.cpu(), dout.double() * x0.double()) < 1e-6
    assert rel_err(dx0.cpu(), dout.double() * (xw.double() + bias.double())) < 1e-6
    assert rel_err(dbias.cpu(), (dout.double() * x0.double()).sum(0)) < 2e-6


@pytest.mark.parametrize("world,n,only_owner", [
    pytest.param(1, 5000, None, id="1"),
    pytest.param(2, 5000, None, id="2"),
    pytest.param(8, 5000, None, id="8"),
    # the radix sort runs over ceil(log2(world)) bits (shard.cuh:54-55): not log2(world) for 3 and 5
    pytest.param(3, 5000, None, id="3"),
    pytest.param(5, 5000, None, id="5"),
    pytest.param(16, 5000, None, id="16"),
    pytest.param(4, 0, None, id="4-empty"),
    pytest.param(5, 5000, 3, id="5-one-owner"),
    pytest.param(16, 1_700_000, None, id="16-1.7M"),
])
def test_shard_bucketize(world, n, only_owner):
    ops = _ops()
    V = 1000
    g = torch.Generator().manual_seed(world + n)
    if only_owner is None:
        ids = torch.randint(0, V, (n,), generator=g)
        if n > 11:
            ids[10] = -5
            ids[11] = V + 1
    else:
        ids = torch.randint(0, V // world, (n,), generator=g) * world + only_owner
    send, perm, inv, counts = ops.raw_shard_bucketize(ids.to(DEV), world, V)
    send, perm, inv, counts = send.cpu(), perm.cpu(), inv.cpu().long(), counts.cpu()
    valid = (ids >= 0) & (ids < V)
    owner = torch.where(valid, ids % world, torch.zeros_like(ids))
    assert counts.tolist() == [int((owner == r).sum()) for r in range(world)]
    if only_owner is not None:
        assert counts.tolist() == [n if r == only_owner else 0 for r in range(world)]
    assert torch.equal(perm[inv], torch.arange(n))            # inverse permutations
    assert (owner[inv][1:] >= owner[inv][:-1]).all()          # bucket order is owner-major
    off = 0
    for r in range(world):                                    # stable inside a bucket
        seg = inv[off:off + int(counts[r])]
        assert (seg[1:] > seg[:-1]).all()
        off += int(counts[r])
    local = torch.where(valid, ids // world, torch.full_like(ids, -1))
    assert torch.equal(send, local[inv])


@pytest.mark.parametrize("K,N", [(624, 400), (351, 7), (400, 1)])
def test_tower_epilogues(K, N):
    ops = _ops()
    M = 333
    g = torch.Generator().manual_seed(K + N)
    x = torch.randn(M, K, generator=g)
    bias = torch.randn(K, generator=g)
    out = ops.raw_tower_split(x.to(DEV), bias.to(DEV), True).cpu().float()
    ref = torch.relu(x + bias)
    hi = ref.to(torch.bfloat16)
    lo = (ref - hi.float()).to(torch.bfloat16)
    assert torch.equal(out[:, :K], hi.float()) and torch.equal(out[:, K:], lo.float())
    assert rel_err(out[:, :K] + out[:, K:], ref) < 2 ** -15
    out2 = ops.raw_tower_split(x.to(DEV), None, False).cpu().float()
    assert rel_err(out2[:, :K] + out2[:, K:], x) < 2 ** -15
    # backward epilogue
    dy = torch.randn(M, K, generator=g)
    dz, db = ops.raw_tower_relu_bwd_split(dy.to(DEV), ops.raw_tower_split(x.to(DEV), bias.to(DEV), True))
    dz = dz.cpu().float()
    dz_ref = dy * (hi.float() > 0)
    assert rel_err(dz[:, :K] + dz[:, K:], dz_ref) < 2 ** -15
    assert rel_err(db.cpu(), dz_ref.double().sum(0)) < 2e-6
    dz2, db2 = ops.raw_tower_relu_bwd_split(dy.to(DEV), None)
    assert rel_err(db2.cpu(), dy.double().sum(0)) < 2e-6
    # weight operand layouts + dW folding
    W = torch.randn(K, N, generator=g)
    W2r, W2c, Wlo = (t.cpu().float() for t in ops.raw_tower_prep_weight(W.to(DEV)))
    whi = W.to(torch.bfloat16).float()
    assert torch.equal(W2r[:K], whi) and torch.equal(W2r[K:], whi)
    assert torch.equal(W2c[:, :N], whi) and torch.equal(W2c[:, N:], whi)
    assert torch.equal(Wlo, (W - whi).to(torch.bfloat16).float())
    Mx = torch.randn(2 * K, 2 * N, generator=g)
    dW = ops.raw_tower_fold_dw(Mx.to(DEV), K, N).cpu()
    assert rel_err(dW, Mx[:K, :N] + Mx[:K, N:] + Mx[K:, :N]) < 1e-6


@pytest.mark.parametrize("last_act", [False, True])
def test_tower_mlp_matches_fp64(last_act):
    from paddlerec_b200 import tower
    g = torch.Generator().manual_seed(11)
    M, sizes = 257, [624, 400, 400, 1]
    x = torch.randn(M, sizes[0], generator=g)
    Ws = [torch.randn(sizes[i], sizes[i + 1], generator=g) / sizes[i] ** 0.5 for i in range(3)]
    bs = [torch.randn(sizes[i + 1], generator=g) * 0.1 for i in range(3)]
    xd = x.double().requires_grad_(True)
    Wd = [w.double().requires_grad_(True) for w in Ws]
    bd = [b.double().requires_grad_(True) for b in bs]
    h = xd
    for i in range(3):
        h = h @ Wd[i] + bd[i]
        if i < 2 or last_act:
            h = torch.relu(h)
    gy = torch.randn(M, 1, generator=g)
    (h * gy.double()).sum().backward()
    xc = x.to(DEV).requires_grad_(True)
    Wc = [w.to(DEV).requires_grad_(True) for w in Ws]
    bc = [b.to(DEV).requires_grad_(True) for b in bs]
    y = tower.mlp(xc, Wc, bc, last_act=last_act)
    (y * gy.to(DEV)).sum().backward()
    assert rel_err(y, h) < 1e-4
    assert rel_err(xc.grad, xd.grad) < 1e-4
    for a, b in zip(Wc + bc, Wd + bd):
        assert rel_err(a.grad, b.grad) < 1e-4


@pytest.mark.parametrize("D", [4, 9, 16])
def test_fused_slot_layout_equals_two_tables(D):
    """The fused slot layout ([D emb | w1 | pad] per 128-byte row) must give exactly the
    same forward and the same gradients as the reference's two-table layout."""
    ops = _ops()
    B, F, Dn, V = 65, 26, 13, 300
    ids, dense, W, W1, dense_w, dense_w1 = make_fm_inputs(B, F, Dn, D, V, seed=40 + D, zipf=True)
    slot, G = ops.fused_slot(D), ops.fused_grad_cols(D)
    assert slot == 32 and G % 4 == 0 and G >= D + 1
    Wf = torch.zeros(V, slot)
    Wf[:, :D] = W
    Wf[:, D] = W1[:, 0]
    Wf[:, D + 1:] = 123.0          # pad columns must never be read
    args = (ids.to(DEV), dense.to(DEV), dense_w.reshape(Dn, D).to(DEV), dense_w1.to(DEV), 0)
    f0, y10, y20, S0 = ops.raw_embed_fm_fwd(W.to(DEV), W1.to(DEV), *args)
    f1, y11, y21, S1 = ops.raw_embed_fm_fwd(Wf.to(DEV), None, *args, D=D)
    assert torch.equal(f0, f1) and torch.equal(y10, y11) and torch.equal(y20, y21)
    g = torch.Generator().manual_seed(D)
    A = torch.randn(B, F + Dn, D, generator=g).to(DEV)
    g1 = torch.randn(B, generator=g).to(DEV)
    g2 = torch.randn(B, generator=g).to(DEV)
    gr = ops.raw_group_ids(ids.to(DEV), V, 0)
    common = (f0, S0, A, g1, g2, dense.to(DEV), gr.seg_offsets, gr.sorted_pos, gr.num, F)
    dW, dW1, ddw, ddw1 = ops.raw_embed_fm_bwd(*common)
    dWf, none, ddwf, _ = ops.raw_embed_fm_bwd(*common, fused_cols=G)
    U = int(gr.num[0])
    assert none is None and dWf.shape[1] == G
    assert torch.equal(dWf[:U, :D], dW[:U]) and torch.equal(dWf[:U, D], dW1[:U])
    assert not dWf[:U, D + 1:].any() and torch.equal(ddw, ddwf)
    # gather of the first G columns of a slot table; optimizer on slots == optimizer on two tables
    rows = ops.raw_gather(Wf.to(DEV), ids.to(DEV), 0, D=G)
    ref = Wf[ids][..., :G] * (ids != 0).unsqueeze(-1)
    assert torch.equal(rows.cpu(), ref)
    sr_f = ops.SelectedRows(gr.unique_ids, dWf, gr.num, V, ncols=G)
    Wd, md, vd = Wf.to(DEV).clone(), torch.zeros(V, slot, device=DEV), torch.zeros(V, slot, device=DEV)
    ops.raw_sparse_adam(Wd, md, vd, sr_f, 1e-2, 0.9, 0.999, 1e-8, 0.9, 0.999)
    Wa, ma, va = W.to(DEV).clone(), torch.zeros(V, D, device=DEV), torch.zeros(V, D, device=DEV)
    ops.raw_sparse_adam(Wa, ma, va, ops.SelectedRows(gr.unique_ids, dW, gr.num, V), 1e-2, 0.9, 0.999,
                        1e-8, 0.9, 0.999)
    Wb, mb, vb = W1.to(DEV).clone(), torch.zeros(V, 1, device=DEV), torch.zeros(V, 1, device=DEV)
    ops.raw_sparse_adam(Wb, mb, vb, ops.SelectedRows(gr.unique_ids, dW1.unsqueeze(1), gr.num, V),
                        1e-2, 0.9, 0.999, 1e-8, 0.9, 0.999)
    assert torch.equal(Wd[:, :D], Wa) and torch.equal(Wd[:, D:D + 1], Wb)
    assert (Wd[:, G:] == 123.0).all()               # slot padding beyond the gradient columns untouched
    dense_grad = sr_f.to_dense()
    assert dense_grad.shape == (V, G) and not dense_grad[0].any()


@pytest.mark.parametrize("B,L,E", [(1, 1, 16), (5, 7, 16), (3, 100, 128), (2, 152, 128), (70, 13, 64)])
def test_din_attention_fused_forward_and_grads(B, L, E):
    """K4 against the reference's op sequence (din/net.py:155-173) in float64; the autograd node
    (fused forward, composite backward) must also give the right gradients."""
    ops = _ops()
    g = torch.Generator().manual_seed(B * 1000 + L + E)
    hist = torch.randn(B, L, E, generator=g) * 0.5
    tseq = torch.randn(B, E, generator=g) * 0.5
    lens = torch.randint(1, L + 1, (B,), generator=g)
    lens[0] = L
    mask = torch.zeros(B, L, 1, dtype=torch.int64)
    for b in range(B):
        mask[b, int(lens[b]):] = int(-1e9)
    W1 = torch.randn(4 * E, 80, generator=g) / (4 * E) ** 0.5
    b1 = torch.randn(80, generator=g) * 0.1
    W2 = torch.randn(80, 40, generator=g) / 80 ** 0.5
    b2 = torch.randn(40, generator=g) * 0.1
    W3 = torch.randn(40, 1, generator=g) / 40 ** 0.5
    b3 = torch.randn(1, generator=g) * 0.1
    params = [W1, b1, W2, b2, W3, b3]
    ref_in = [t.double().requires_grad_(True) for t in [hist, tseq] + params]
    ref = nets.din_attention_unit(ref_in[0], ref_in[1], mask, *ref_in[2:])
    gout = torch.randn(B, E, generator=g)
    (ref * gout.double()).sum().backward()
    dev_in = [t.to(DEV).requires_grad_(True) for t in [hist, tseq] + params]
    out = ops.din_attention(dev_in[0], dev_in[1], mask.to(DEV), *dev_in[2:])
    assert rel_err(out, ref) < 2e-5
    out_nomask = ops.raw_din_attn_fwd(hist.to(DEV), tseq.to(DEV), None, *[p.to(DEV) for p in params])[0]
    ref_nomask = nets.din_attention_unit(hist.double(), tseq.double(), None,
                                         *[p.double() for p in params])
    assert rel_err(out_nomask, ref_nomask) < 2e-5
    (out * gout.to(DEV)).sum().backward()
    for a, b in zip(dev_in, ref_in):
        if float(b.grad.abs().max()) < 1e-12:
            assert float(a.grad.abs().max()) < 1e-6
        else:
            assert rel_err(a.grad, b.grad) < 1e-4
    w = ops.raw_din_attn_fwd(hist.to(DEV), tseq.to(DEV), mask.to(DEV), *[p.to(DEV) for p in params])[1]
    assert rel_err(w.sum(1).cpu(), torch.ones(B)) < 1e-5
    for b in range(B):
        assert float(w[b, int(lens[b]):].abs().sum()) == 0.0     # masked positions get zero weight


@pytest.mark.parametrize("use_cvm", [False, True])
def test_cvm(use_cvm):
    """continuous_value_model against oracle/nets.py:cvm (forward) and Paddle's documented
    cvm_grad semantics (show/click written into the first two gradient columns)."""
    ops = _ops()
    N, D = 1000, 11
    g = torch.Generator().manual_seed(3)
    x = torch.rand(N, D + 2, generator=g) * 5
    sc = torch.rand(N, 2, generator=g) * 3
    xd = x.to(DEV).requires_grad_(True)
    y = ops.continuous_value_model(xd, sc.to(DEV), use_cvm)
    ref = nets.cvm(x.double(), use_cvm)
    assert y.shape == ref.shape and rel_err(y, ref) < 1e-6
    dy = torch.randn(y.shape, generator=g)
    y.backward(dy.to(DEV))
    dx = xd.grad.cpu()
    assert torch.equal(dx[:, :2], sc)
    assert torch.equal(dx[:, 2:], dy[:, 2:] if use_cvm else dy)


@pytest.mark.parametrize("D", [8, 9, 16, 64])
def test_gather_pool_sum_lod(D):
    """Multi-hot slots: sum-pooled lookups over LoD key lists (empty bags, padding keys, hot keys)
    and their backward through the shared segmented reduce."""
    from paddlerec_b200 import nn as bnn
    ops = _ops()
    V, n_bags = 200, 300
    g = torch.Generator().manual_seed(D)
    lens = torch.randint(0, 6, (n_bags,), generator=g)
    lens[5] = 0
    lens[7] = 150                                   # one long bag
    offsets = torch.zeros(n_bags + 1, dtype=torch.int64)
    offsets[1:] = torch.cumsum(lens, 0)
    nnz = int(offsets[-1])
    keys = torch.randint(0, V, (nnz,), generator=g)
    keys[::9] = 17                                   # a hot key (>64 occurrences)
    emb = bnn.Embedding(V, D, padding_idx=0, init_std=0.1, device=DEV)
    W = emb.weight.detach().cpu().double()
    out = emb.forward_pooled(keys.to(DEV), offsets.to(DEV))
    ref = torch.zeros(n_bags, D, dtype=torch.float64)
    Wr = W.clone().requires_grad_(True)
    rows = Wr[keys] * (keys != 0).unsqueeze(1)
    ref = torch.zeros(n_bags, D, dtype=torch.float64).index_add(
        0, torch.repeat_interleave(torch.arange(n_bags), lens), rows)
    assert rel_err(out, ref) < 2e-6 and not out[5].any()
    gout = torch.randn(n_bags, D, generator=g)
    (out * gout.to(DEV)).sum().backward()
    (ref * gout.double()).sum().backward()
    assert rel_err(emb.grad_rows.to_dense(), Wr.grad) < 3e-6


# ---- uint64 feasigns -> rows (E2 / §8(f) row 2) ---------------------------------------------------
@pytest.mark.parametrize("V,reserve_zero", [(1000001, True), (2, True), (1, False), (10**8, False),
                                            ((1 << 40) + 7, True)])
def test_hash_keys_bit_exact(V, reserve_zero):
    from oracle import readers

    ops = _ops()
    rng = np.random.default_rng(V % 97)
    n = 100003
    keys = rng.integers(0, 1 << 63, n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, n, dtype=np.uint64)
    keys[:5] = np.array([0, 1, (1 << 64) - 1, 1 << 63, 0], np.uint64)
    slots = rng.integers(0, 26, n).astype(np.int32)
    for sl in (None, slots):
        want = readers.hash_keys(keys, V, sl, reserve_zero)
        got = ops.raw_hash_keys(torch.from_numpy(keys).to(DEV), V,
                                None if sl is None else torch.from_numpy(sl).to(DEV), reserve_zero)
        assert got.dtype == torch.int64 and got.shape == (n,)
        assert np.array_equal(got.cpu().numpy(), want)
        assert want.min() >= 0 and want.max() < V
        if reserve_zero:
            assert (want[keys == 0] == 0).all() and (want[keys != 0] >= 1).all()
    # int64 tensors holding the same bits give the same rows; shape is preserved
    as_i64 = torch.from_numpy(keys.view(np.int64)).to(DEV).reshape(-1, 1)[: n - 3]
    got2 = ops.raw_hash_keys(as_i64, V, None, reserve_zero)
    assert got2.shape == as_i64.shape
    assert np.array_equal(got2.cpu().numpy()[:, 0], readers.hash_keys(keys[: n - 3], V, None, reserve_zero))


def test_hash_keys_feeds_the_gather_and_spreads_uniformly():
    """Hashed multi-slot lookup end to end: parse -> fold on the device -> gather; and the fold's
    occupancy over V rows is that of a uniform hash (no slot aliasing)."""
    from oracle import readers

    ops = _ops()
    V, D, n = 4096, 16, 1 << 18
    rng = np.random.default_rng(7)
    raw = rng.integers(1, 5000, n).astype(np.uint64)          # small raw ids, as in real logs
    slots = rng.integers(0, 26, n).astype(np.int32)
    rows = ops.raw_hash_keys(torch.from_numpy(raw).to(DEV), V, torch.from_numpy(slots).to(DEV), True)
    assert np.array_equal(rows.cpu().numpy(), readers.hash_keys(raw, V, slots, True))
    counts = torch.bincount(rows, minlength=V).double()[1:]
    distinct = len(set(zip(raw.tolist(), slots.tolist())))
    # balls-in-bins: expected empty fraction exp(-distinct/(V-1)); none here, and max load bounded
    assert (counts == 0).float().mean() < 0.01 and counts.max() < 12 * n / (V - 1)
    assert distinct > 100000
    W = torch.randn(V, D, device=DEV)
    W[0] = 0
    out = ops.raw_gather(W, rows, 0)
    assert torch.equal(out, W[rows])


def test_hash_keys_rejects_bad_arguments():
    ops = _ops()
    from paddlerec_b200._lib import B200RecError

    k = torch.zeros(4, dtype=torch.uint64, device=DEV)
    with pytest.raises(B200RecError, match="too small"):
        ops.raw_hash_keys(k, 1, None, True)
    with pytest.raises(TypeError):
        ops.raw_hash_keys(k.to(torch.float32), 10)
    with pytest.raises(B200RecError, match="CUDA"):
        ops.raw_hash_keys(torch.zeros(4, dtype=torch.int64), 10)
    assert ops.raw_hash_keys(k[:0], 10).numel() == 0


# ---- K6: DLRM dot interaction ----------------------------------------------------------------------
@pytest.mark.parametrize("B,N,d", [(1, 2, 1), (5, 5, 3), (33, 27, 16), (1000, 27, 16), (7, 27, 9),
                                   (64, 40, 64), (9, 27, 128), (3, 128, 4)])
@pytest.mark.parametrize("self_interaction", [False, True])
def test_dot_interact_fwd_bwd(B, N, d, self_interaction):
    ops = _ops()
    g = torch.Generator().manual_seed(B * 1000 + N * 10 + d)
    T = torch.randn(B, N, d, generator=g, dtype=torch.float64)
    Tref = T.clone().requires_grad_(True)
    Rref = nets.dot_interact(Tref, self_interaction)
    dR = torch.randn(Rref.shape, generator=g, dtype=torch.float64)
    Rref.backward(dR)
    Tg = T.to(torch.float32).to(DEV).requires_grad_(True)
    R = ops.dot_interact(Tg, self_interaction)
    assert R.shape == Rref.shape == (B, ops.dot_interact_width(N, d, self_interaction))
    R.backward(dR.to(torch.float32).to(DEV))
    # d-term fp32 dot products vs float64: 2e-6 of the largest magnitude
    assert rel_err(R, Rref) < 2e-6
    assert rel_err(Tg.grad, Tref.grad) < 2e-6
    assert torch.equal(R[:, :d], Tg.detach()[:, N - 1])          # the x block is a copy
    if self_interaction:
        iu = torch.triu_indices(N, N, 0)
        assert (R[:, d:][:, (iu[0] == iu[1]).to(DEV)] == 0).all()  # the reference's zero diagonal
    # deterministic: no atomics anywhere
    R2 = ops.raw_dot_interact_fwd(Tg.detach(), self_interaction)
    dT2 = ops.raw_dot_interact_bwd(Tg.detach(), dR.to(torch.float32).to(DEV), self_interaction)
    assert torch.equal(R2, R.detach()) and torch.equal(dT2, Tg.grad)


def test_dot_interact_rejects_bad_shapes():
    ops = _ops()
    from paddlerec_b200._lib import B200RecError

    with pytest.raises(B200RecError, match="bad sizes"):
        ops.raw_dot_interact_fwd(torch.zeros(2, 1, 4, device=DEV))            # N < 2
    with pytest.raises(B200RecError, match="bad sizes"):
        ops.raw_dot_interact_fwd(torch.zeros(2, 129, 4, device=DEV))
    with pytest.raises(ValueError):
        ops.raw_dot_interact_bwd(torch.zeros(2, 3, 4, device=DEV), torch.zeros(2, 5, device=DEV))
    assert ops.raw_dot_interact_fwd(torch.zeros(0, 3, 4, device=DEV)).shape == (0, 7)


@pytest.mark.skipif(__import__("os").environ.get("B200REC_TEST_EXPERIMENTAL") != "1",
                    reason="experimental K6 v2 kernels: opt in with B200REC_TEST_EXPERIMENTAL=1")
@pytest.mark.parametrize("B,N,d", [(1, 2, 4), (33, 27, 16), (1000, 27, 16), (64, 40, 64), (9, 27, 128),
                                   (3, 128, 4), (5000, 27, 8)])
@pytest.mark.parametrize("self_interaction", [False, True])
def test_dot_interact_v2_matches_v1(B, N, d, self_interaction, monkeypatch):
    """The float4 / cp.async variant (B200REC_K6_V2=1) against the validated default: forward
    bit-identical (same products in the same order), backward too (same j order per output)."""
    ops = _ops()
    g = torch.Generator().manual_seed(B + N + d)
    T = torch.randn(B, N, d, generator=g).to(DEV)
    dR = torch.randn(B, ops.dot_interact_width(N, d, self_interaction), generator=g).to(DEV)
    monkeypatch.delenv("B200REC_K6_V2", raising=False)
    R1 = ops.raw_dot_interact_fwd(T, self_interaction)
    dT1 = ops.raw_dot_interact_bwd(T, dR, self_interaction)
    monkeypatch.setenv("B200REC_K6_V2", "1")
    R2 = ops.raw_dot_interact_fwd(T, self_interaction)
    dT2 = ops.raw_dot_interact_bwd(T, dR, self_interaction)
    assert torch.equal(R1, R2)
    assert torch.equal(dT1, dT2)


def test_embedding_used_twice_merges_selected_rows():
    """ADVICE r1: Paddle merge-adds the SelectedRows gradients of a table that is looked up twice
    in one forward (shared embedding) or across micro-batches; the table gradient must equal the
    dense autograd gradient of the same computation."""
    from paddlerec_b200 import nn as bnn
    g = torch.Generator().manual_seed(5)
    V, D = 97, 8
    emb = bnn.Embedding(V, D, padding_idx=0, init_std=0.1, device=DEV)
    ids1 = torch.randint(0, V, (33, 4), generator=g).to(DEV)
    ids2 = torch.randint(0, V, (20, 3), generator=g).to(DEV)
    w1 = torch.randn(33, 4, D, generator=g).to(DEV)
    w2 = torch.randn(20, 3, D, generator=g).to(DEV)
    ((emb(ids1) * w1).sum() + (emb(ids2) * w2).sum()).backward()
    got = emb.grad_rows.to_dense()
    Wd = emb.weight.detach().double().clone().requires_grad_(True)
    m1 = (ids1 != 0).unsqueeze(2)
    m2 = (ids2 != 0).unsqueeze(2)
    ((Wd[ids1] * m1 * w1.double()).sum() + (Wd[ids2] * m2 * w2.double()).sum()).backward()
    assert rel_err(got, Wd.grad) < 1e-6
    assert not got[0].any()


def test_auc_update_kernel_matches_host_metric():
    """b200rec_auc_update (device histograms, one launch) == the torch bucketing of functional.Auc
    on the CPU, and the AUC itself against sklearn's exact value."""
    from sklearn.metrics import roc_auc_score
    from paddlerec_b200 import functional as BF
    g = torch.Generator().manual_seed(17)
    n = 50000
    y = (torch.rand(n, generator=g) < 0.3).long()
    p = (torch.rand(n, generator=g) * 0.6 + 0.3 * y.float() * torch.rand(n, generator=g)).clamp(0, 1)
    p[0], p[1] = 0.0, 1.0
    dev, host = BF.Auc(), BF.Auc()
    for lo in range(0, n, 12500):
        dev.update(p[lo:lo + 12500].to(DEV).reshape(-1, 1), y[lo:lo + 12500].to(DEV).reshape(-1, 1))
        host.update(p[lo:lo + 12500].reshape(-1, 1), y[lo:lo + 12500].reshape(-1, 1))
    assert torch.equal(dev.stats()[0].cpu(), host.stats()[0])
    assert torch.equal(dev.stats()[1].cpu(), host.stats()[1])
    assert abs(dev.accumulate() - roc_auc_score(y.numpy(), p.numpy())) < 2e-3
