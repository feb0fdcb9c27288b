"""The peer-memory shard exchange (csrc/shard.cuh) on ONE GPU: W virtual ranks, checked bit for bit
against the single-GPU path.

The three peer-memory kernels (shard_gather_push, shard_push_rows, shard_fm_grads_push) only store
through the base pointers of their PeerTable.  Here the receive buffers of all virtual ranks are
slices of ONE device tensor, so the real kernels run the whole pull and push exactly as they would
over NVLink, at every world size up to kMaxPeers, and the single-GPU kernels give an exact reference.

The segment tables are built here, NOT by ShardExchange._bucketize_and_count (they are what is under
test): the per-rank count matrix C[r, o] comes from the real raw_shard_bucketize, and every
all_to_all_single of the count exchange becomes an in-process transpose:
    send_seg_r = [0, cumsum C[r]]            recv_counts_o[r] = C[r, o]
    dst_pull_o[r] = send_seg_r[o]            recv_seg_o = [0, cumsum recv_counts_o]
    dst_push_r[o] = recv_seg_o[r]            recv_ids_o = cat_r send_ids_r[send_seg_r[o]:send_seg_r[o+1]]

Every receive buffer is filled with a NaN sentinel before a step; afterwards every guard row and every
element a rank should not have received must still hold the sentinel bits.  One stream orders all
calls, so the publishing barriers of PeerBuffers are no-ops here.
"""
import ctypes

import pytest
import torch

from tests.test_gpu_at_scale import U, assert_loops, assert_within, row_shape, seg_chain

pytestmark = pytest.mark.gpu

DEV = "cuda"
SENT = 0x7FC0FFEE          # quiet-NaN bit pattern of the untouched buffer memory
GUARD = 3                  # sentinel rows between two receive buffers

# ---- C++ constants mirrored here (file:line of the definition) ---------------------------------
PUSH_THREADS = 256         # shard.cuh:116 kPushThreads
MAX_PEERS = 16             # shard.cuh:118 kMaxPeers
FUSED_PUSH_CTAS_PER_SM = 32  # shard.cuh:361 grid = min(ceil(n*G/4/256), 32*SM)
HOT_THRESHOLD = 64         # segreduce.cuh:26 kHotThreshold


def _ops():
    from paddlerec_b200 import ops
    return ops


def _sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cdiv(a, b):
    return -(-a // b)


@pytest.fixture(autouse=True)
def hbm_budget(request):
    """The largest case (4 ranks of 65536 x 26 slots) needs a few GB; skip when the shared GPU has
    less free."""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < 8e9:
        pytest.skip("needs ~8 GB of free HBM (%.1f GB free)" % (free / 1e9))
    torch.cuda.reset_peak_memory_stats()
    yield
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    print("[peak] %s: %.2f GB" % (request.node.name, peak / 1e9))
    assert peak <= 6e9, "%s allocated %.1f GB" % (request.node.name, peak / 1e9)


@pytest.fixture(autouse=True)
def clear_oob_count():
    """These tests feed out-of-range ids on purpose.  The library counts them in one global counter
    that other tests expect to find at zero, so reset it after each test."""
    yield
    _ops().raw_oob_count(reset=True)


# ---- harness --------------------------------------------------------------------------------------
def _ptr_array(ptrs):
    return (ctypes.c_uint64 * len(ptrs))(*ptrs)


class _Arena:
    """Receive buffers of `world` virtual ranks in ONE tensor of row pitch `cols`: per rank
    [guard | rows (cap) | guard | grads (cap_g)], then a last guard."""

    def __init__(self, world, cap, cap_g, cols):
        self.world, self.cap, self.cap_g, self.cols = world, cap, cap_g, cols
        per = GUARD + cap + GUARD + cap_g
        self.buf = torch.empty(world * per + GUARD, cols, device=DEV)
        self.rows_at = [GUARD + r * per for r in range(world)]
        self.grads_at = [a + cap + GUARD for a in self.rows_at]
        base, pitch = self.buf.data_ptr(), cols * 4
        self.rows_ptrs = _ptr_array([base + a * pitch for a in self.rows_at])
        self.grads_ptrs = _ptr_array([base + a * pitch for a in self.grads_at])

    def rows(self, r):
        return self.buf[self.rows_at[r]:self.rows_at[r] + self.cap]

    def grads(self, r):
        return self.buf[self.grads_at[r]:self.grads_at[r] + self.cap_g]

    def fill(self):
        self.buf.view(torch.int32).fill_(SENT)

    def check_untouched(self, rows_written, grads_written, width):
        """Only the first rows_written[r] / grads_written[r] rows of each buffer, first `width`
        columns, may have been stored to."""
        may = torch.zeros(self.buf.shape, dtype=torch.bool, device=DEV)
        for r in range(self.world):
            may[self.rows_at[r]:self.rows_at[r] + rows_written[r], :width] = True
            may[self.grads_at[r]:self.grads_at[r] + grads_written[r], :width] = True
        bad = (self.buf.view(torch.int32) != SENT) & ~may
        if bool(bad.any()):
            i = int(bad.reshape(-1).nonzero()[0])
            raise AssertionError("store outside the receive segments: %d elements, first at row %d "
                                 "col %d" % (int(bad.sum()), i // self.cols, i % self.cols))


class _DevicePeer:
    """Stands in for sharded.PeerBuffers: rank `rank`'s view of an _Arena.  All ranks run on one
    stream, so publishing needs no barrier."""

    def __init__(self, arena, rank):
        self.cap, self.cap_g, self.cols, self.world = arena.cap, arena.cap_g, arena.cols, arena.world
        self.rows, self.grads = arena.rows(rank), arena.grads(rank)
        self.rows_ptrs, self.grads_ptrs = arena.rows_ptrs, arena.grads_ptrs

    def publish_rows(self):
        pass

    def publish_grads(self):
        pass


class _Plans:
    """ExchangePlans of every virtual rank plus the host copies of the segment tables."""

    def __init__(self, ids_per_rank, world, V):
        from paddlerec_b200 import sharded
        ops = _ops()
        outs = [ops.raw_shard_bucketize(ids.reshape(-1), world, V) for ids in ids_per_rank]
        C = torch.stack([o[3] for o in outs]).cpu()                # C[r, o]
        zero = torch.zeros(1, dtype=torch.int64)
        self.world = world
        self.send_seg = [torch.cat([zero, C[r].cumsum(0)]).tolist() for r in range(world)]
        self.recv_seg = [torch.cat([zero, C[:, o].cumsum(0)]).tolist() for o in range(world)]
        self.n = [int(ids.numel()) for ids in ids_per_rank]
        self.m = [s[-1] for s in self.recv_seg]
        self.plans = []
        for x in range(world):
            recv_ids = torch.cat([outs[r][0][self.send_seg[r][x]:self.send_seg[r][x + 1]]
                                  for r in range(world)])
            tables = {"send_seg": torch.tensor(self.send_seg[x], device=DEV),
                      "recv_seg": torch.tensor(self.recv_seg[x], device=DEV),
                      "dst_pull": torch.tensor([self.send_seg[r][x] for r in range(world)],
                                               device=DEV),
                      "dst_push": torch.tensor([self.recv_seg[o][x] for o in range(world)],
                                               device=DEV)}
            self.plans.append(sharded.ExchangePlan(self.n[x], outs[x][1], outs[x][2], C[x].tolist(),
                                                   C[:, x].tolist(), recv_ids, None, tables))

    def to_owners(self, per_requester):
        """The all-to-all of the push: owner o gets requester r's bucket o, in rank order."""
        return [torch.cat([per_requester[r][self.send_seg[r][o]:self.send_seg[r][o + 1]]
                           for r in range(self.world)]) for o in range(self.world)]

    def from_owners(self, per_owner):
        """The all-to-all of the pull: requester r gets owner o's segment r, in rank order."""
        return [torch.cat([per_owner[o][self.recv_seg[o][r]:self.recv_seg[o][r + 1]]
                           for o in range(self.world)]) for r in range(self.world)]

    def cap(self):
        """(cap, cap_g) of receive buffers that hold every rank's rows and gradients."""
        return max(max(self.n), 1), max(max(self.m), 1)


def _local_pad(rank):
    return 0 if rank == 0 else -1          # global padding id 0 lives on rank 0 (sharded.py:8)


def _uniform_ids(n, V, g):
    ids = torch.randint(0, V, (n,), generator=g, device=DEV)
    ids[torch.rand(n, generator=g, device=DEV) < 0.05] = 0
    if n > 20:
        ids[3], ids[7], ids[11] = -3, V, V + 5
    return ids


# ---- the kernels, called through ops.raw_shard_* ---------------------------------------------------
COLS = [1, 2, 9, 20, 31, 62, 64, 128]


@pytest.mark.parametrize("layout", ["tight", "strided"])
@pytest.mark.parametrize("cols", COLS)
@pytest.mark.parametrize("world", [1, 2, 3, 4, 8, 16])
def test_gather_push_and_push_rows(world, cols, layout):
    """shard_gather_push and shard_push_rows for every VEC (1/2/4) and TPR up to 32.  Step 0:
    uniform ids with padding, negative and >= V ids, and the last rank has n = 0.  Step 1: every id
    is owned by one rank (all other segments empty), same buffers.  n * D/VEC is not a multiple of
    256*4, so the `c < total` tails run.  "strided": the shard and the pushed rows have
    row pitch > cols with sentinel columns that must not leak, and ld_dst > cols."""
    ops = _ops()
    vec, tpr = row_shape(cols)
    assert tpr <= 32
    V = 4099
    strided = layout == "strided"
    ldw = cols + 3 * vec if strided else cols
    ld_dst = cols + vec if strided else cols
    g = torch.Generator(device=DEV).manual_seed(1000 * world + cols + (7 if strided else 0))
    W = torch.randn(V, ldw, generator=g, device=DEV)
    W.view(torch.int32)[:, cols:] = SENT
    shards = [W[o::world].contiguous() for o in range(world)]
    step_ids = [
        [_uniform_ids(0 if (world > 1 and r == world - 1) else 700 + 131 * r, V, g)
         for r in range(world)],
        [torch.randint(0, (V - world // 2) // world, (500 + 97 * r,), generator=g, device=DEV) * world
         + world // 2 for r in range(world)],
    ]
    plan_sets = [_Plans(ids, world, V) for ids in step_ids]
    cap = max(max(p.cap()[0] for p in plan_sets), _cdiv(max(p.cap()[1] for p in plan_sets), 2))
    arena = _Arena(world, cap, 2 * cap, ld_dst)          # reused by both steps
    for step, (ids, P) in enumerate(zip(step_ids, plan_sets)):
        what = "world=%d cols=%d %s step %d" % (world, cols, layout, step)
        assert any(n * (cols // vec) % (PUSH_THREADS * 4) for n in P.n)
        if step == 1:
            assert sum(m > 0 for m in P.m) == 1, "one owner only"
        arena.fill()
        for o in range(world):
            p = P.plans[o]
            ops.raw_shard_gather_push(shards[o], p.recv_ids, _local_pad(o), cols,
                                      p.tables["recv_seg"], p.tables["dst_pull"], arena.rows_ptrs,
                                      ld_dst, world)
        src = []
        for r in range(world):
            rows = torch.randn(P.n[r], ldw, generator=g, device=DEV)
            rows.view(torch.int32)[:, cols:] = SENT
            src.append(rows)
            p = P.plans[r]
            ops.raw_shard_push_rows(rows, cols, p.tables["send_seg"], p.tables["dst_push"],
                                    arena.grads_ptrs, ld_dst, world)
        torch.cuda.synchronize()
        arena.check_untouched(P.n, P.m, cols)
        # pull: W_global[ids] in bucket order (zeros for padding and out-of-range ids) and the same
        # bits as the all-to-all path (raw_gather on the owner + the transpose, sharded.py:290-295)
        gathered = [ops.raw_gather(shards[o], P.plans[o].recv_ids, _local_pad(o), cols)
                    for o in range(world)]
        a2a = P.from_owners(gathered)
        for r in range(world):
            got = arena.rows(r)[:P.n[r], :cols]
            gid = ids[r][P.plans[r].inv_perm.long()]
            ok = (gid > 0) & (gid < V)
            want = torch.where(ok[:, None], W[gid.clamp(0, V - 1), :cols], 0.0)
            assert torch.equal(got, want), "%s: pulled rows of rank %d" % (what, r)
            assert torch.equal(got, a2a[r]), "%s: pull != all-to-all path, rank %d" % (what, r)
        # push: requester r's bucket o lands at recv_seg_o[r] + i of owner o
        want = P.to_owners([s[:, :cols] for s in src])
        for o in range(world):
            assert torch.equal(arena.grads(o)[:P.m[o], :cols], want[o]), (
                "%s: pushed rows of owner %d" % (what, o))


def test_gather_push_fused_table_slot():
    """The pull of a FusedTable shard (nn.py:255-263): rows of 64 floats holding
    [D emb | w1 | pad] (G = 20 floats) and the Adam moments m, v in the same slot.  Only the G
    gradient columns move; the moment columns are set to the sentinel and must not leak."""
    from paddlerec_b200 import nn as bnn
    ops = _ops()
    world, D, V = 4, 16, 20011
    tab = bnn.FusedTable(V, D, padding_idx=0, init_std=0.1, device=DEV)
    G = tab.grad_cols
    assert tab.slot == 64 and tab.moment_cols == (G, 2 * G)
    W = tab.weight.detach()
    g = torch.Generator(device=DEV).manual_seed(5)
    W[0, :D + 1] = torch.randn(D + 1, generator=g, device=DEV)     # padding must come out as zeros
    W.view(torch.int32)[:, G:] = SENT
    shards = [W[o::world].contiguous() for o in range(world)]
    ids = [_uniform_ids(4000 + 333 * r, V, g) for r in range(world)]
    P = _Plans(ids, world, V)
    cap, cap_g = P.cap()
    arena = _Arena(world, cap, cap_g, G)
    arena.fill()
    for o in range(world):
        p = P.plans[o]
        ops.raw_shard_gather_push(shards[o], p.recv_ids, _local_pad(o), G, p.tables["recv_seg"],
                                  p.tables["dst_pull"], arena.rows_ptrs, G, world)
    arena.check_untouched(P.n, [0] * world, G)
    for r in range(world):
        gid = ids[r][P.plans[r].inv_perm.long()]
        ok = (gid > 0) & (gid < V)
        want = torch.where(ok[:, None], W[gid.clamp(0, V - 1), :G], 0.0)
        assert torch.equal(arena.rows(r)[:P.n[r]], want), "rank %d" % r


# ---- fused FM-gradient push ----------------------------------------------------------------------
def _fm_problem(world, B_list, F, Dn, D, with_dfeat, seed, V=10007):
    g = torch.Generator(device=DEV).manual_seed(seed)
    ids = [_uniform_ids(B * F, V, g).reshape(B, F) for B in B_list]
    P = _Plans(ids, world, V)
    ranks = []
    for B in B_list:
        ranks.append(dict(
            feat=torch.randn(B, F + Dn, D, generator=g, device=DEV),
            S=torch.randn(B, D, generator=g, device=DEV),
            dfeat=torch.randn(B, F + Dn, D, generator=g, device=DEV) if with_dfeat else None,
            gy1=torch.randn(B, generator=g, device=DEV),
            gy2=torch.randn(B, generator=g, device=DEV),
            dense=torch.rand(B, Dn, generator=g, device=DEV)))
    return P, ranks


def _trivial_groups(n):
    return (torch.arange(n + 1, dtype=torch.int32, device=DEV),
            torch.full((2,), n, dtype=torch.int32, device=DEV))


def _check_fm_grads_push(world, B_list, D, with_dfeat, seed, F=26, Dn=13):
    """Runs the two-kernel path (raw_embed_fm_bwd with trivial groups, fused_cols=G, then
    push_rows, sharded.py:451-455) and the fused kernel (sharded.py:316-328) into the same
    receive buffers and compares them.  Both reduce to 0 + fmaf(g2, s - e, d) (embed_fm.cuh:657
    vs shard.cuh:255), so they must be equal; column D is gy1, the pad columns are 0, and columns
    0..D-1 are within 2u(|g2||s - e| + |d|) of the fp64 value."""
    ops = _ops()
    G = ops.fused_grad_cols(D)
    P, ranks = _fm_problem(world, B_list, F, Dn, D, with_dfeat, seed)
    arena = _Arena(world, 1, P.cap()[1], G)
    what = "world=%d D=%d dfeat=%s" % (world, D, with_dfeat)
    arena.fill()
    full_dense = []
    for r, x in enumerate(ranks):
        p, n = P.plans[r], P.n[r]
        iota, num = _trivial_groups(n)
        dW, _, ddw, ddw1 = ops.raw_embed_fm_bwd(x["feat"], x["S"], x["dfeat"], x["gy1"], x["gy2"],
                                                x["dense"], iota, p.inv_perm, num, F, fused_cols=G)
        full_dense.append((ddw, ddw1))
        ops.raw_shard_push_rows(dW[:n], G, p.tables["send_seg"], p.tables["dst_push"],
                                arena.grads_ptrs, G, world)
        del dW
    arena.check_untouched([0] * world, P.m, G)
    two_kernel = [arena.grads(o)[:P.m[o]].clone() for o in range(world)]
    arena.fill()
    zero_groups = torch.zeros(2, dtype=torch.int32, device=DEV)
    for r, x in enumerate(ranks):
        p, n = P.plans[r], P.n[r]
        ops.raw_shard_fm_grads_push(x["feat"], x["S"], x["dfeat"], x["gy1"], x["gy2"], p.inv_perm, F,
                                    G, p.tables["send_seg"], p.tables["dst_push"], arena.grads_ptrs,
                                    G, world)
        # the fused path keeps only the dense-feature gradients of K2 (sharded.py:448-450): they
        # must not depend on the (empty) segment table
        iota, _ = _trivial_groups(n)
        _, _, ddw, ddw1 = ops.raw_embed_fm_bwd(x["feat"], x["S"], x["dfeat"], x["gy1"], x["gy2"],
                                               x["dense"], iota, p.inv_perm, zero_groups, F,
                                               fused_cols=G)
        assert torch.equal(ddw, full_dense[r][0]) and torch.equal(ddw1, full_dense[r][1]), (
            "%s: ddense_w of the zero-segment call, rank %d" % (what, r))
    arena.check_untouched([0] * world, P.m, G)
    for o in range(world):
        assert torch.equal(arena.grads(o)[:P.m[o]], two_kernel[o]), (
            "%s: fused push != K2 + push_rows at owner %d" % (what, o))
    del two_kernel
    got = P.from_owners([arena.grads(o)[:P.m[o]] for o in range(world)])   # bucket order
    for r, x in enumerate(ranks):
        pos = P.plans[r].inv_perm.long()
        b, f = pos // F, pos % F
        assert torch.equal(got[r][:, D], x["gy1"][b]), "%s: column D != gy1, rank %d" % (what, r)
        assert torch.equal(got[r][:, D + 1:], torch.zeros_like(got[r][:, D + 1:])), (
            "%s: pad columns, rank %d" % (what, r))
        e = x["feat"][b, f].double()
        s = x["S"][b].double()
        g2 = x["gy2"][b].double()[:, None]
        d = x["dfeat"][b, f].double() if with_dfeat else torch.zeros_like(e)
        want = g2 * (s - e) + d
        assert_within(got[r][:, :D], want, 2 * U * (g2.abs() * (s - e).abs() + d.abs()),
                      "%s: gradient columns, rank %d" % (what, r))
        del e, s, g2, d, want


@pytest.mark.parametrize("with_dfeat", [False, True])
@pytest.mark.parametrize("D", [4, 12, 16, 28])
def test_fm_grads_push(D, with_dfeat):
    """G = fused_grad_cols(D) in {8, 16, 20, 32}; 3 ranks with different batch sizes."""
    _check_fm_grads_push(3, [300, 517, 64], D, with_dfeat, seed=D + 100 * with_dfeat)


def test_fm_grads_push_grid_stride():
    """The bench shape: B = 65536 per rank, F = 26, D = 16, 4 ranks.  Every CTA of the grid-stride
    loop (grid = min(ceil(n*G/4/256), 32*SM)) makes >= 3 passes."""
    ops = _ops()
    world, B, F, D = 4, 65536, 26, 16
    G = ops.fused_grad_cols(D)
    chunks = B * F * G // 4
    grid = min(_cdiv(chunks, PUSH_THREADS), FUSED_PUSH_CTAS_PER_SM * _sm())
    assert_loops("shard_fm_grads_push: grid-stride passes per CTA", chunks // (grid * PUSH_THREADS))
    _check_fm_grads_push(world, [B] * world, D, True, seed=65536, F=F)


# ---- the whole FM block through ShardExchange vs the single-GPU FusedTable path ------------------
def _sharded_fm_step(exs, P, shards, ids, dense, dense_w, dense_w1, gy1, gy2, dfeat, F, D, G, Bper,
                     fused_push):
    """One step of _ShardedEmbedFM (sharded.py:402-465, fused table) for every virtual rank, phase
    by phase: every owner's pull, then every requester's K1; every requester's push, then every
    owner's owner_reduce."""
    from paddlerec_b200 import sharded
    ops = _ops()
    world = len(exs)
    rows = [exs[o].pull(P.plans[o], shards[o], _local_pad(o), G) for o in range(world)]
    fwd = []
    for r in range(world):
        sl = slice(r * Bper, (r + 1) * Bper)
        fwd.append(ops.raw_embed_fm_fwd(rows[r], None, P.plans[r].perm.reshape(Bper, F), dense[sl],
                                        dense_w, dense_w1, -1, D=D))
    recv = []
    for r in range(world):
        sl = slice(r * Bper, (r + 1) * Bper)
        p, n = P.plans[r], P.n[r]
        feat, _, _, S = fwd[r]
        d_r = dfeat[sl] if dfeat is not None else None
        iota, num = _trivial_groups(n)
        gr = exs[r].push_fm_grads(p, feat, S, d_r, gy1[sl], gy2[sl], F, G)
        assert (gr is not None) == fused_push
        if gr is None:
            dW, _, _, _ = ops.raw_embed_fm_bwd(feat, S, d_r, gy1[sl], gy2[sl], dense[sl], iota,
                                               p.inv_perm, num, F, fused_cols=G)
            gr = exs[r].push(p, dW[:n])
        recv.append(gr)
    srs = [exs[o].owner_reduce(P.plans[o], recv[o], sharded.shard_rows(exs[o].V, o, world),
                               _local_pad(o)) for o in range(world)]
    return fwd, srs


@pytest.mark.parametrize("ids_kind", ["uniform", "zipf"])
@pytest.mark.parametrize("fused_push", [False, True])
@pytest.mark.parametrize("world", [2, 4, 8])
def test_sharded_fm_block_matches_single_gpu(world, fused_push, ids_kind, monkeypatch):
    """DeepFM's FM block on a FusedTable sharded over `world` virtual ranks (rank r holds slice r of
    the global batch), two steps with different ids on the same buffers, against raw_embed_fm_fwd /
    raw_embed_fm_bwd on the global table.

    Forward: K1 over the pulled [n, G] rows and K1 over the [V, 64] global slots see the same row
    values and pick the same K1 variant (embed_fm.cuh:599-615): feat, y1, y2, S are equal.
    Backward: the owner receives the per-slot rows in global position order, and its segment reduce
    adds them in that order, as K2 does on one GPU.  Segments of <= kHotThreshold positions are
    summed sequentially on both sides: equal.  Longer ones go to the hot kernel, whose strided split
    depends on GPB = 256/TPR with TPR from D on one side and from G on the other
    (segreduce.cuh:79,93): both sides are held to seg_chain(count) * u * sum|terms| of the fp64 sum
    of the per-slot terms."""
    from paddlerec_b200 import nn as bnn
    from paddlerec_b200 import sharded
    ops = _ops()
    monkeypatch.setattr(sharded, "FUSED_PUSH", fused_push)
    F, Dn, D = 26, 13, 16
    zipf = ids_kind == "zipf"
    V = 50000 if zipf else 100000
    B = 4096 if zipf else 1024           # global batch; Zipf: id 1 takes ln 2 / ln V = 6.4 %
    Bper = B // world
    g = torch.Generator(device=DEV).manual_seed(world * 10 + fused_push + 100 * zipf)
    tab = bnn.FusedTable(V, D, padding_idx=0, init_std=0.1, device=DEV)
    G = tab.grad_cols
    W = tab.weight.detach()
    W[0, :D + 1] = torch.randn(D + 1, generator=g, device=DEV)
    W.view(torch.int32)[:, G:] = SENT            # Adam moments in the slot: never read
    shards = [W[o::world].contiguous() for o in range(world)]
    dense_w = torch.randn(Dn, D, generator=g, device=DEV) * 0.1
    dense_w1 = torch.randn(Dn, generator=g, device=DEV) * 0.1
    exs = [sharded.ShardExchange(V, r, world, None, ops, owner_pad=_local_pad(r))
           for r in range(world)]
    arena = None
    for step in range(2):
        what = "world=%d fused_push=%s %s step %d" % (world, fused_push, ids_kind, step)
        if zipf:
            u = torch.rand(B, F, generator=g, device=DEV, dtype=torch.float64)
            ids = (V ** u).to(torch.int64).clamp_(1, V - 1)
            ids[torch.rand(B, F, generator=g, device=DEV) < 0.02] = 0
        else:
            ids = _uniform_ids(B * F, V, g).reshape(B, F)
        dense = torch.rand(B, Dn, generator=g, device=DEV)
        gy1 = torch.randn(B, generator=g, device=DEV)
        gy2 = torch.randn(B, generator=g, device=DEV)
        dfeat = torch.randn(B, F + Dn, D, generator=g, device=DEV) if step == 0 else None
        P = _Plans([ids[r * Bper:(r + 1) * Bper] for r in range(world)], world, V)
        if arena is None:
            cap, cap_g = P.cap()
            arena = _Arena(world, int(cap * 1.25), 2 * int(cap * 1.25), G)
            for r in range(world):
                exs[r].inject_peer(_DevicePeer(arena, r), G)
        assert max(P.m) <= arena.cap_g
        arena.fill()
        fwd, srs = _sharded_fm_step(exs, P, shards, ids, dense, dense_w, dense_w1, gy1, gy2, dfeat,
                                    F, D, G, Bper, fused_push)
        torch.cuda.synchronize()
        arena.check_untouched(P.n, P.m, G)

        # forward vs K1 over the global table
        ref = ops.raw_embed_fm_fwd(W, None, ids, dense, dense_w, dense_w1, 0, D=D)
        for r in range(world):
            sl = slice(r * Bper, (r + 1) * Bper)
            for name, a, b in zip(("feat", "y1", "y2", "S"), fwd[r], ref):
                assert torch.equal(a, b[sl]), "%s: %s of rank %d" % (what, name, r)

        # backward vs K2 over the global batch
        feat, _, _, S = ref
        flat = ids.reshape(-1)
        gr = ops.raw_group_ids(flat, V, 0)
        rows, _, _, _ = ops.raw_embed_fm_bwd(feat, S, dfeat, gy1, gy2, dense, gr.seg_offsets,
                                             gr.sorted_pos, gr.num, F, fused_cols=G)
        Ug = int(gr.num[0])
        ref_ids, ref_rows = gr.unique_ids[:Ug], rows[:Ug]
        sh_ids = torch.cat([sr.rows[:sr.count()] * world + o for o, sr in enumerate(srs)])
        sh_rows = torch.cat([sr.value[:sr.count()] for sr in srs])
        order_ref, order_sh = torch.argsort(ref_ids), torch.argsort(sh_ids)
        ref_ids, ref_rows = ref_ids[order_ref], ref_rows[order_ref]
        sh_ids, sh_rows = sh_ids[order_sh], sh_rows[order_sh]
        assert torch.equal(sh_ids, ref_ids), "%s: set of updated rows" % what
        assert torch.equal(sh_rows[:, D + 1:], torch.zeros_like(sh_rows[:, D + 1:])), what
        ok = (flat > 0) & (flat < V)
        counts = torch.bincount(flat[ok], minlength=V)[ref_ids]
        light = counts <= HOT_THRESHOLD
        if not zipf:
            assert bool(light.all()), "uniform ids must stay below the hot-segment threshold"
            assert int(counts.max()) >= 2
        assert torch.equal(sh_rows[light], ref_rows[light]), "%s: merged rows (light)" % what
        if zipf:
            assert int(counts.max()) > 2048, "a hot id spans several chunks"
            n = flat.numel()
            iota, num = _trivial_groups(n)
            terms, _, _, _ = ops.raw_embed_fm_bwd(feat, S, dfeat, gy1, gy2, dense, iota,
                                                  torch.arange(n, dtype=torch.int32, device=DEV),
                                                  num, F, fused_cols=G)
            t = terms[:n][ok].double()
            exact = torch.zeros(V, G, dtype=torch.float64, device=DEV).index_add_(0, flat[ok], t)
            mag = torch.zeros(V, G, dtype=torch.float64, device=DEV).index_add_(0, flat[ok], t.abs())
            hot = ~light
            c = counts[hot]
            want, m = exact[ref_ids[hot], :D + 1], mag[ref_ids[hot], :D + 1]
            assert_within(ref_rows[hot][:, :D + 1], want, seg_chain(c, D)[:, None] * U * m,
                          "%s: single-GPU hot rows" % what)
            assert_within(sh_rows[hot][:, :D + 1], want, seg_chain(c, G)[:, None] * U * m,
                          "%s: owner hot rows" % what)


# ---- argument checks ------------------------------------------------------------------------------
def test_shard_launchers_reject_bad_arguments():
    """Every check runs with n = 0, so nothing launches: a bad world, an unsupported D, a bad
    fused-gradient width, a null peer pointer and a peer base that the vector store cannot use must
    raise; the same calls with valid arguments must not."""
    from paddlerec_b200._lib import B200RecError
    ops = _ops()
    buf = torch.zeros(64, 160, device=DEV)
    base = buf.data_ptr()
    assert base % 256 == 0
    seg = torch.zeros(MAX_PEERS + 2, dtype=torch.int64, device=DEV)
    none = torch.empty(0, dtype=torch.int64, device=DEV)

    def ptrs(world=2, bad=None, value=0):
        p = [base] * max(world, 1)
        if bad is not None:
            p[bad] = value
        return _ptr_array(p)

    def gather(world=2, D=16, p=None):
        ops.raw_shard_gather_push(buf, none, -1, D, seg, seg, ptrs(world) if p is None else p, 160,
                                  world)

    def push(world=2, D=16, p=None):
        ops.raw_shard_push_rows(buf[:0], D, seg, seg, ptrs(world) if p is None else p, 160, world)

    def fm(world=2, D=16, G=20, p=None):
        F, Dn = 26, 13
        ops.raw_shard_fm_grads_push(torch.zeros(0, F + Dn, D, device=DEV), torch.zeros(0, D, device=DEV),
                                    None, torch.zeros(0, device=DEV), torch.zeros(0, device=DEV),
                                    torch.zeros(0, dtype=torch.int32, device=DEV), F, G, seg, seg,
                                    ptrs(world) if p is None else p, G, world)

    # valid calls (the pointers past `world` are not looked at)
    for D in (1, 2, 9, 16, 128):
        gather(D=D)
        push(D=D)
        gather(D=D, p=ptrs(2, bad=1, value=base + 4 * row_shape(D)[0]))
    gather(world=MAX_PEERS, p=ptrs(MAX_PEERS + 1, bad=MAX_PEERS, value=0))
    fm()
    fm(D=4, G=8)
    fm(p=ptrs(2, bad=1, value=base + 16))
    for world in (0, MAX_PEERS + 1):
        for call in (gather, push, fm):
            with pytest.raises(B200RecError, match="world"):
                call(world=world, p=ptrs(MAX_PEERS + 1))
    for D in (33, 130):
        for call in (gather, push):
            with pytest.raises(B200RecError, match="unsupported D"):
                call(D=D)
    with pytest.raises(B200RecError, match="G >= D"):
        fm(D=16, G=16)
    with pytest.raises(B200RecError, match="D % 4"):
        fm(D=18, G=20)
    for bad in (0, 1):
        for call in (gather, push, fm):
            with pytest.raises(B200RecError, match="null"):
                call(p=ptrs(2, bad=bad, value=0))
    for D, off in ((16, 4), (16, 8), (20, 12), (2, 4), (62, 2)):
        for call in (gather, push):
            with pytest.raises(B200RecError, match="aligned"):
                call(D=D, p=ptrs(2, bad=1, value=base + off))
    for off in (4, 8, 12):
        with pytest.raises(B200RecError, match="aligned"):
            fm(p=ptrs(2, bad=1, value=base + off))
