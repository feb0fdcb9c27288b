"""Cross-check against the reference's own code: its models/rank/*/net.py, executed unmodified on
oracle/paddle_shim.py with other seeds and shapes than the golden vectors of test_oracle_golden.py,
against oracle/nets.py — forward and every parameter gradient, float64 — and its three Python readers
on their bundled sample files against oracle/readers.py and the native parsers.  What the reference
computed is stored under tests/golden/ (reference_live_*.npz, minted by make_live_golden.py)."""
import gzip
import os

import numpy as np
import pytest
import torch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(autouse=True)
def _f64():
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    yield
    torch.set_default_dtype(prev)


def _case(tag, case):
    """(named parameters with the reference's aliases restored, inputs, reference output, gradients)"""
    z = np.load(os.path.join(GOLD, "reference_live_%s.npz" % tag))
    pre = case + "/"
    tensors = {}
    for k in z.files:
        if k.startswith(pre + "tensor/"):
            tensors[int(k.rsplit("/", 1)[1])] = torch.from_numpy(z[k]).double().requires_grad_(True)
    named = {k[len(pre + "param/"):]: tensors[int(z[k])] for k in z.files if k.startswith(pre + "param/")}
    inputs = {k[len(pre + "input/"):]: torch.from_numpy(z[k]) for k in z.files if k.startswith(pre + "input/")}
    grads = {k[len(pre + "grad/"):]: torch.from_numpy(z[k]) for k in z.files if k.startswith(pre + "grad/")}
    assert named and set(grads) == set(named)
    return named, inputs, torch.from_numpy(z[pre + "out"]), grads


def _slots(inputs):
    ids = inputs["ids"]
    return [ids[:, i:i + 1] for i in range(ids.shape[1])], inputs["dense"]


def _same(ref_out, ref_grads, ora_out, named):
    assert (ref_out - ora_out).abs().max() < 1e-12
    gs = torch.autograd.grad(ora_out.square().sum(), list(named.values()), allow_unused=True)
    for (k, p), g in zip(named.items(), gs):
        g = torch.zeros_like(p) if g is None else g
        assert (ref_grads[k] - g).abs().max() < 1e-10, k


@pytest.mark.parametrize("seed,D,B", [(1, 5, 3), (2, 12, 9)])
def test_deepfm_live(seed, D, B):
    from oracle import nets
    named, inputs, out, grads = _case("deepfm", "deepfm_%d_%d_%d" % (seed, D, B))
    ids, dense = _slots(inputs)
    _same(out, grads, nets.deepfm_forward(named, ids, dense, 3), named)


@pytest.mark.parametrize("mix,stacked", [(False, False), (True, True)])
def test_dcn_v2_live(mix, stacked):
    from oracle import nets
    named, inputs, out, grads = _case("dcn", "dcn_v2_%d_%d" % (mix, stacked))
    ids, dense = _slots(inputs)
    ora = nets.dcn_v2_forward(named, ids, dense, n_fc=2, cross_num=3, is_stacked=stacked,
                              use_low_rank_mixture=mix, num_experts=2)
    _same(out, grads, ora, named)


def test_din_and_wide_deep_live():
    from oracle import nets
    named, inputs, out, grads = _case("wide", "wide_deep")
    ids, dense = _slots(inputs)
    _same(out, grads, nets.wide_deep_forward(named, ids, dense, 2), named)

    named, inputs, out, grads = _case("din", "din")
    hi, hc, ti, tc, mask = (inputs[k] for k in ("hi", "hc", "ti", "tc", "mask"))
    L = hi.shape[1]
    args = (hi, hc, ti, tc, None, mask, ti.unsqueeze(1).repeat(1, L), tc.unsqueeze(1).repeat(1, L))
    _same(out, grads, nets.din_forward(named, *args), named)


@pytest.mark.parametrize("self_interaction,B,d", [(False, 6, 4), (True, 9, 8)])
def test_dlrm_live(self_interaction, B, d):
    """dlrm/net.py (train mode: BatchNorm on batch statistics), incl. the self_interaction=True
    branch whose diagonal entries evaluate to 0."""
    from oracle import nets
    named, inputs, out, grads = _case("dlrm", "dlrm_%d_%d_%d" % (self_interaction, B, d))
    ids, dense = _slots(inputs)
    ora = nets.dlrm_forward(named, ids, dense, n_bot=2, n_top=2, self_interaction=self_interaction)
    _same(out, grads, ora, named)


def test_readers_live():
    """The reference's three Python readers on the reference's own bundled sample files, against
    oracle/readers.py and the native parsers."""
    from oracle import readers
    from paddlerec_b200 import dataio

    z = np.load(os.path.join(GOLD, "reference_live_readers.npz"))
    sample = gzip.decompress(open(os.path.join(GOLD, "ref_deepfm_sample_train.txt.gz"), "rb").read())
    ids_ref, dense_ref = z["reader/deepfm/ids"], z["reader/deepfm/dense"]
    label, ids, dense = dataio.parse_slot_text(sample)
    assert np.array_equal(label[:, 0], ids_ref[:, 0]) and np.array_equal(ids, ids_ref[:, 1:])
    assert np.array_equal(dense, dense_ref)
    oi, od = readers.slot_text_packed(sample.decode().split("\n"), ["click"] + [str(i) for i in range(1, 27)],
                                      "dense_feature", 13)
    assert np.array_equal(oi, ids_ref) and np.array_equal(od, dense_ref)

    # the reference's dcn_v2 sample file is the same bytes as the deepfm one
    label, ids, dense = dataio.parse_slot_text(sample, dataio.CRITEO_DCN_V2)
    assert np.array_equal(ids, z["reader/dcn_v2/ids"])
    # log(v+1): numpy's and libm's double log may differ in the last place before the float32 cast
    assert np.allclose(dense, z["reader/dcn_v2/dense"], rtol=2e-7, atol=0)

    din_sample = os.path.join(GOLD, "ref_din_sample_data.txt")
    n = int(z["reader/din/n_samples"])
    batches = list(dataio.DinBatchReader([din_sample], 8, as_torch=False))
    assert len(batches) == n // 8 > 0
    for b, batch in enumerate(batches):
        for j in range(8):
            assert np.array_equal(batch[j], z["reader/din/%d/%d" % (b, j)]), (b, j)
