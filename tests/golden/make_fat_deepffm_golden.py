"""Mint tests/golden/fat_deepffm_d10.npz and fat_deepffm_d10_init.npz by EXECUTING THE REFERENCE'S
OWN models/rank/fat_deepffm/net.py (unmodified) in float64, in eval mode (dropout off, as the other
goldens with dropout: SURVEY.md Q5), on top of oracle/paddle_shim.py plus the APIs from
tests/fat_deepffm_oracle.install_fat_apis, the way make_golden.py mints the other models' vectors
(and with its file layout).

Run in the authoring container only (needs the reference checkout):
    python tests/golden/make_fat_deepffm_golden.py
Edge cases: id 0 is a REAL row (no padding_idx), the same id at two fields of one sample, one id
shared across the batch.  Every parameter and input is rounded to an fp32-representable value, so
an fp32 run starts from exactly the golden's numbers.
  * fat_deepffm_d10: dense_w is overridden with small random values so that every path carries
    gradient, and the zero dense values are replaced; every pooled block's top two values differ
    (asserted), so fp32 and fp64 pick the same argmax.
  * fat_deepffm_d10_init: the reference's own dense_w = 1.0 and the zero dense values, where every
    dense block is an exact tie and the first-maximum rule decides where the pool's gradient goes
    (dense values scaled by 0.05 so that the sigmoid is not saturated).
"""
from __future__ import annotations

import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

from make_golden import check_oracle, criteo_batch, grads_of, save  # noqa: E402
from oracle import nets, paddle_shim  # noqa: E402
from tests import fat_deepffm_oracle  # noqa: E402

# 8 sparse and 4 dense fields rather than Criteo's 26 and 13: the attention MLP is two
# NF^2 x NF^2 Linears, which at NF = 39 would put 4.6 M fp64 weights (and their gradients, ~60 MB)
# in the file.  The kernels are checked at NF = 39 against fp64 in tests/test_gpu_fat_deepffm.py.
V, F, Dn, D, LAYERS = 53, 8, 4, 10, [32, 16]


def _fp32(t):
    return t.float().double()


def make(tag, override_dense_w):
    paddle_shim.install()
    fat_deepffm_oracle.install_fat_apis()
    ref = paddle_shim.import_reference_net("fat_deepffm")
    torch.manual_seed(5150)
    layer = ref.FAT_DeepFFMLayer(V, D, Dn, F, LAYERS)
    layer.eval()
    named = dict(layer.named_parameters())
    g = torch.Generator().manual_seed(707)
    with torch.no_grad():
        for k, v in named.items():
            v.copy_(_fp32(v))
        if override_dense_w:
            named["cen.dense_w"].copy_(_fp32(torch.randn(named["cen.dense_w"].shape, generator=g,
                                                         dtype=torch.float64) * 0.1))
        named["bias"].fill_(0.05)
        # the attention MLP starts with zero biases: small ones make its ReLUs see both signs
        for k in ("cen.fc.ReductionLinear.bias", "cen.fc.AdditionLinear.bias"):
            named[k].copy_(_fp32(torch.randn(named[k].shape, generator=g, dtype=torch.float64) * 0.1))
    ids, dense, label = criteo_batch(g, 12, V, F, Dn)
    if not override_dense_w:
        # dense_w = 1.0 with Criteo-sized dense values saturates the sigmoid (p within 1e-4 of 1),
        # where an fp32 gradient has no correct digits; smaller values keep the ties and the zeros
        dense = dense * 0.05
    dense = _fp32(dense)
    NF = F + Dn
    if override_dense_w:
        # a zero dense value makes its whole dense row a tie: that case belongs to the init golden
        dense[dense == 0] = 0.25
        feat = torch.cat([named["cen.embedding.weight"][ids],
                          dense.unsqueeze(2) * named["cen.dense_w"]], 1).reshape(-1, NF * NF, D)
        top2 = feat.detach().float().topk(2, dim=-1).values
        assert bool((top2[..., 0] > top2[..., 1]).all()), "a pooled block has a tie in fp32"
    sparse_inputs = [ids[:, i:i + 1] for i in range(F)]
    pred = layer(sparse_inputs, dense)
    loss = nets.log_loss(pred, label.to(pred.dtype)).mean()
    check_oracle("fat_deepffm %s" % tag, pred,
                 fat_deepffm_oracle.fat_deepffm_forward(named, sparse_inputs, dense, NF))
    save("fat_deepffm_%s" % tag, named, {"ids": ids, "dense": dense, "label": label}, pred, loss,
         grads_of(loss, named))


if __name__ == "__main__":
    torch.set_default_dtype(torch.float64)
    make("d10", True)
    make("d10_init", False)
