"""Mint tests/golden/ffm_d9.npz and ffm_d16.npz by EXECUTING THE REFERENCE'S OWN
models/rank/ffm/net.py (unmodified) in float64 on top of oracle/paddle_shim.py (plus `add_n`, from
tests/ffm_oracle.py), the same way make_golden.py mints the other models' vectors (and with its
file layout).

Run in the authoring container only (needs the reference checkout):
    python tests/golden/make_ffm_golden.py
Edge cases: id 0 is a REAL row (FFM has no padding_idx), the same id at two fields of one sample,
one id shared across the batch.  The reference initialises dense_w_one and dense_w to 1.0, which
saturates the sigmoid (p(1-p) == 0 in fp32) on many Criteo rows; both are overridden with small
random values so that every path carries gradient.
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
from tests import ffm_oracle  # noqa: E402


def make_ffm(D, tag):
    paddle_shim.install()
    ffm_oracle.install_add_n()
    ref = paddle_shim.import_reference_net("ffm")
    torch.manual_seed(4040 + D)
    V, F, Dn = 53, 26, 13
    layer = ref.FFMLayer(V, D, Dn, F + Dn)
    named = dict(layer.named_parameters())
    with torch.no_grad():
        named["ffm.dense_w_one"].normal_(0, 0.1)
        named["ffm.dense_w"].normal_(0, 0.1)
        named["bias"].fill_(0.05)
    g = torch.Generator().manual_seed(606)
    ids, dense, label = criteo_batch(g, 12, V)
    sparse_inputs = [ids[:, i:i + 1] for i in range(F)]
    pred = layer(sparse_inputs, dense)
    loss = nets.log_loss(pred, label.to(pred.dtype)).mean()
    check_oracle("ffm D=%d" % D, pred, ffm_oracle.ffm_forward(named, sparse_inputs, dense, F + Dn))
    save("ffm_%s" % tag, named, {"ids": ids, "dense": dense, "label": label}, pred, loss,
         grads_of(loss, named))


if __name__ == "__main__":
    torch.set_default_dtype(torch.float64)
    make_ffm(9, "d9")      # the reference's D (config.yaml)
    make_ffm(16, "d16")
