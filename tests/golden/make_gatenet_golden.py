"""Mint tests/golden/gatenet_*.npz by EXECUTING THE REFERENCE'S OWN models/rank/gatenet/net.py
(unmodified) in float64 on top of oracle/paddle_shim.py (plus `Layer.add_parameter`, from
tests/gatenet_oracle.py), with make_golden.py's file layout plus `out/logit`, the last layer's output
before the sigmoid (captured with a forward hook on `last_layer`).

Run in the authoring container only (needs the reference checkout):
    python tests/golden/make_gatenet_golden.py
Cases, all at the reference's config.yaml shape (D = 9, fc [512, 256, 128, 32], 26 + 13 fields) and
a small V:
  gatenet_init    both gates at the reference's initialisation: the logit is ~1e-12 (SURVEY Q18)
  gatenet_scaled  both gates, hidden-gate weights scaled up so that the logit is O(1)
  gatenet_embed   embedding gate only
  gatenet_hidden  hidden gates only, at the reference's initialisation
Edge cases: id 0 is a REAL row (no padding_idx), the same id at two fields of one sample, one id
shared across the batch.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

from make_golden import check_oracle, criteo_batch, grads_of  # noqa: E402
from oracle import nets, paddle_shim  # noqa: E402
from tests import gatenet_oracle  # noqa: E402

FC = [64, 32, 16, 8]


def make_gatenet(tag, use_embedding_gate, use_hidden_gate, gate_scale=None):
    paddle_shim.install()
    gatenet_oracle.install_add_parameter()
    ref = paddle_shim.import_reference_net("gatenet")
    torch.manual_seed(7070)
    V, F, Dn, D = 53, 26, 13, 9
    layer = ref.GateDNNLayer(V, D, Dn, F, FC, use_embedding_gate, use_hidden_gate)
    named = dict(layer.named_parameters())
    if gate_scale is not None:
        with torch.no_grad():
            for i in range(len(FC)):
                named["hidden_gate_weight_%d" % i].mul_(gate_scale[i])
    captured = {}
    layer.last_layer.register_forward_hook(lambda m, i, o: captured.__setitem__("logit", o))
    g = torch.Generator().manual_seed(818)
    ids, dense, label = criteo_batch(g, 12, V)
    sparse_inputs = [ids[:, i:i + 1] for i in range(F)]
    pred = layer(sparse_inputs, dense)
    loss = nets.log_loss(pred, label.to(pred.dtype)).mean()
    check_oracle("gatenet %s" % tag, pred, gatenet_oracle.gatenet_forward(
        named, sparse_inputs, dense, len(FC), use_embedding_gate, use_hidden_gate))
    logit = captured["logit"]
    err = (logit - gatenet_oracle.gatenet_logit(named, sparse_inputs, dense, len(FC),
                                                use_embedding_gate, use_hidden_gate)).abs().max()
    assert float(err) <= 1e-12 * max(1.0, float(logit.abs().max())), err
    out = {"param/" + k: v.detach().numpy() for k, v in named.items()}
    out.update({"in/ids": ids.numpy(), "in/dense": dense.numpy(), "in/label": label.numpy(),
                "out/pred": pred.detach().numpy(), "out/loss": loss.detach().numpy(),
                "out/logit": logit.detach().numpy()})
    out.update({"grad/" + k: v.numpy() for k, v in grads_of(loss, named).items()})
    path = os.path.join(HERE, "gatenet_%s.npz" % tag)
    np.savez_compressed(path, **out)
    print("wrote %s (%d arrays, %.1f KB), logit rms %.3e" % (
        path, len(out), os.path.getsize(path) / 1024, float(logit.square().mean().sqrt())))


if __name__ == "__main__":
    torch.set_default_dtype(torch.float64)
    make_gatenet("init", True, True)
    make_gatenet("scaled", True, True, gate_scale=[5.0, 20.0, 100.0, 100.0])
    make_gatenet("embed", True, False)
    make_gatenet("hidden", False, True)
