"""Mint tests/golden/esmm_*.npz by EXECUTING THE REFERENCE'S OWN models/multitask/esmm/net.py
(unmodified) in float64 on top of oracle/paddle_shim.py (plus `paddle.slice`, from
tests/esmm_oracle.py), and tests/golden/esmm_reader_batches.npz from the reference's own
esmm_reader.py over the two sample files under tests/golden/esmm_sample/.

Run in the authoring container only (needs the reference checkout):
    python tests/golden/make_esmm_golden.py
Model cases, at D = 12, 23 fields of 3 ids, a small V and fc [32, 16] (not [256, 64], so each file
stays under 0.4 MB):
  esmm_init       the reference's initialisation
  esmm_saturated  both last layers scaled so that both towers' logit gaps pass 20 with both signs
Each holds the parameters, the inputs, the two towers' logits (`out/z_ctr`, `out/z_cvr`, captured
with forward hooks on the last Linears), the six outputs, the loss and every gradient.
Edge cases in both: the same id twice in one bag, one id in several fields and samples, an
all-padding bag, a sample whose every bag is padding, buy = 1 only where click = 1.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

from make_golden import grads_of  # noqa: E402
from tests import esmm_oracle  # noqa: E402

FC = [32, 16]
V, D, F, L, B = 61, 12, 23, 3, 12
OUTS = ("ctr_out", "ctr_one", "cvr_out", "cvr_one", "ctcvr_prop", "ctcvr_one")


def esmm_batch(g):
    ids = torch.randint(1, V, (B, F, L), generator=g)
    ids[0, 2, 1] = ids[0, 2, 0]           # the same id twice in one bag
    ids[3:, 0, 0] = 17                    # one id in several samples ...
    ids[4, 5, 1] = ids[6, 9, 2] = 17      # ... and fields
    ids[0, 7, :] = 0                      # an all-padding bag
    ids[2, 3, 1:] = 0                     # a bag padded after one id
    ids[1] = 0                            # a sample whose every bag is padding
    clk = (torch.rand(B, 1, generator=g) < 0.5).to(torch.int64)
    buy = clk * (torch.rand(B, 1, generator=g) < 0.5).to(torch.int64)
    clk[5, 0] = buy[5, 0] = 1
    clk[6, 0], buy[6, 0] = 1, 0
    return ids, clk, buy


def make_esmm(tag, last_scale=None):
    ref = esmm_oracle.install_esmm_apis()
    torch.manual_seed(2024)
    layer = ref.ESMMLayer(V, D, F, FC, FC)
    named = dict(layer.named_parameters())
    n_ctr, n_cvr = esmm_oracle.tower_sizes(named)
    if last_scale is not None:
        with torch.no_grad():
            for i in (n_ctr - 1, n_ctr + n_cvr - 1):
                named["linear_%d.weight" % i].mul_(last_scale)
    captured = {}
    getattr(layer, "linear_%d" % (n_ctr - 1)).register_forward_hook(
        lambda m, i, o: captured.__setitem__("z_ctr", o))
    getattr(layer, "linear_%d" % (n_ctr + n_cvr - 1)).register_forward_hook(
        lambda m, i, o: captured.__setitem__("z_cvr", o))
    g = torch.Generator().manual_seed(919)
    ids, clk, buy = esmm_batch(g)
    inputs = [ids[:, f, :] for f in range(F)]
    outs = layer(inputs)
    loss = esmm_oracle.esmm_loss(outs[1], clk, outs[5], buy)
    mine = esmm_oracle.esmm_forward(named, inputs, n_ctr, n_cvr)
    for name, a, b in zip(OUTS, outs, mine):
        assert float((a - b).detach().abs().max()) <= 1e-12, name
    if last_scale is not None:
        for z in (captured["z_ctr"], captured["z_cvr"]):
            gap = (z[:, 1] - z[:, 0]).detach()
            assert float(gap.max()) > 20 and float(gap.min()) < -20, gap
    out = {"param/" + k: v.detach().numpy() for k, v in named.items()}
    out.update({"in/ids": ids.numpy(), "in/clk": clk.numpy(), "in/buy": buy.numpy(),
                "out/loss": loss.detach().numpy(), "out/z_ctr": captured["z_ctr"].detach().numpy(),
                "out/z_cvr": captured["z_cvr"].detach().numpy()})
    out.update({"out/" + n: o.detach().numpy() for n, o in zip(OUTS, outs)})
    out.update({"grad/" + k: v.numpy() for k, v in grads_of(loss, named).items()})
    path = os.path.join(HERE, "esmm_%s.npz" % tag)
    np.savez_compressed(path, **out)
    print("wrote %s (%d arrays, %.1f KB)" % (path, len(out), os.path.getsize(path) / 1024))


def make_reader_batches():
    reader = esmm_oracle.load_reference_reader()
    out = {}
    for split in ("train", "test"):
        path = os.path.join(HERE, "esmm_sample", split, "small.txt")
        samples = list(reader.RecDataset([path], {"hyper_parameters.max_len": 3}))
        out[split + "/ids"] = np.stack([np.stack(s[:F]) for s in samples])
        out[split + "/clk"] = np.stack([s[F] for s in samples])
        out[split + "/buy"] = np.stack([s[F + 1] for s in samples])
    path = os.path.join(HERE, "esmm_reader_batches.npz")
    np.savez_compressed(path, **out)
    print("wrote %s (%.1f KB)" % (path, os.path.getsize(path) / 1024))


if __name__ == "__main__":
    torch.set_default_dtype(torch.float64)
    make_esmm("init")
    make_esmm("saturated", last_scale=60.0)
    make_reader_batches()
