"""CPU restatement of the reference's ESMM network (TEST INFRASTRUCTURE, like oracle/nets.py, whose
`embedding` and `log_loss` it uses): models/multitask/esmm/net.py op for op, in the reference's
order, over a dict of parameters keyed by the reference's state_dict names.  Pinned to the goldens
minted from the reference's own net.py (tests/golden/make_esmm_golden.py, tests/test_esmm.py)."""
from __future__ import annotations

import importlib.util
import os
import sys

import torch

from oracle import nets, paddle_shim

REFERENCE_ROOT = "/root/reference"


def tower_sizes(params):
    """(n_ctr, n_cvr): Linear layers per tower.  The CTR tower is linear_0..linear_{n_ctr-1}, ending at
    the first layer of width 2 (esmm/net.py:42-79 numbers the CVR tower on from there)."""
    n = len([k for k in params if k.startswith("linear_") and k.endswith(".weight")])
    n_ctr = next(i for i in range(n) if params["linear_%d.weight" % i].shape[1] == 2) + 1
    return n_ctr, n - n_ctr


def esmm_logits(p, inputs, n_ctr: int, n_cvr: int):
    """(z_ctr, z_cvr), the two towers' [B,2] outputs before the softmax — esmm/net.py:85-107."""
    emb = []
    for data in inputs:                                                           # :88-93
        emb.append(nets.embedding(p["embedding.weight"], data, padding_idx=0).sum(1))
    concat_emb = torch.cat(emb, dim=1)                                            # :94
    out = []
    for first, n in ((0, n_ctr), (n_ctr, n_cvr)):                                 # :96-107
        y = concat_emb
        for i in range(first, first + n):
            y = y @ p["linear_%d.weight" % i] + p["linear_%d.bias" % i]
            if i < first + n - 1:
                y = torch.relu(y)
        out.append(y)
    return out[0], out[1]


def esmm_forward(p, inputs, n_ctr: int, n_cvr: int):
    """The six outputs of ESMMLayer.forward (:85-111): ctr_out, ctr_one, cvr_out, cvr_one,
    ctcvr_prop, ctcvr_one."""
    z_ctr, z_cvr = esmm_logits(p, inputs, n_ctr, n_cvr)
    ctr_out = torch.softmax(z_ctr, dim=-1)
    cvr_out = torch.softmax(z_cvr, dim=-1)
    ctr_one = ctr_out[:, 1:2]
    cvr_one = cvr_out[:, 1:2]
    ctcvr_one = ctr_one * cvr_one
    ctcvr_prop = torch.cat([1 - ctcvr_one, ctcvr_one], dim=1)
    return ctr_out, ctr_one, cvr_out, cvr_one, ctcvr_prop, ctcvr_one


def esmm_loss(ctr_one, clk, ctcvr_one, buy):
    """dygraph_model.py:56-67: mean(log_loss(ctr_one, clk) + log_loss(ctcvr_one, buy)), eps 1e-4."""
    return (nets.log_loss(ctr_one, clk.to(ctr_one.dtype)) +
            nets.log_loss(ctcvr_one, buy.to(ctcvr_one.dtype))).mean()


def _slice(x, axes, starts, ends):
    for axis, s, e in zip(axes, starts, ends):
        x = x.narrow(axis, s, e - s)
    return x


def install_esmm_apis(reference_root: str = REFERENCE_ROOT):
    """Give the paddle shim the one API esmm/net.py needs beyond the rank models (`paddle.slice`,
    :99-100) and load the reference's models/multitask/esmm/net.py, unmodified, by path."""
    paddle_shim.install()
    sys.modules["paddle"].slice = _slice
    path = os.path.join(reference_root, "models", "multitask", "esmm", "net.py")
    spec = importlib.util.spec_from_file_location("ref_esmm_net", path)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def load_reference_reader(reference_root: str = REFERENCE_ROOT):
    """The reference's esmm_reader.py, unmodified, on the shim's paddle.io."""
    paddle_shim.install()
    path = os.path.join(reference_root, "models", "multitask", "esmm", "esmm_reader.py")
    spec = importlib.util.spec_from_file_location("ref_esmm_reader", path)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m
