"""CPU restatement of the reference's GateNet network (TEST INFRASTRUCTURE, like oracle/nets.py, whose
`embedding` it uses): models/rank/gatenet/net.py op for op, in the reference's order, over a dict of
parameters keyed by the reference's state_dict names.  Pinned to the goldens minted from the
reference's own net.py (tests/golden/make_gatenet_golden.py, tests/test_gatenet.py)."""
from __future__ import annotations

import sys

import torch

from oracle import nets


def gatenet_logit(p, sparse_inputs, dense_inputs, n_fc: int, use_embedding_gate: bool,
                  use_hidden_gate: bool):
    """GateDNNLayer.forward up to last_layer — gatenet/net.py:85-119 (no padding_idx)."""
    table = p["embedding.weight"]
    D = table.shape[1]
    sparse_embs = []
    for i, s_input in enumerate(sparse_inputs):                                   # :88-108
        emb = nets.embedding(table, s_input).reshape(-1, D)
        if use_embedding_gate:
            gate = (emb * p["embedding_gate_weight_%d" % i]).sum(-1, keepdim=True)
            emb = emb * torch.sigmoid(gate)
        sparse_embs.append(emb)
    y = torch.cat(sparse_embs + [dense_inputs], dim=1)                            # :110
    for i in range(n_fc):                                                         # :112-118
        y = torch.relu(y @ p["linear_%d.weight" % i] + p["linear_%d.bias" % i])
        if use_hidden_gate:
            y = y * torch.tanh(y @ p["hidden_gate_weight_%d" % i])
    return y @ p["last_layer.weight"] + p["last_layer.bias"]                      # :119


def gatenet_forward(p, sparse_inputs, dense_inputs, n_fc, use_embedding_gate, use_hidden_gate):
    return torch.sigmoid(gatenet_logit(p, sparse_inputs, dense_inputs, n_fc, use_embedding_gate,
                                       use_hidden_gate))                          # :120


def install_add_parameter():
    """Give the paddle shim's Layer the one API gatenet/net.py needs beyond the other rank models
    (`Layer.add_parameter`, :42-43, :82-83), so the reference's net.py runs on it unmodified."""
    paddle = sys.modules["paddle"]
    paddle.nn.Layer.add_parameter = lambda self, name, param: self.register_parameter(name, param) \
        or param
    return paddle


def flags(params):
    """(n_fc, use_embedding_gate, use_hidden_gate) of a parameter dict."""
    n_fc = len([k for k in params if k.startswith("linear_") and k.endswith(".weight")])
    return (n_fc, any(k.startswith("embedding_gate_weight_") for k in params),
            any(k.startswith("hidden_gate_weight_") for k in params))
