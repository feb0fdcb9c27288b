"""GateNet network — same class, constructor arguments, forward signature, initialisers and state_dict
names as the reference's models/rank/gatenet/net.py (GateDNNLayer :20-121).

  embedding gate (:88-103) + concat (:110)  ONE fused gather kernel each way (b200rec_gate_embed_*);
                                            without the gate, the plain b200rec_gather as Wide&Deep
  hidden layers + hidden gates (:112-118)   the wgmma tower in 'bf16x3' precision (tower.mlp with
                                            gates=: the gate GEMM's epilogue applies y * tanh(acc));
                                            in 'fp32' / 'tf32' the reference's op sequence in torch
  last_layer + sigmoid (:119-120)

Reference behaviour kept on purpose (SURVEY.md Q18): at the reference's initialisation the hidden
gates make the signal vanish (each gated layer is roughly quadratic in a small non-negative y), so
the logit is ~1e-12 and pred is 0.5 in fp32; the table is Uniform(-1, 1) with no padding row; the
embedding gate is one scalar per field applied to the sum over the row's columns.
"""
from __future__ import annotations

import math

import torch
import torch.nn as tnn

from ... import nn as bnn
from ... import ops
from ... import tower


class GateDNNLayer(tnn.Module):
    def __init__(self, sparse_feature_number, sparse_feature_dim, dense_feature_dim, num_field,
                 layer_sizes, use_embedding_gate, use_hidden_gate, device="cuda"):
        super().__init__()
        self.sparse_feature_number = sparse_feature_number
        self.sparse_feature_dim = sparse_feature_dim
        self.dense_feature_dim = dense_feature_dim
        self.num_field = num_field
        self.layer_sizes = list(layer_sizes)
        self.use_embedding_gate = bool(use_embedding_gate)
        self.use_hidden_gate = bool(use_hidden_gate)
        self.embedding_gate_weight = []
        if self.use_embedding_gate:                                               # :32-43
            for i in range(num_field):
                w = tnn.Parameter(torch.empty(1, device=device).normal_(0.0, 1.0))
                self.register_parameter("embedding_gate_weight_%d" % i, w)
                self.embedding_gate_weight.append(w)
        self.embedding = bnn.Embedding(sparse_feature_number, sparse_feature_dim,    # :44-50
                                       padding_idx=None, init="uniform", device=device)
        sizes = [sparse_feature_dim * num_field + dense_feature_dim] + self.layer_sizes
        self.last_layer = bnn.Linear(sizes[-1], 1,                                # :55-61
                                     weight_std=1.0 / math.sqrt(sizes[-1])).to(device)
        self._mlp_layers = []
        self._hidden_gate_weight = []
        for i in range(len(self.layer_sizes)):                                    # :62-83
            linear = bnn.Linear(sizes[i], sizes[i + 1],
                                weight_std=1.0 / math.sqrt(sizes[i])).to(device)
            self.add_module("linear_%d" % i, linear)
            self._mlp_layers.append(linear)
            act = tnn.ReLU()
            self.add_module("act_%d" % i, act)
            self._mlp_layers.append(act)
            if self.use_hidden_gate:
                n = sizes[i + 1]
                G = tnn.Parameter(torch.empty(n, n, device=device).normal_(0.0, 1.0 / math.sqrt(n)))
                self.register_parameter("hidden_gate_weight_%d" % i, G)
                self._hidden_gate_weight.append(G)

    def _tower_input(self, sparse_inputs, dense_inputs):
        ids = (torch.cat(list(sparse_inputs), dim=1) if isinstance(sparse_inputs, (list, tuple))
               else sparse_inputs)
        B = ids.shape[0]
        D = self.sparse_feature_dim
        if self.use_embedding_gate:                                               # :88-103, :110
            gate_w = torch.cat(self.embedding_gate_weight)                        # [F], once
            return ops.gate_embed(gate_w, self.embedding.weight, ids, dense_inputs, self.embedding, D)
        emb = self.embedding(ids).reshape(B, -1)                                  # :104-108
        return torch.cat([emb, dense_inputs], dim=1)                              # :110

    def logit(self, sparse_inputs, dense_inputs):
        """The last layer's output before the sigmoid, [B, 1]."""
        x = self._tower_input(sparse_inputs, dense_inputs)
        linears = [m for m in self._mlp_layers if isinstance(m, bnn.Linear)]
        if bnn.get_matmul_precision() == "bf16x3" and x.is_cuda:
            Ws = [m.weight for m in linears] + [self.last_layer.weight]
            bs = [m.bias for m in linears] + [self.last_layer.bias]
            gates = self._hidden_gate_weight if self.use_hidden_gate else None
            return tower.mlp(x, Ws, bs, gates=gates)
        for i, linear in enumerate(linears):                                      # :112-118
            x = torch.relu(linear(x))
            if self.use_hidden_gate:
                x = x * torch.tanh(bnn._LinearFn.apply(x, self._hidden_gate_weight[i], None))
        return self.last_layer(x)                                                 # :119

    def forward(self, sparse_inputs, dense_inputs):
        y = self.logit(sparse_inputs, dense_inputs)
        if y.is_cuda:
            return ops.sum_sigmoid(y)                                             # :120
        return torch.sigmoid(y)
