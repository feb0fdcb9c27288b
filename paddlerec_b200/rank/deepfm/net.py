"""DeepFM network — same classes, constructor arguments, forward signature and state_dict names as
the reference's models/rank/deepfm/net.py (DeepFMLayer :21-49, FM :52-139, DNN :142-174), with the
FM body replaced by ONE fused sm_90a kernel (b200rec_embed_fm_fwd / _bwd).

Reference quirks kept on purpose (SURVEY.md Appendix C): `self.bias` exists but is never added to
the logit (Q1); both tables use padding_idx=0 (row 0 reads as zeros and gets no gradient).
"""
from __future__ import annotations

import math

import torch
import torch.nn as tnn

from ... import nn as bnn
from ... import ops
from ... import tower


class DeepFMLayer(tnn.Module):
    def __init__(self, sparse_feature_number, sparse_feature_dim, dense_feature_dim,
                 sparse_num_field, layer_sizes, device="cuda", fused_table=None):
        super().__init__()
        self.sparse_feature_number = sparse_feature_number
        self.sparse_feature_dim = sparse_feature_dim
        self.dense_feature_dim = dense_feature_dim
        self.sparse_num_field = sparse_num_field
        self.layer_sizes = layer_sizes

        self.fm = FM(sparse_feature_number, sparse_feature_dim, dense_feature_dim,
                     sparse_num_field, device=device, fused_table=fused_table)
        self.dnn = DNN(sparse_feature_number, sparse_feature_dim, dense_feature_dim,
                       dense_feature_dim + sparse_num_field, layer_sizes, device=device)
        self.bias = tnn.Parameter(torch.zeros(1, device=device))  # unused, as in net.py:36-39

    def forward(self, sparse_inputs, dense_inputs):
        y_first_order, y_second_order, feat_embeddings = self.fm(sparse_inputs, dense_inputs)
        y_dnn = self.dnn(feat_embeddings)
        if y_dnn.is_cuda:   # net.py:47 — the two adds and the sigmoid as one kernel each way
            return ops.sum_sigmoid(y_first_order, y_second_order, y_dnn)
        return torch.sigmoid(y_first_order + y_second_order + y_dnn)


class FM(bnn.FusedTableOwner):
    """`fused_table` (default: on when D+1 fits one 128-byte slot) stores both tables as
    bnn.FusedTable; state_dict keys stay `embedding.weight` / `embedding_one.weight`."""

    def __init__(self, sparse_feature_number, sparse_feature_dim, dense_feature_dim,
                 sparse_num_field, device="cuda", fused_table=None):
        super().__init__()
        self.sparse_feature_number = sparse_feature_number
        self.sparse_feature_dim = sparse_feature_dim
        self.dense_feature_dim = dense_feature_dim
        self.dense_emb_dim = sparse_feature_dim
        self.sparse_num_field = sparse_num_field
        self.init_value_ = 0.1
        std = self.init_value_ / math.sqrt(float(sparse_feature_dim))
        # net.py:66-86 — two tables indexed by the same ids
        self.fused = (sparse_feature_dim + 1 <= 32) if fused_table is None else bool(fused_table)
        if self.fused:
            self._fused = bnn.FusedTable(sparse_feature_number, sparse_feature_dim, padding_idx=0,
                                         init_std=std, device=device)
        else:
            self.embedding_one = bnn.Embedding(sparse_feature_number, 1, padding_idx=0,
                                               init_std=std, device=device)
            self.embedding = bnn.Embedding(sparse_feature_number, sparse_feature_dim,
                                           padding_idx=0, init_std=std, device=device)
            self._pair = bnn.EmbeddingPair(self.embedding, self.embedding_one)
        # net.py:89-103
        self.dense_w_one = tnn.Parameter(torch.empty(dense_feature_dim, device=device))
        self.dense_w = tnn.Parameter(
            torch.empty(1, dense_feature_dim, self.dense_emb_dim, device=device))
        tnn.init.trunc_normal_(self.dense_w_one, 0.0, std, -2 * std, 2 * std)
        tnn.init.trunc_normal_(self.dense_w, 0.0, std, -2 * std, 2 * std)

    def table_grad_dense(self):
        """(dW [V,D], dW1 [V,1]) dense gradients of the two tables (tests / small tables)."""
        if self.fused:
            return self._fused.grad_dense()
        z = lambda e: (e.grad_rows.to_dense() if e.grad_rows is not None  # noqa: E731
                       else torch.zeros_like(e.weight))
        return z(self.embedding), z(self.embedding_one)

    def forward(self, sparse_inputs, dense_inputs):
        # net.py:107 concat of the 26 [B,1] slots; a ready-made [B,26] tensor is accepted too
        if isinstance(sparse_inputs, (list, tuple)):
            ids = torch.cat(list(sparse_inputs), dim=1)
        else:
            ids = sparse_inputs
        if self.fused:
            feat, y1, y2, _S = ops.embed_fm(self._fused.weight, None, ids, dense_inputs,
                                            self.dense_w, self.dense_w_one, 0, self._fused,
                                            D=self.sparse_feature_dim)
        else:
            feat, y1, y2, _S = ops.embed_fm(self.embedding.weight, self.embedding_one.weight, ids,
                                            dense_inputs, self.dense_w, self.dense_w_one, 0,
                                            self._pair)
        return y1, y2, feat


class DNN(tnn.Module):
    def __init__(self, sparse_feature_number, sparse_feature_dim, dense_feature_dim, num_field,
                 layer_sizes, device="cuda"):
        super().__init__()
        self.sparse_feature_dim = sparse_feature_dim
        self.num_field = num_field
        self.layer_sizes = layer_sizes
        sizes = [sparse_feature_dim * num_field] + list(layer_sizes) + [1]
        self._mlp_layers = []
        for i in range(len(layer_sizes) + 1):
            linear = bnn.Linear(sizes[i], sizes[i + 1], weight_std=1.0 / math.sqrt(sizes[i]))
            linear.to(device)
            self.add_module("linear_%d" % i, linear)
            self._mlp_layers.append(linear)
            if i < len(layer_sizes):
                act = tnn.ReLU()
                self.add_module("act_%d" % i, act)
                self._mlp_layers.append(act)

    def forward(self, feat_embeddings):
        y_dnn = feat_embeddings.reshape(-1, self.num_field * self.sparse_feature_dim)
        if bnn.get_matmul_precision() == "bf16x3" and y_dnn.is_cuda:
            # one autograd node: tensor-core GEMMs + fused bias/ReLU/split epilogues (tower.py)
            linears = [m for m in self._mlp_layers if isinstance(m, bnn.Linear)]
            return tower.mlp(y_dnn, [m.weight for m in linears], [m.bias for m in linears])
        for layer in self._mlp_layers:
            y_dnn = layer(y_dnn)
        return y_dnn
