"""FFM network — same classes, constructor arguments, forward signature, initialisers and state_dict
names as the reference's models/rank/ffm/net.py (FFMLayer :22-46, FFM :49-133), with the gather and
the field-aware second-order term replaced by ONE fused sm_90a kernel each way
(b200rec_ffm_fwd / _bwd).

`sparse_num_field` is the TOTAL number of fields NF (the reference's dygraph_model passes
sparse_inputs_slots - 1 + dense_input_dim); the 26 sparse slots are NF - dense_feature_dim of them.
Both tables live in one bnn.FusedTable of rows [NF*D emb | w1 | pad]; its state_dict still shows
`ffm.embedding.weight` [V, NF*D] and `ffm.embedding_one.weight` [V, 1].

Reference behaviour kept on purpose (SURVEY.md Appendix C): no padding_idx (id 0 is a real row);
`dense_w_one` and `dense_w` start at 1.0, which saturates the sigmoid on many Criteo rows at
initialisation; `bias` IS added to the logit here (unlike DeepFM's).
"""
from __future__ import annotations

import math

import torch
import torch.nn as tnn

from ... import nn as bnn
from ... import ops


class FFMLayer(tnn.Module):
    def __init__(self, sparse_feature_number, sparse_feature_dim, dense_feature_dim,
                 sparse_num_field, device="cuda"):
        super().__init__()
        self.sparse_feature_number = sparse_feature_number
        self.sparse_feature_dim = sparse_feature_dim
        self.dense_feature_dim = dense_feature_dim
        self.sparse_num_field = sparse_num_field
        self.ffm = FFM(sparse_feature_number, sparse_feature_dim, dense_feature_dim,
                       sparse_num_field, device=device)
        self.bias = tnn.Parameter(torch.zeros(1, device=device))              # net.py:34-37

    def forward(self, sparse_inputs, dense_inputs):
        # net.py:41-44: sigmoid(y_first_order + y_second_order + bias); the bias rides in y1
        y1, y2 = self.ffm.terms(sparse_inputs, dense_inputs, self.bias)
        if y1.is_cuda:
            return ops.sum_sigmoid(y1, y2)
        return torch.sigmoid(y1 + y2)


class FFM(bnn.FusedTableOwner):
    def __init__(self, sparse_feature_number, sparse_feature_dim, dense_feature_dim,
                 sparse_num_field, device="cuda"):
        super().__init__()
        self.sparse_feature_number = sparse_feature_number
        self.sparse_feature_dim = sparse_feature_dim
        self.dense_feature_dim = dense_feature_dim
        self.dense_emb_dim = sparse_feature_dim
        self.sparse_num_field = sparse_num_field
        self.init_value_ = 0.1
        std = self.init_value_ / math.sqrt(float(sparse_feature_dim))
        R = sparse_feature_dim * sparse_num_field
        # net.py:65-83 — embedding_one [V,1] and embedding [V, NF*D], TruncatedNormal(0, 0.1/sqrt(D))
        self._fused = bnn.FusedTable(sparse_feature_number, R, padding_idx=None, init_std=std,
                                     device=device)
        # net.py:86-97 — Constant(1.0)
        self.dense_w_one = tnn.Parameter(torch.ones(dense_feature_dim, device=device))
        self.dense_w = tnn.Parameter(torch.ones(1, dense_feature_dim, R, device=device))

    def terms(self, sparse_inputs, dense_inputs, bias=None):
        """(y1 [B,1] (+ bias), y2 [B,1]) — net.py:101-132 as one kernel."""
        if isinstance(sparse_inputs, (list, tuple)):
            ids = torch.cat(list(sparse_inputs), dim=1)                        # net.py:101
        else:
            ids = sparse_inputs
        return ops.ffm(self._fused.weight, ids, dense_inputs, self.dense_w, self.dense_w_one, bias,
                       self._fused.pad, self._fused, self.sparse_feature_dim)

    def forward(self, sparse_inputs, dense_inputs):
        return self.terms(sparse_inputs, dense_inputs)

    def table_grad_dense(self):
        """(dW [V, NF*D], dW1 [V,1]) dense gradients of the two tables (tests / small tables)."""
        return self._fused.grad_dense()
