"""FAT-DeepFFM network — same classes, constructor arguments, forward signatures, initialisers and
state_dict names as the reference's models/rank/fat_deepffm/net.py (FAT_DeepFFMLayer :22-57,
CENLayer :60-151, DNNLayer :154-208, DeepFFM :211-251), with the gather, CENet's max pool and
attention product and the field-aware Hadamard pairs replaced by fused sm_90a kernels
(b200rec_fat_ffm_*).

The table is one bnn.FusedTable in FFM's layout with a single name: rows [NF*D emb | 0 | pad],
state_dict `cen.embedding.weight` [V, NF*D].  CENLayer.forward returns the attention weights and
the gather context instead of the [B, NF*NF, D] weighted embeddings, and DeepFFM.forward consumes
that pair, so nothing of size [B, NF, NF*D] is formed.  The attention MLP (two NF^2 x NF^2 Linears)
and the DNN are GEMMs: the wgmma tower under bf16x3 on CUDA, bnn.Linear otherwise.

Reference behaviour kept on purpose (SURVEY.md Q17): no padding_idx (id 0 is a real row);
`dense_w` starts at 1.0; Dropout(0.5) after every DNN sublayer, the logit included; the max pool's
gradient goes to the FIRST maximum of each block.
"""
from __future__ import annotations

import collections
import math

import torch
import torch.nn as tnn

from ... import nn as bnn
from ... import ops
from ... import tower


class FAT_DeepFFMLayer(tnn.Module):
    def __init__(self, sparse_feature_number, sparse_feature_dim, dense_feature_dim,
                 sparse_num_field, layer_sizes, device="cuda"):
        super().__init__()
        self.sparse_feature_number = sparse_feature_number
        self.sparse_feature_dim = sparse_feature_dim
        self.dense_feature_dim = dense_feature_dim
        self.sparse_num_field = sparse_num_field
        self.layer_sizes = layer_sizes
        self.num_fields = sparse_num_field + dense_feature_dim
        self.cen = CENLayer(sparse_feature_number, dense_feature_dim, self.num_fields,
                            sparse_feature_dim, reduction=1, device=device)
        self.dnn = DNNLayer(sparse_feature_number, sparse_feature_dim, dense_feature_dim,
                            sparse_num_field, layer_sizes)
        self.deepffm = DeepFFM(sparse_feature_number, sparse_feature_dim, dense_feature_dim,
                               sparse_num_field)
        self.bias = tnn.Parameter(torch.zeros(1, device=device))              # net.py:43-46
        self.dnn.to(device)

    def forward(self, sparse_inputs, dense_inputs):
        cen_out = self.cen(sparse_inputs, dense_inputs, bias=self.bias)       # net.py:50
        y_first_order, dnn_input = self.deepffm(cen_out, bias=self.bias)      # :52, bias rides in y1
        y_dnn = self.dnn(dnn_input)                                           # :54
        if y_dnn.is_cuda:                                                     # :56
            return ops.sum_sigmoid(y_first_order, y_dnn)
        return torch.sigmoid(y_first_order + y_dnn)


class CENLayer(bnn.FusedTableOwner):
    def __init__(self, sparse_feature_number, dense_feature_dim, num_fields, sparse_feature_dim,
                 reduction=8, activation=None, device="cuda"):
        super().__init__()
        self.feature_dim = sparse_feature_dim
        self.num_fields = num_fields
        self.sparse_feature_number = sparse_feature_number
        self.dense_feature_dim = dense_feature_dim
        self.init_value_ = 0.1
        R = sparse_feature_dim * num_fields
        # net.py:76-84 — embedding [V, NF*D], TruncatedNormal(0, 0.1/sqrt(D)), no padding_idx
        self._fused = bnn.FusedTable(sparse_feature_number, R, padding_idx=None,
                                     init_std=self.init_value_ / math.sqrt(float(sparse_feature_dim)),
                                     device=device, names=("embedding.weight",))
        # net.py:87-92 — Constant(1.0)
        self.dense_w = tnn.Parameter(torch.ones(1, dense_feature_dim, R, device=device))
        inputs_num_fields = num_fields * num_fields
        reduced_num_fields = inputs_num_fields // reduction
        # net.py:94-103 — paddle.nn.Linear defaults (XavierUniform weight, zero bias)
        self.fc = tnn.Sequential(collections.OrderedDict([
            ("ReductionLinear", bnn.Linear(inputs_num_fields, reduced_num_fields)),
            ("ReductionActivation", tnn.ReLU()),
            ("AdditionLinear", bnn.Linear(reduced_num_fields, inputs_num_fields)),
            ("AdditionActivation", tnn.ReLU()),
        ])).to(device)

    def forward(self, sparse_inputs, dense_inputs, bias=None):
        """-> (attn [B, NF*NF], link): the attention weights of net.py:137 and the gather context
        that DeepFFM applies them with (the reference returns their product, [B, NF*NF, D]).
        `bias` (FAT_DeepFFMLayer's) is passed so that its gradient comes from the one table pass."""
        if isinstance(sparse_inputs, (list, tuple)):
            ids = torch.cat(list(sparse_inputs), dim=1)                      # net.py:108-109
        else:
            ids = sparse_inputs
        link = ops.FatLink(self._fused.weight, ids, dense_inputs, self.dense_w, self._fused.pad,
                           self._fused, self.feature_dim)
        pooled = ops.fat_ffm_pool(link, self.dense_w, bias)                  # :107-132
        return self.attention(pooled), link                                  # :137

    def attention(self, pooled):
        """relu(relu(pooled @ W1 + b1) @ W2 + b2) — self.fc of net.py:98-103."""
        if bnn.get_matmul_precision() == "bf16x3" and pooled.is_cuda:
            lin = (self.fc.ReductionLinear, self.fc.AdditionLinear)
            return tower.mlp(pooled, [m.weight for m in lin], [m.bias for m in lin], last_act=True)
        return self.fc(pooled)

    def table_grad_dense(self):
        """dW [V, NF*D], the dense gradient of the table (tests / small tables)."""
        return self._fused.grad_dense()[0]


class DNNLayer(tnn.Module):
    def __init__(self, sparse_feature_number, sparse_feature_dim, dense_feature_dim,
                 sparse_num_field, layer_sizes, dropout_rate=0.5, is_H=True):
        super().__init__()
        self.sparse_feature_dim = sparse_feature_dim
        self.dense_feature_dim = dense_feature_dim
        self.num_field = dense_feature_dim + sparse_num_field
        self.layer_sizes = layer_sizes
        self.sparse_num_field = sparse_num_field
        self.is_H = is_H
        if not is_H:
            raise NotImplementedError("only the Hadamard interaction (is_H=True) is built")
        self.input_size = int(sparse_feature_dim * self.num_field * (self.num_field - 1) / 2)
        self.drop_out = tnn.Dropout(p=dropout_rate)
        sizes = [self.input_size] + list(layer_sizes) + [1]
        self._mlp_layers = []
        for i in range(len(layer_sizes) + 1):
            linear = bnn.Linear(sizes[i], sizes[i + 1], weight_std=1.0 / math.sqrt(sizes[i]),
                                weight_l2_decay=1e-7)   # L2Decay(1e-7), net.py:187-193
            self.add_module("linear_%d" % i, linear)
            self._mlp_layers.append(linear)
            if i < len(layer_sizes):
                act = tnn.ReLU()
                self.add_module("act_%d" % i, act)
                self._mlp_layers.append(act)

    def forward(self, feat_embeddings):
        y_dnn = feat_embeddings.reshape(feat_embeddings.shape[0], -1)
        if not self.training and bnn.get_matmul_precision() == "bf16x3" and y_dnn.is_cuda:
            linears = [m for m in self._mlp_layers if isinstance(m, bnn.Linear)]
            return tower.mlp(y_dnn, [m.weight for m in linears], [m.bias for m in linears])
        for layer in self._mlp_layers:   # net.py:204-208: dropout after EVERY sublayer, logit too
            y_dnn = self.drop_out(layer(y_dnn))
        return y_dnn


class DeepFFM(tnn.Module):
    def __init__(self, sparse_feature_number, sparse_feature_dim, dense_feature_dim,
                 sparse_num_field, is_H=True):
        super().__init__()
        self.num_field = sparse_num_field + dense_feature_dim
        self.sparse_feature_dim = sparse_feature_dim
        self.is_H = is_H

    def forward(self, feat_embedding, bias=None):
        """feat_embedding = CENLayer's (attn, link).  -> (y_first_order [B,1] (+ bias),
        y_field_aware_out [B, P*D]) of net.py:219-251 as one kernel."""
        attn, link = feat_embedding
        return ops.fat_ffm_interact(link, attn, bias)
