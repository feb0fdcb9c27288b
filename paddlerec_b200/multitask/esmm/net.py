"""ESMM network — same class, constructor arguments, outputs, initialisers and state_dict names as
the reference's models/multitask/esmm/net.py (ESMMLayer :21-111).

  23 lookups + sum pool + concat (:88-95)   ONE pooled gather each way (Embedding.forward_pooled:
                                            every field is a bag of max_len ids; id 0 is padding)
  two Linear/ReLU towers (:97-107)          'bf16x3': the wgmma tower (tower.mlp, last_act=True) once
                                            per tower on the same pooled input; 'fp32' / 'tf32':
                                            bnn.Linear layers
  softmax x2, slice, multiply, concat       ONE fused kernel each way on CUDA (ops.esmm_head); off
  (:99-111)                                 CUDA the reference's op sequence in torch

Reference behaviour kept on purpose (SURVEY.md Q19): the CVR tower learns only through the product
ctcvr_one = ctr_one * cvr_one; both towers register their ReLUs as `act_%d`, so the CVR tower's
overwrite the CTR tower's (no parameters, no effect); the table is Uniform(-1, 1) with row 0 zeroed
as the padding row.
"""
from __future__ import annotations

import math

import torch
import torch.nn as tnn

from ... import nn as bnn
from ... import ops
from ... import tower


def torch_head(h_ctr, h_cvr, W_ctr, b_ctr, W_cvr, b_cvr):
    """The reference's head (:97-111) as torch ops: the six outputs from the last hidden layers."""
    ctr_out = torch.softmax(h_ctr @ W_ctr + b_ctr, dim=-1)
    cvr_out = torch.softmax(h_cvr @ W_cvr + b_cvr, dim=-1)
    ctr_one = ctr_out[:, 1:2]
    cvr_one = cvr_out[:, 1:2]
    ctcvr_one = ctr_one * cvr_one
    ctcvr_prop = torch.cat([1 - ctcvr_one, ctcvr_one], dim=1)
    return ctr_out, ctr_one, cvr_out, cvr_one, ctcvr_prop, ctcvr_one


class ESMMLayer(tnn.Module):
    def __init__(self, sparse_feature_number, sparse_feature_dim, num_field, ctr_layer_sizes,
                 cvr_layer_sizes, device="cuda"):
        super().__init__()
        self.sparse_feature_number = sparse_feature_number
        self.sparse_feature_dim = sparse_feature_dim
        self.num_field = num_field
        self.ctr_layer_sizes = list(ctr_layer_sizes)
        self.cvr_layer_sizes = list(cvr_layer_sizes)
        self.embedding = bnn.Embedding(sparse_feature_number, sparse_feature_dim,     # :33-40
                                       padding_idx=0, init="uniform", device=device)
        self._ctr_linears = self._tower(self.ctr_layer_sizes, 0, device)              # :42-59
        self._cvr_linears = self._tower(self.cvr_layer_sizes,                         # :61-79
                                        len(self.ctr_layer_sizes) + 1, device)

    def _tower(self, layer_sizes, first, device):
        sizes = [self.sparse_feature_dim * self.num_field] + layer_sizes + [2]
        linears = []
        for i in range(len(layer_sizes) + 1):
            linear = bnn.Linear(sizes[i], sizes[i + 1],
                                weight_std=1.0 / math.sqrt(sizes[i])).to(device)
            self.add_module("linear_%d" % (first + i), linear)
            linears.append(linear)
            if i < len(layer_sizes):
                self.add_module("act_%d" % i, tnn.ReLU())    # both towers use act_%d (Q19)
        return linears

    def pooled_input(self, inputs):
        """[B, num_field * D]: each field's ids summed over its bag (:88-95).  `inputs` is the
        reference's list of num_field [B, max_len] tensors or one [B, num_field, max_len] tensor."""
        ids = torch.stack(list(inputs), dim=1) if isinstance(inputs, (list, tuple)) else inputs
        B, F, L = ids.shape
        offsets = torch.arange(0, B * F * L + 1, L, dtype=torch.int64, device=ids.device)
        x = self.embedding.forward_pooled(ids.reshape(-1), offsets)
        return x.reshape(B, F * self.sparse_feature_dim)

    @staticmethod
    def _hidden(x, linears):
        hidden = linears[:-1]
        if hidden and bnn.get_matmul_precision() == "bf16x3" and x.is_cuda:
            return tower.mlp(x, [m.weight for m in hidden], [m.bias for m in hidden], last_act=True)
        for m in hidden:
            x = torch.relu(m(x))
        return x

    def forward(self, inputs):
        """(ctr_out, ctr_prop_one, cvr_out, cvr_prop_one, ctcvr_prop, ctcvr_prop_one), as :111."""
        x = self.pooled_input(inputs)
        h_ctr = self._hidden(x, self._ctr_linears)
        h_cvr = self._hidden(x, self._cvr_linears)
        lc, lv = self._ctr_linears[-1], self._cvr_linears[-1]
        head = ops.esmm_head if x.is_cuda else torch_head
        return head(h_ctr, h_cvr, lc.weight, lc.bias, lv.weight, lv.bias)
