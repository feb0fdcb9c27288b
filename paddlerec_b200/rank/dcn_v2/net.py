"""DCN-V2 network — same classes / constructor arguments / state_dict names as the reference's
models/rank/dcn_v2/net.py (DCN_V2Layer :21-137, DNNLayer :140-184, DeepCrossLayer :187-211,
CrossNetV2 :214-226, CrossNetMix :229-320).

CUDA path: the 26-slot lookup is b200rec_gather (+ sorted segment-reduce backward); every
CrossNetV2 layer is ONE hand-written wgmma GEMM whose epilogue applies bias, Hadamard and residual
and emits the next layer's operand (ops._CrossV2Tc); the MLP is the wgmma tower (tower.py) in
eval mode and per-layer wgmma Linears around the reference's dropouts in train mode.  CrossNetMix is re-associated from the reference's per-sample
[B,in,1] batched GEMVs into three batched GEMMs over all experts (mathematically identical).
Quirks kept (SURVEY.md Q5, Q10, Q13): Dropout(0.5) after every Linear AND every ReLU in train
mode; L2Decay(1e-7) on the DNN weights (applied by the optimizer, optim._apply_regularizers); dense_emb is a full Linear(13 -> 13*D).
"""
from __future__ import annotations

import math

import torch
import torch.nn as tnn
import torch.nn.functional as F

from ... import nn as bnn
from ... import ops
from ... import tower


class DCN_V2Layer(tnn.Module):
    def __init__(self, sparse_feature_number, sparse_feature_dim, dense_feature_dim,
                 sparse_num_field, layer_sizes, cross_num, is_Stacked, use_low_rank_mixture,
                 low_rank, num_experts, device="cuda"):
        super().__init__()
        self.sparse_feature_dim = sparse_feature_dim
        self.dense_feature_dim = dense_feature_dim
        self.sparse_num_field = sparse_num_field
        self.layer_sizes = layer_sizes
        self.is_Stacked = is_Stacked
        std = 0.1 / math.sqrt(float(sparse_feature_dim))
        self.embedding = bnn.Embedding(sparse_feature_number, sparse_feature_dim, padding_idx=0,
                                       init_std=std, device=device)
        self.dense_emb = bnn.Linear(dense_feature_dim, sparse_feature_dim * dense_feature_dim)
        self.DeepCrossLayer_ = DeepCrossLayer(sparse_num_field, sparse_feature_dim,
                                              dense_feature_dim, cross_num, use_low_rank_mixture,
                                              low_rank, num_experts)
        self.DNN_ = DNNLayer(sparse_feature_dim, dense_feature_dim, sparse_num_field, layer_sizes,
                             dropout_rate=0.5)
        in_dim = (dense_feature_dim + sparse_num_field) * sparse_feature_dim
        if is_Stacked:
            self.fc = bnn.Linear(layer_sizes[-1], 1, weight_std=1.0 / math.sqrt(layer_sizes[-1]))
        else:
            self.fc = bnn.Linear(
                layer_sizes[-1] + in_dim, 1,
                weight_std=1.0 / math.sqrt(layer_sizes[-1] + dense_feature_dim * sparse_num_field))
        for m in (self.dense_emb, self.DeepCrossLayer_, self.DNN_, self.fc):
            m.to(device)

    def forward(self, sparse_inputs, dense_inputs):
        ids = (torch.cat(list(sparse_inputs), dim=1) if isinstance(sparse_inputs, (list, tuple))
               else sparse_inputs)
        emb = self.embedding(ids)                                             # net.py:95
        emb = emb.reshape(-1, self.sparse_num_field * self.sparse_feature_dim)
        feat = torch.cat([emb, self.dense_emb(dense_inputs)], 1)              # :103-107
        cross_out = self.DeepCrossLayer_(feat)
        if self.is_Stacked:
            logit = self.fc(self.DNN_(cross_out))
        else:
            logit = self.fc(torch.cat([self.DNN_(feat), cross_out], dim=-1))
        return ops.sum_sigmoid(logit) if logit.is_cuda else torch.sigmoid(logit)


class DNNLayer(tnn.Module):
    def __init__(self, sparse_feature_dim, dense_feature_dim, sparse_num_field, layer_sizes,
                 dropout_rate=0.5):
        super().__init__()
        self.input_size = int((sparse_num_field + dense_feature_dim) * sparse_feature_dim)
        self.drop_out = tnn.Dropout(p=dropout_rate)
        sizes = [self.input_size] + list(layer_sizes)
        self._mlp_layers = []
        for i in range(len(layer_sizes)):
            linear = bnn.Linear(sizes[i], sizes[i + 1], weight_std=1.0 / math.sqrt(sizes[i]),
                                weight_l2_decay=1e-7)   # L2Decay(1e-7), net.py:166-168
            self.add_module("linear_%d" % i, linear)
            self._mlp_layers.append(linear)
            act = tnn.ReLU()
            self.add_module("act_%d" % i, act)
            self._mlp_layers.append(act)

    def forward(self, x):
        if not self.training and bnn.get_matmul_precision() == "bf16x3" and x.is_cuda:
            linears = [m for m in self._mlp_layers if isinstance(m, bnn.Linear)]
            return tower.mlp(x, [m.weight for m in linears], [m.bias for m in linears],
                             last_act=True)
        for layer in self._mlp_layers:        # net.py:178-184: dropout after EVERY sublayer
            x = self.drop_out(layer(x))
        return x


class DeepCrossLayer(tnn.Module):
    def __init__(self, sparse_num_field, sparse_feature_dim, dense_feature_dim, cross_num,
                 use_low_rank_mixture, low_rank, num_experts):
        super().__init__()
        self.input_dim = (sparse_num_field + dense_feature_dim) * sparse_feature_dim
        if use_low_rank_mixture:
            self.crossNet = CrossNetMix(self.input_dim, layer_num=cross_num, low_rank=low_rank,
                                        num_experts=num_experts)
        else:
            self.crossNet = CrossNetV2(self.input_dim, cross_num)

    def forward(self, feat_embeddings):
        return self.crossNet(feat_embeddings)


class CrossNetV2(tnn.Module):
    def __init__(self, input_dim, num_layers):
        super().__init__()
        self.num_layers = num_layers
        self.cross_layers = tnn.ModuleList(bnn.Linear(input_dim, input_dim)
                                           for _ in range(num_layers))

    def forward(self, X_0):
        X_0 = X_0.contiguous()
        X_i, planes = X_0, None
        for layer in self.cross_layers:       # X_i + X_0 * (X_i W + b): GEMM + fused epilogue
            X_i, planes = ops.cross_v2(X_0, X_i, layer.weight, layer.bias, bnn.mm,
                                       bnn.get_matmul_precision() if X_i.is_cuda else "fp32",
                                       xl_planes=planes)
        return X_i


def _xavier_normal(*shape):
    """paddle.nn.initializer.XavierNormal: N(0, 2/(fan_in+fan_out)); for an [E, in, r] parameter
    Paddle's fans are shape[0]*r and shape[1]*r (receptive field = prod(shape[2:]))."""
    rf = 1
    for s in shape[2:]:
        rf *= s
    fan_in, fan_out = shape[0] * rf, shape[1] * rf
    return torch.empty(*shape).normal_(0.0, math.sqrt(2.0 / (fan_in + fan_out)))


class CrossNetMix(tnn.Module):
    """net.py:229-320.  Two evaluation orders of the same mathematics:
      * reference order (per expert, fp32 library batched GEMMs) — exact path, any device;
      * tensor-core order (bf16x3 precision on CUDA): the E projections V_e^T x are ONE
        [B,in]x[in,E*r] GEMM, and because the gate is a per-sample scalar,
            sum_e g_e * (x0 * (U_e v_e + b)) = x0 * ( [g_1 v_1 | .. | g_E v_E] U_cat^T + b )
        (softmax gates sum to 1), i.e. ONE [B,E*r]x[E*r,in] GEMM followed by the very same fused
        K3 epilogue as CrossNetV2.  ~60x fewer fp32-pipe FLOPs than the per-sample GEMV form."""

    def __init__(self, in_features, layer_num=2, low_rank=32, num_experts=4):
        super().__init__()
        self.layer_num, self.num_experts, self.low_rank = layer_num, num_experts, low_rank
        self.U_list = tnn.ParameterList(
            [tnn.Parameter(_xavier_normal(num_experts, in_features, low_rank)) for _ in range(layer_num)])
        self.V_list = tnn.ParameterList(
            [tnn.Parameter(_xavier_normal(num_experts, in_features, low_rank)) for _ in range(layer_num)])
        self.C_list = tnn.ParameterList(
            [tnn.Parameter(_xavier_normal(num_experts, low_rank, low_rank)) for _ in range(layer_num)])
        self.gating = tnn.ModuleList([bnn.Linear(in_features, 1) for _ in range(num_experts)])
        self.bias = tnn.ParameterList(
            [tnn.Parameter(torch.zeros(in_features, 1)) for _ in range(layer_num)])

    def forward(self, inputs):
        if bnn.get_matmul_precision() == "bf16x3" and inputs.is_cuda:
            return self._forward_tensor_core(inputs.contiguous())
        x_0 = inputs
        x_l = inputs
        Wg = torch.cat([g.weight for g in self.gating], dim=1)                 # [in, E]
        bg = torch.cat([g.bias for g in self.gating], dim=0)                   # [E]
        for i in range(self.layer_num):
            gate = torch.softmax(x_l @ Wg + bg, dim=1)                         # net.py:287,315
            v = torch.tanh(torch.einsum("bi,eir->ebr", x_l, self.V_list[i]))   # :291-294
            v = torch.tanh(torch.einsum("ebr,esr->ebs", v, self.C_list[i]))    # :296-297
            u = torch.einsum("ebr,eir->ebi", v, self.U_list[i])                # :300
            dot_ = x_0.unsqueeze(0) * (u + self.bias[i].reshape(1, 1, -1))     # :303-304
            x_l = torch.einsum("ebi,be->bi", dot_, gate) + x_l                 # :314-317
        return x_l

    def _forward_tensor_core(self, x_0):
        E, r = self.num_experts, self.low_rank
        B, C = x_0.shape
        x_l = x_0
        Wg = torch.cat([g.weight for g in self.gating], dim=1)
        bg = torch.cat([g.bias for g in self.gating], dim=0)
        for i in range(self.layer_num):
            gate = torch.softmax(x_l @ Wg + bg, dim=1)                                  # [B,E]
            V_cat = self.V_list[i].permute(1, 0, 2).reshape(C, E * r)                    # [in, E*r]
            v = torch.tanh(ops.split_mm(x_l, V_cat)).reshape(B, E, r)
            v = torch.tanh(torch.einsum("ber,esr->bes", v, self.C_list[i]))              # r x r, fp32
            gv = (v * gate.unsqueeze(2)).reshape(B, E * r)
            U_cat_t = self.U_list[i].permute(0, 2, 1).reshape(E * r, C)                  # [E*r, in]
            xw = ops.split_mm(gv, U_cat_t)
            x_l = ops.cross_combine(x_0, x_l, xw, self.bias[i].reshape(-1))
        return x_l
