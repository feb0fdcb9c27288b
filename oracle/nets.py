"""CPU restatement of the reference's rank networks (TEST INFRASTRUCTURE — see oracle/__init__.py).

Each function follows the reference source op for op, in the reference's execution order, over a
dict of parameters keyed by the reference's state_dict names (SURVEY.md Appendix B).  Tensors are
torch CPU tensors; the dtype is whatever the parameters carry (float32 for timing / fp32 parity,
float64 for golden vectors).  Gradients come from torch autograd, i.e. they are NOT the
hand-derived formulas the CUDA kernels implement.

Paddle semantics encoded here (public API docs; cannot be re-verified: Paddle is not installed):
  Embedding(padding_idx=p): output row all-zero where id==p, no gradient to row p;
  Linear: y = x @ W + b with W [in, out];  log_loss eps = 1e-4;  softmax default axis -1;
  Dropout: identity in eval (parity tests run eval).
"""
from __future__ import annotations

from typing import Dict, List, Sequence

import torch

Params = Dict[str, torch.Tensor]


def embedding(W: torch.Tensor, ids: torch.Tensor, padding_idx=None) -> torch.Tensor:
    """paddle.nn.Embedding forward (lookup_table_v2)."""
    out = W[ids]
    if padding_idx is not None:
        out = out * (ids != padding_idx).unsqueeze(-1).to(W.dtype)
    return out


def linear(x, W, b=None):
    y = x @ W
    return y if b is None else y + b


def log_loss(pred, label, eps=1e-4):
    """paddle.nn.functional.log_loss — models/rank/deepfm/dygraph_model.py:53-58."""
    return -label * torch.log(pred + eps) - (1.0 - label) * torch.log(1.0 - pred + eps)


def bce_with_logits(logit, label):
    """paddle.nn.functional.binary_cross_entropy_with_logits(mean) — din/dygraph_model.py:58-61."""
    return (torch.clamp(logit, min=0) - logit * label + torch.log1p(torch.exp(-logit.abs()))).mean()


# ---------------------------------------------------------------------------------------- DeepFM
def deepfm_fm(p: Params, sparse_inputs: Sequence[torch.Tensor], dense_inputs: torch.Tensor):
    """FM.forward — models/rank/deepfm/net.py:105-139.  Returns (y1, y2, feat)."""
    ids = torch.cat(list(sparse_inputs), dim=1)                                   # :107
    sparse_emb_one = embedding(p["fm.embedding_one.weight"], ids, 0)              # :108  [B,26,1]
    dense_emb_one = (dense_inputs * p["fm.dense_w_one"]).unsqueeze(2)             # :110-111
    y_first_order = sparse_emb_one.sum(1) + dense_emb_one.sum(1)                  # :113-114 [B,1]
    sparse_embeddings = embedding(p["fm.embedding.weight"], ids, 0)               # :117 [B,26,D]
    dense_embeddings = dense_inputs.unsqueeze(2) * p["fm.dense_w"]                # :118-119
    feat = torch.cat([sparse_embeddings, dense_embeddings], 1)                    # :120 [B,39,D]
    summed = feat.sum(1)                                                          # :123
    summed_sq = summed.square()                                                   # :117
    sq_sum = feat.square().sum(1)                                                 # :129-132
    y_second_order = 0.5 * (summed_sq - sq_sum).sum(1, keepdim=True)              # :134-137
    return y_first_order, y_second_order, feat


def mlp_relu(p: Params, prefix: str, x: torch.Tensor, n_layers: int, last_act: bool = False):
    """Linear/ReLU stack with `linear_%d` names (DNN of deepfm/net.py:152-174, wide_deep :55-71)."""
    for i in range(n_layers):
        x = linear(x, p["%slinear_%d.weight" % (prefix, i)], p["%slinear_%d.bias" % (prefix, i)])
        if i < n_layers - 1 or last_act:
            x = torch.relu(x)
    return x


def deepfm_forward(p: Params, sparse_inputs, dense_inputs, n_fc: int):
    """DeepFMLayer.forward — net.py:41-49 (`bias` is never used)."""
    y1, y2, feat = deepfm_fm(p, sparse_inputs, dense_inputs)
    B = feat.shape[0]
    y_dnn = mlp_relu(p, "dnn.", feat.reshape(B, -1), n_fc + 1)                    # :169-174
    return torch.sigmoid(y1 + y2 + y_dnn)


# ---------------------------------------------------------------------------------------- DCN-V2
def cross_net_v2(p: Params, prefix: str, x0, num_layers: int):
    """CrossNetV2.forward — models/rank/dcn_v2/net.py:222-226."""
    xi = x0
    for i in range(num_layers):
        xi = xi + x0 * linear(xi, p["%scross_layers.%d.weight" % (prefix, i)],
                              p["%scross_layers.%d.bias" % (prefix, i)])
    return xi


def cross_net_mix(p: Params, prefix: str, inputs, layer_num: int, num_experts: int):
    """CrossNetMix.forward — models/rank/dcn_v2/net.py:278-320 (squeeze on axis 2 only, Q13)."""
    x_0 = inputs.unsqueeze(2)
    x_l = x_0
    for i in range(layer_num):
        outs, gates = [], []
        for e in range(num_experts):
            gates.append(linear(x_l.squeeze(2), p["%sgating.%d.weight" % (prefix, e)],
                                p["%sgating.%d.bias" % (prefix, e)]))             # :287
            v_x = torch.matmul(p["%sV_list.%d" % (prefix, i)][e].t(), x_l)        # :291
            v_x = torch.tanh(v_x)
            v_x = torch.matmul(p["%sC_list.%d" % (prefix, i)][e], v_x)            # :296
            v_x = torch.tanh(v_x)
            uv_x = torch.matmul(p["%sU_list.%d" % (prefix, i)][e], v_x)           # :300
            dot_ = uv_x + p["%sbias.%d" % (prefix, i)]                            # :303
            dot_ = x_0 * dot_                                                     # :304
            outs.append(dot_.squeeze(2))
        outs = torch.stack(outs, 2)                                               # [B,in,E]
        gates = torch.stack(gates, 1)                                             # [B,E,1]
        moe_out = torch.matmul(outs, torch.softmax(gates, dim=1))                 # :314-316
        x_l = moe_out + x_l
    return x_l.squeeze(2)


def dcn_v2_forward(p: Params, sparse_inputs, dense_inputs, *, n_fc: int, cross_num: int,
                   is_stacked: bool, use_low_rank_mixture: bool, num_experts: int = 4):
    """DCN_V2Layer.forward — models/rank/dcn_v2/net.py:89-137, eval mode (Dropout = identity)."""
    ids = torch.cat(list(sparse_inputs), dim=1)
    emb = embedding(p["embedding.weight"], ids, 0)                                # :95
    B = emb.shape[0]
    emb = emb.reshape(B, -1)                                                      # :99-101
    dense_emb = linear(dense_inputs, p["dense_emb.weight"], p["dense_emb.bias"])  # :103-104
    feat = torch.cat([emb, dense_emb], 1)                                         # :106-107
    pre = "DeepCrossLayer_.crossNet."
    cross = (cross_net_mix(p, pre, feat, cross_num, num_experts) if use_low_rank_mixture
             else cross_net_v2(p, pre, feat, cross_num))
    if is_stacked:
        dnn_out = mlp_relu(p, "DNN_.", cross, n_fc, last_act=True)                # :178-184
        logit = linear(dnn_out, p["fc.weight"], p["fc.bias"])
    else:
        dnn_out = mlp_relu(p, "DNN_.", feat, n_fc, last_act=True)
        logit = linear(torch.cat([dnn_out, cross], -1), p["fc.weight"], p["fc.bias"])
    return torch.sigmoid(logit)


# ------------------------------------------------------------------------------------------- DIN
def din_attention_unit(hist, tseq, mask, W1, b1, W2, b2, W3, b3):
    """The attention unit alone — models/rank/din/net.py:155-173: concat [h, t, h-t, h*t], the
    512->80->40->1 sigmoid MLP, mask added BEFORE the E^-0.5 scaling (Q7), softmax over the
    history, weighted sum.  hist [B,L,E], tseq [B,E] (the target tiled over L by the reader,
    dinReader.py:85-90), mask [B,L,1] in {0,-1e9} or None.  Checker for the fused K4 kernels."""
    E = hist.shape[2]
    t = tseq.unsqueeze(1).expand_as(hist)
    concat = torch.cat([hist, t, hist - t, hist * t], dim=2)                      # :155-161
    x = torch.sigmoid(linear(concat, W1, b1))                                     # :163-164
    x = torch.sigmoid(linear(x, W2, b2))
    x = linear(x, W3, b3)
    if mask is not None:
        x = x + mask.reshape(x.shape).to(x.dtype)                                 # :166
    weight = torch.softmax(x.transpose(1, 2) * (E ** -0.5), dim=-1)               # :167-169
    return torch.matmul(weight, hist).reshape(-1, E)                              # :171-173


def din_forward(p: Params, hist_item_seq, hist_cat_seq, target_item, target_cat, label, mask,
                target_item_seq, target_cat_seq):
    """DINLayer.forward — models/rank/din/net.py:139-184.  `att.*` are the attention-unit linears
    that the reference's sub-layer name collision hides from its state_dict (SURVEY.md Q6)."""
    hist_item_emb = embedding(p["hist_item_emb_attr.weight"], hist_item_seq)
    hist_cat_emb = embedding(p["hist_cat_emb_attr.weight"], hist_cat_seq)
    target_item_emb = embedding(p["target_item_emb_attr.weight"], target_item)
    target_cat_emb = embedding(p["target_cat_emb_attr.weight"], target_cat)
    target_item_seq_emb = embedding(p["target_item_seq_emb_attr.weight"], target_item_seq)
    target_cat_seq_emb = embedding(p["target_cat_seq_emb_attr.weight"], target_cat_seq)
    item_b = embedding(p["item_b_attr.weight"], target_item)                      # :147
    hist = torch.cat([hist_item_emb, hist_cat_emb], 2)                            # :149
    tseq = torch.cat([target_item_seq_emb, target_cat_seq_emb], 2)                # :150-151
    target = torch.cat([target_item_emb, target_cat_emb], 1)                      # :152-153
    concat = torch.cat([hist, tseq, hist - tseq, hist * tseq], 2)                 # :155-161
    x = concat
    for i in range(3):                                                            # :163-164
        x = linear(x, p["att.linear_%d.weight" % i], p["att.linear_%d.bias" % i])
        if i < 2:
            x = torch.sigmoid(x)
    E = hist.shape[2]
    atten = x + mask.to(x.dtype)                                                  # :166
    atten = atten.transpose(1, 2)                                                 # :167
    atten = atten * (E ** -0.5)                                                   # :168
    weight = torch.softmax(atten, dim=-1)                                         # :169
    output = torch.matmul(weight, hist).reshape(-1, E)                            # :171-173
    con = linear(output, p["linearCon.weight"], p["linearCon.bias"])              # :175-176
    x = torch.cat([con, target], 1)                                               # :178
    for i in range(3):                                                            # :180-181
        x = linear(x, p["linear_%d.weight" % i], p["linear_%d.bias" % i])
        if i < 2:
            x = torch.sigmoid(x)
    return x + item_b                                                             # :183


# ------------------------------------------------------------------------------------- Wide&Deep
def wide_deep_forward(p: Params, sparse_inputs, dense_inputs, n_fc: int):
    """WideDeepLayer.forward — models/rank/wide_deep/net.py:73-101 (non-gpubox branch)."""
    wide = linear(dense_inputs, p["wide_part.weight"], p["wide_part.bias"])       # :75
    D = p["embedding.weight"].shape[1]
    embs = [embedding(p["embedding.weight"], s).reshape(-1, D) for s in sparse_inputs]  # :90-93
    deep = torch.cat(embs + [dense_inputs], 1)                                    # :95
    deep = mlp_relu(p, "", deep, n_fc + 1)                                        # :96-97
    return torch.sigmoid(wide + deep)                                             # :99-101


def wide_deep_forward_gpubox(p: Params, sparse_inputs, dense_inputs, n_fc: int):
    """WideDeepLayer.forward, `sync_mode == "gpubox"` branch — models/rank/wide_deep/net.py:80-88:
    the table rows are [show, click, embedding(D)] (sparse_embedding size [V, D+2]) and every
    looked-up row goes through continuous_value_model(emb, show_click, use_cvm=False), which keeps
    only the embedding columns in forward.  (Its backward writes the sample's show/click into the
    two dropped gradient columns: cvm_grad — checked separately, it is not a derivative.)"""
    wide = linear(dense_inputs, p["wide_part.weight"], p["wide_part.bias"])       # :75
    D = p["embedding.weight"].shape[1] - 2
    embs = [cvm(embedding(p["embedding.weight"], s).reshape(-1, D + 2), False)     # :81-88
            for s in sparse_inputs]
    deep = torch.cat(embs + [dense_inputs], 1)                                    # :95
    deep = mlp_relu(p, "", deep, n_fc + 1)                                        # :96-97
    return torch.sigmoid(wide + deep)                                             # :99-101


def cvm(emb_with_show_click: torch.Tensor, use_cvm: bool) -> torch.Tensor:
    """continuous_value_model forward (wide_deep/net.py:87-88): input [N, D+2] whose first two
    columns are show/click.  use_cvm=False drops them; True maps them to
    log(show+1), log(click+1)-log(show+1)."""
    if not use_cvm:
        return emb_with_show_click[:, 2:]
    show = torch.log(emb_with_show_click[:, 0:1] + 1.0)
    click = torch.log(emb_with_show_click[:, 1:2] + 1.0) - show
    return torch.cat([show, click, emb_with_show_click[:, 2:]], 1)


# ---- DLRM (models/rank/dlrm/net.py) ---------------------------------------------------------------
def batch_norm_train(x, weight, bias, eps=1e-5):
    """paddle.nn.BatchNorm1D in train mode (public API docs): per-feature batch mean and BIASED
    batch variance, y = (x - mu) / sqrt(var + eps) * weight + bias."""
    mu = x.mean(0, keepdim=True)
    var = ((x - mu) ** 2).mean(0, keepdim=True)
    return (x - mu) / torch.sqrt(var + eps) * weight + bias


def batch_norm_running(mean, var, x, momentum=0.9):
    """Running statistics after one train step: moving = moving*momentum + batch*(1-momentum), with
    the biased batch variance (paddle.nn.BatchNorm1D docs)."""
    mu = x.mean(0)
    bv = ((x - mu) ** 2).mean(0)
    return mean * momentum + mu * (1 - momentum), var * momentum + bv * (1 - momentum)


def dlrm_mlp(p: Params, prefix: str, x, n_layers: int):
    """MLPLayer.forward — dlrm/net.py:121-171.  The guard `i != len(units_list) - 1` (:135) is true
    for every i of enumerate(units_list[:-1]), so EVERY layer, the last included, is
    Linear -> ReLU -> BatchNorm1D and the `else` branch (:152-165) never runs."""
    for i in range(n_layers):
        x = linear(x, p["%sdense_%d.weight" % (prefix, i)], p["%sdense_%d.bias" % (prefix, i)])
        x = torch.relu(x)
        x = batch_norm_train(x, p["%snorm_%d.weight" % (prefix, i)], p["%snorm_%d.bias" % (prefix, i)])
    return x


def dot_interact(T, self_interaction: bool = False):
    """net.py:103-115 on T [B, N, d] (x = last row): Z = T T^T; the strict upper triangle in
    row-major order — with self_interaction the diagonal positions are selected too but hold 0,
    because triu(Z, 1) has already zeroed them (:105-113); R = concat([x, Zflat]) (:115)."""
    B, N, d = T.shape
    Z = torch.bmm(T, T.transpose(1, 2))
    iu = torch.triu_indices(N, N, 0 if self_interaction else 1, device=T.device)
    flat = Z[:, iu[0], iu[1]]
    if self_interaction:
        flat = torch.where((iu[0] == iu[1]).unsqueeze(0), torch.zeros((), dtype=T.dtype, device=T.device), flat)
    return torch.cat([T[:, N - 1, :], flat], 1)


def dlrm_forward(p: Params, sparse_inputs, dense_inputs, *, n_bot: int, n_top: int,
                 self_interaction: bool = False):
    """DLRMLayer.forward — dlrm/net.py:76-118.  Returns the raw [B, 2] scores (train mode)."""
    x = dlrm_mlp(p, "bot_mlp.", dense_inputs, n_bot)                               # :86
    d = x.shape[1]
    embs = [embedding(p["embedding.weight"], s).reshape(-1, d) for s in sparse_inputs]  # :89-94
    T = torch.cat(embs + [x], 1).reshape(x.shape[0], len(embs) + 1, d)             # :97-100
    R = dot_interact(T, self_interaction)                                          # :103-115
    return dlrm_mlp(p, "top_mlp.", R, n_top)                                       # :117


def softmax_cross_entropy(logits, label):
    """paddle.nn.functional.cross_entropy(input, label) with hard int64 labels [B,1], mean
    (dlrm/dygraph_model.py:58-62)."""
    lse = torch.logsumexp(logits, 1)
    picked = logits.gather(1, label.reshape(-1, 1).to(torch.int64)).squeeze(1)
    return (lse - picked).mean()
