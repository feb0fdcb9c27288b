"""CPU restatement of the reference's FFM network (TEST INFRASTRUCTURE, like oracle/nets.py, whose
`embedding` and conventions it uses): models/rank/ffm/net.py op for op, in the reference's order,
over a dict of parameters keyed by the reference's state_dict names.  Pinned to the goldens minted
from the reference's own net.py (tests/golden/make_ffm_golden.py, tests/test_ffm.py)."""
from __future__ import annotations

import sys

import torch

from oracle import nets


def ffm_terms(p, sparse_inputs, dense_inputs, num_field: int):
    """FFM.forward — models/rank/ffm/net.py:99-133 (no padding_idx).  Returns (y1, y2) [B,1]."""
    ids = torch.cat(list(sparse_inputs), dim=1)                                   # :101
    sparse_emb_one = nets.embedding(p["ffm.embedding_one.weight"], ids)           # :102
    dense_emb_one = (dense_inputs * p["ffm.dense_w_one"]).unsqueeze(2)            # :104-105
    y_first_order = sparse_emb_one.sum(1) + dense_emb_one.sum(1)                  # :107-108
    sparse_embeddings = nets.embedding(p["ffm.embedding.weight"], ids)            # :111
    dense_embeddings = dense_inputs.unsqueeze(2) * p["ffm.dense_w"]               # :112-113
    feat = torch.cat([sparse_embeddings, dense_embeddings], 1)                    # :114-115
    D = feat.shape[2] // num_field
    fa = feat.reshape(-1, num_field, num_field, D)                                # :117-122
    terms = []
    for i in range(num_field):                                                    # :124-130
        for j in range(i + 1, num_field):
            terms.append((fa[:, i, j, :] * fa[:, j, i, :]).sum(1, keepdim=True))
    y_second_order = add_n(terms)                                                 # :132
    return y_first_order, y_second_order


def ffm_forward(p, sparse_inputs, dense_inputs, num_field: int):
    """FFMLayer.forward — ffm/net.py:39-46: the bias IS added (unlike DeepFM's)."""
    y1, y2 = ffm_terms(p, sparse_inputs, dense_inputs, num_field)
    return torch.sigmoid(y1 + y2 + p["bias"])                                     # :44


def add_n(inputs):
    """paddle.add_n: the element-wise sum of a list of same-shaped tensors (public API docs)."""
    return torch.stack(list(inputs), 0).sum(0)


def install_add_n():
    """Give the paddle shim (oracle/paddle_shim.py, installed first) the one API that ffm/net.py
    needs beyond the other rank models, so the reference's ffm/net.py runs on it unmodified."""
    paddle = sys.modules["paddle"]
    paddle.add_n = add_n
    return paddle
