"""CPU restatement of the reference's FAT-DeepFFM network (TEST INFRASTRUCTURE, like oracle/nets.py,
whose `embedding` and conventions it uses): models/rank/fat_deepffm/net.py op for op, in the
reference's order, over a dict of parameters keyed by the reference's state_dict names, in eval
mode (Dropout is the identity).  Pinned to the goldens minted from the reference's own net.py
(tests/golden/make_fat_deepffm_golden.py, tests/test_fat_deepffm.py)."""
from __future__ import annotations

import sys

import torch

from oracle import nets


def adaptive_max_pool1d_to_1(x):
    """paddle.nn.AdaptiveMaxPool1D(output_size=1) on [N, C, L] -> [N, C, 1].  The gradient goes to
    the FIRST maximum of each row (torch's CPU adaptive_max_pool1d and Paddle's public
    max_pool2d_with_index kernel both keep the first index on ties)."""
    first = (x == x.max(-1, keepdim=True).values).to(torch.int8).argmax(-1, keepdim=True)
    return torch.gather(x, -1, first)


def cen(p, sparse_inputs, dense_inputs, num_fields):
    """CENLayer.forward — fat_deepffm/net.py:105-151 (no padding_idx)."""
    ids = torch.cat(list(sparse_inputs), dim=1)                                   # :108-109
    sparse_embeddings = nets.embedding(p["cen.embedding.weight"], ids)            # :110-112
    dense_embeddings = dense_inputs.unsqueeze(2) * p["cen.dense_w"]               # :116-117
    feat = torch.cat([sparse_embeddings, dense_embeddings], 1)                    # :119-121
    D = feat.shape[2] // num_fields
    feat = feat.reshape(-1, num_fields * num_fields, D)                           # :122-124
    pooled = adaptive_max_pool1d_to_1(feat)                                       # :128
    pooled = torch.flatten(pooled, 1, -1)                                         # :133-134
    h = torch.relu(nets.linear(pooled, p["cen.fc.ReductionLinear.weight"],         # :137
                               p["cen.fc.ReductionLinear.bias"]))
    attn_w = torch.relu(nets.linear(h, p["cen.fc.AdditionLinear.weight"], p["cen.fc.AdditionLinear.bias"]))
    attn_w = tile(attn_w, [D])                                                    # :144
    attn_w = split(attn_w, D, 1)                                                  # :145
    attn_w = torch.stack(attn_w, 2)                                               # :146
    return feat * attn_w                                                          # :149


def deepffm(outputs, num_field, D):
    """DeepFFM.forward — fat_deepffm/net.py:219-251 (is_H=True)."""
    y_first_order = outputs.sum(2).sum(1, keepdim=True)                           # :221-222
    fa = outputs.reshape(-1, num_field, num_field, D)                             # :226-228
    terms = []
    for i in range(num_field):                                                    # :230-246
        for j in range(i + 1, num_field):
            terms.append(fa[:, i, j, :] * fa[:, j, i, :])
    return y_first_order, torch.cat(terms, 1)                                     # :250


def dnn(p, x, n_layers):
    """DNNLayer.forward in eval mode — fat_deepffm/net.py:204-208."""
    y = x.reshape(x.shape[0], -1)
    for i in range(n_layers):
        y = nets.linear(y, p["dnn.linear_%d.weight" % i], p["dnn.linear_%d.bias" % i])
        if i < n_layers - 1:
            y = torch.relu(y)
    return y


def fat_deepffm_parts(p, sparse_inputs, dense_inputs, num_fields):
    """(y_first_order [B,1], y_dnn [B,1]) of FAT_DeepFFMLayer.forward, net.py:48-54."""
    D = p["cen.embedding.weight"].shape[1] // num_fields
    outputs = cen(p, sparse_inputs, dense_inputs, num_fields)
    y1, h = deepffm(outputs, num_fields, D)
    n_layers = len([k for k in p if k.startswith("dnn.linear_") and k.endswith(".weight")])
    return y1, dnn(p, h, n_layers)


def fat_deepffm_forward(p, sparse_inputs, dense_inputs, num_fields):
    """FAT_DeepFFMLayer.forward — net.py:48-57: the bias IS added."""
    y1, y_dnn = fat_deepffm_parts(p, sparse_inputs, dense_inputs, num_fields)
    return torch.sigmoid(y1 + y_dnn + p["bias"])                                  # :56


def tile(x, repeat_times):
    """paddle.tile: repeat x along each axis; a repeat_times shorter than x.ndim is padded with
    leading 1s (so [D] on a [B, C] tensor repeats the last axis D times)."""
    rt = [1] * (x.dim() - len(repeat_times)) + list(repeat_times)
    return x.repeat(*rt)


def split(x, num_or_sections, axis=0):
    """paddle.split: an int splits `axis` into that many equal parts, a list into parts of those
    sizes; returns a list of tensors."""
    if isinstance(num_or_sections, int):
        return list(torch.split(x, x.shape[axis] // num_or_sections, dim=axis))
    return list(torch.split(x, list(num_or_sections), dim=axis))


def flatten(x, start_axis=0, stop_axis=-1, name=None):
    """paddle.flatten: merge axes start_axis..stop_axis into one."""
    return torch.flatten(x, start_axis, stop_axis)


def install_fat_apis():
    """Give the paddle shim (oracle/paddle_shim.py, installed first) the APIs that
    fat_deepffm/net.py needs beyond the other rank models, so the reference's net runs on it
    unmodified."""
    import types

    import torch.nn as tnn

    paddle = sys.modules["paddle"]
    nn = sys.modules["paddle.nn"]

    class AdaptiveMaxPool1D(nn.Layer):
        """paddle.nn.AdaptiveMaxPool1D(output_size=1): [N, C, L] -> [N, C, 1], the maximum over L;
        its gradient goes to the first maximum."""

        def __init__(self, output_size, return_mask=False, name=None):
            super().__init__()
            assert output_size == 1 and not return_mask

        def forward(self, x):
            return adaptive_max_pool1d_to_1(x)

    class Sequential(nn.Layer):
        """paddle.nn.Sequential(*layers): layers given bare or as (name, layer) tuples; a tuple's
        name becomes the sublayer's name (and so its state_dict prefix).  Runs them in order."""

        def __init__(self, *layers):
            super().__init__()
            self._order = []
            for i, item in enumerate(layers):
                name, layer = item if isinstance(item, tuple) else (str(i), item)
                self.add_module(name, layer)
                self._order.append(name)

        def forward(self, x):
            for name in self._order:
                x = self._modules[name](x)
            return x

    layer_mod = sys.modules.get("paddle.nn.layer") or types.ModuleType("paddle.nn.layer")
    sys.modules["paddle.nn.layer"] = layer_mod
    nn.layer = layer_mod
    layer_mod.AdaptiveMaxPool1D = nn.AdaptiveMaxPool1D = AdaptiveMaxPool1D
    nn.Sequential = Sequential
    paddle.flatten = flatten
    paddle.tile = tile
    paddle.split = split
    del tnn
    return paddle
