"""Host-side building blocks with Paddle's layer semantics, backed by the b200rec C ABI.

What each class mirrors (reference = /root/reference):
  Embedding   paddle.nn.Embedding(V, D, padding_idx, sparse=True)    e.g. models/rank/deepfm/net.py:66-86
  Linear      paddle.nn.Linear: y = x @ W + b with W:[in,out]        e.g. models/rank/deepfm/net.py:156-163
  matmul precision: the tower GEMMs are the only tensor-core work on this path (cuBLAS through
  torch); `set_matmul_precision` picks fp32 (exact, SIMT), tf32, or bf16x3 (3 bf16 tensor-core
  GEMMs on a hi/lo split, ~2^-16 relative error — meets the 1e-4 logit bar).
"""
from __future__ import annotations

import math
from typing import List, Optional

import torch
import torch.nn as tnn

from . import ops

_PRECISION = "fp32"


def set_matmul_precision(mode: str) -> None:
    """'fp32' | 'tf32' | 'bf16x3' for every Linear / CrossNet GEMM of this package."""
    global _PRECISION
    if mode not in ("fp32", "tf32", "bf16x3"):
        raise ValueError("matmul precision must be fp32, tf32 or bf16x3")
    _PRECISION = mode


def get_matmul_precision() -> str:
    return _PRECISION


def _split_bf16(a: torch.Tensor):
    hi = a.to(torch.bfloat16)
    lo = (a - hi.to(torch.float32)).to(torch.bfloat16)
    return hi, lo


def mm(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """a @ b for fp32 operands in the configured precision (no autograd: used inside Functions)."""
    if _PRECISION == "fp32":
        prev = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = False
        try:
            return torch.mm(a, b)
        finally:
            torch.backends.cuda.matmul.allow_tf32 = prev
    if _PRECISION == "tf32":
        prev = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = True
        try:
            return torch.mm(a, b)
        finally:
            torch.backends.cuda.matmul.allow_tf32 = prev
    a_hi, a_lo = _split_bf16(a)
    b_hi, b_lo = _split_bf16(b)
    out = torch.mm(a_hi, b_hi, out_dtype=torch.float32)
    out += torch.mm(a_hi, b_lo, out_dtype=torch.float32)
    out += torch.mm(a_lo, b_hi, out_dtype=torch.float32)
    return out


class _LinearFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, W, b):
        ctx.save_for_backward(x, W)
        y = mm(x, W)
        if b is not None:
            y += b
        return y

    @staticmethod
    def backward(ctx, dy):
        x, W = ctx.saved_tensors
        dy = dy.contiguous()
        dx = mm(dy, W.t()) if ctx.needs_input_grad[0] else None
        dW = mm(x.t(), dy) if ctx.needs_input_grad[1] else None
        db = dy.sum(0) if ctx.needs_input_grad[2] else None
        return dx, dW, db


class Linear(tnn.Module):
    """paddle.nn.Linear: weight is [in_features, out_features] (transposed w.r.t. torch)."""

    def __init__(self, in_features: int, out_features: int, weight_std: Optional[float] = None,
                 xavier: bool = False, bias: bool = True, weight_l2_decay: float = 0.0,
                 truncated: bool = False):
        super().__init__()
        self.in_features, self.out_features = in_features, out_features
        self.weight = tnn.Parameter(torch.empty(in_features, out_features))
        if weight_l2_decay:
            # ParamAttr(regularizer=L2Decay(c)): the optimizer adds c*w to this parameter's
            # gradient (after clipping) — optim._Base._apply_regularizers
            self.weight.l2_decay = float(weight_l2_decay)
        self.bias = tnn.Parameter(torch.zeros(out_features)) if bias else None
        if xavier:  # paddle XavierUniform: U(-sqrt(6/(fan_in+fan_out)), +)
            lim = math.sqrt(6.0 / (in_features + out_features))
            tnn.init.uniform_(self.weight, -lim, lim)
        elif weight_std is not None and truncated:  # paddle TruncatedNormal(std): resample beyond 2 sigma
            tnn.init.trunc_normal_(self.weight, 0.0, weight_std, -2.0 * weight_std, 2.0 * weight_std)
        elif weight_std is not None:
            tnn.init.normal_(self.weight, 0.0, weight_std)
        else:  # paddle.nn.Linear default: XavierUniform as well
            lim = math.sqrt(6.0 / (in_features + out_features))
            tnn.init.uniform_(self.weight, -lim, lim)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if _PRECISION == "bf16x3" and x.is_cuda and ops.tc_backend():
            return ops.tc_linear(x, self.weight, self.bias)      # hand-written wgmma GEMMs
        lead = x.shape[:-1]
        y = _LinearFn.apply(x.reshape(-1, self.in_features), self.weight, self.bias)
        return y.reshape(*lead, self.out_features)


class BatchNorm1D(tnn.Module):
    """paddle.nn.BatchNorm1D(num_features, momentum=0.9, epsilon=1e-5) on [B, C] activations: state
    `weight`, `bias`, `_mean`, `_variance` (the reference's checkpoint names).  Train mode
    normalises with the batch mean and the biased batch variance (library kernel:
    torch.nn.functional.batch_norm) and moves the running statistics by (1 - momentum) with the
    BIASED variance, which is Paddle's rule — torch's own running update uses the unbiased one, so
    the buffers are updated here, not by the library call."""

    def __init__(self, num_features: int, momentum: float = 0.9, epsilon: float = 1e-5):
        super().__init__()
        self.weight = tnn.Parameter(torch.ones(num_features))
        self.bias = tnn.Parameter(torch.zeros(num_features))
        self.register_buffer("_mean", torch.zeros(num_features))
        self.register_buffer("_variance", torch.ones(num_features))
        self.momentum, self.epsilon = momentum, epsilon

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if not self.training:
            return torch.nn.functional.batch_norm(x, self._mean, self._variance, self.weight,
                                                  self.bias, False, 0.0, self.epsilon)
        with torch.no_grad():
            var, mu = torch.var_mean(x, dim=0, unbiased=False)
            self._mean.mul_(self.momentum).add_(mu, alpha=1.0 - self.momentum)
            self._variance.mul_(self.momentum).add_(var, alpha=1.0 - self.momentum)
        return torch.nn.functional.batch_norm(x, None, None, self.weight, self.bias, True, 0.0,
                                              self.epsilon)


_HOOKS = {}


def _autograd_hook(device) -> torch.Tensor:
    """A requires_grad scalar per device: keeps autograd walking into a gather whose table has no
    dense grad (its backward returns None for it, so nothing is ever accumulated)."""
    h = _HOOKS.get(device)
    if h is None:
        h = torch.zeros(1, device=device, requires_grad=True)
        _HOOKS[device] = h
    return h


class Embedding(tnn.Module):
    """paddle.nn.Embedding(num_embeddings, embedding_dim, padding_idx, sparse=True).

    The table is a Parameter that never gets a dense `.grad`: backward leaves a merged
    `ops.SelectedRows` in `self.grad_rows`, consumed by paddlerec_b200.optim."""

    def __init__(self, num_embeddings: int, embedding_dim: int, padding_idx: Optional[int] = None,
                 init_std: Optional[float] = None, init: str = "truncated_normal",
                 device=None):
        super().__init__()
        self.num_embeddings, self.embedding_dim = num_embeddings, embedding_dim
        if padding_idx is not None and padding_idx < 0:
            padding_idx = num_embeddings + padding_idx  # paddle wraps negative padding_idx
        self.padding_idx = padding_idx
        w = torch.empty(num_embeddings, embedding_dim, device=device)
        self.weight = tnn.Parameter(w, requires_grad=False)
        # the SelectedRows gradient lives ON the parameter tensor (like Paddle's param.grad), so an
        # optimizer built from `model.parameters()` finds it without knowing about modules
        self.weight.is_sparse_table = True
        self.weight.grad_rows = None
        self.reset_parameters(init, init_std)

    @property
    def grad_rows(self) -> Optional[ops.SelectedRows]:
        return getattr(self.weight, "grad_rows", None)

    @property
    def pad(self) -> int:
        return -1 if self.padding_idx is None else int(self.padding_idx)

    @torch.no_grad()
    def reset_parameters(self, init: str, std: Optional[float]) -> None:
        w = self.weight
        if init == "truncated_normal":  # paddle TruncatedNormal: resample outside +-2 sigma
            tnn.init.trunc_normal_(w, 0.0, std or 1.0, -2.0 * (std or 1.0), 2.0 * (std or 1.0))
        elif init == "uniform":  # paddle Uniform(): U(-1, 1)
            w.uniform_(-1.0, 1.0)
        elif init == "xavier_uniform":
            lim = math.sqrt(6.0 / (self.num_embeddings + self.embedding_dim))
            w.uniform_(-lim, lim)
        elif init == "zeros":
            w.zero_()
        elif init == "empty":
            pass
        else:
            raise ValueError(init)
        if self.padding_idx is not None and init != "empty":
            w[self.padding_idx].zero_()  # paddle dygraph zeroes the padding row at construction

    def accept(self, sr: ops.SelectedRows) -> None:
        if self.grad_rows is not None:      # shared table / micro-batch accumulation: merge-add
            sr = ops.merge_selected_rows(self.grad_rows, sr)
        self.weight.grad_rows = sr

    def forward(self, ids: torch.Tensor) -> torch.Tensor:
        return ops.gather(self.weight, ids, self.pad, self, _autograd_hook(ids.device))

    def forward_pooled(self, keys: torch.Tensor, offsets: torch.Tensor) -> torch.Tensor:
        """Multi-hot slot: sum of the rows of each variable-length key list (LoD offsets)."""
        return ops.gather_pool_sum(self.weight, keys, offsets, self.pad, self,
                                   _autograd_hook(keys.device))

    def forward_seqpool_cvm(self, keys, offsets, n_slots: int, show_click, use_cvm: bool):
        """All multi-hot slots of a batch at once: sum-pool + CVM (ops.fused_seqpool_cvm)."""
        return ops.fused_seqpool_cvm(self.weight, keys, offsets, n_slots, show_click, use_cvm,
                                     self.pad, self, _autograd_hook(keys.device))

    def clear_grad(self) -> None:
        self.weight.grad_rows = None

    def _apply(self, fn, *a, **kw):  # keep the tags if .to()/.cuda() replaces the tensor
        out = super()._apply(fn, *a, **kw)
        self.weight.is_sparse_table = True
        if not hasattr(self.weight, "grad_rows"):
            self.weight.grad_rows = None
        return out


class FusedTable(tnn.Module):
    """Fused layout for a pair of tables that are always looked up with the same ids (DeepFM's
    second-order [V,D] and first-order [V,1], models/rank/deepfm/net.py:66-86): ONE array of
    128-byte slots `[D emb | w1 | pad]`.

    Why: a random 64-byte row costs a full 128-byte DRAM access and so does a random 4-byte
    scalar (tools/microbench/gather_variants.cu measures it), so the reference's two-table layout moves
    256 B per looked-up id for 68 useful bytes; the slot moves 128 B.  Same for the optimizer.

    state_dict() still exposes the reference's two keys (`embedding.weight` [V,D] and
    `embedding_one.weight` [V,1], as views of the slot array) and loads from them, so checkpoints
    stay interchangeable.  The gradient is one SelectedRows of width D+1 (+pad) on `weight`.

    With one name (`names=("embedding.weight",)`) the slot holds a single table [D emb | 0 | pad]
    in the same layout, so the FFM-family kernels read it unchanged: the w1 column starts at zero,
    its gradient column is always zero, and views, state_dict and grad_dense show only the
    embedding."""

    def __init__(self, num_embeddings, embedding_dim, padding_idx=None, init_std=None, device=None,
                 names=("embedding.weight", "embedding_one.weight"), attr="_fused",
                 moments_in_slot=True):
        super().__init__()
        D = embedding_dim
        self.num_embeddings, self.embedding_dim = num_embeddings, D
        self.slot, self.grad_cols = ops.fused_slot(D), ops.fused_grad_cols(D)
        # Optimizer state inside the slot: [w (G cols) | m (G) | v (G) | pad] in 2 x 128 bytes, so a
        # lazy-Adam update touches 2 lines per row instead of 3 (and the three lines it needs share
        # a DRAM page); the forward still reads only the first line.  Falls back to separate
        # moment arrays when 3*G floats do not fit 64.
        self.moment_cols = None
        if moments_in_slot and 3 * self.grad_cols <= 64 and self.slot == 32:
            self.slot = 64
            self.moment_cols = (self.grad_cols, 2 * self.grad_cols)
        self.padding_idx = padding_idx
        self._names, self._attr = names, attr
        w = torch.zeros(num_embeddings, self.slot, device=device)
        std = init_std or 1.0
        if num_embeddings > 0:
            ncols = D + 1 if len(names) == 2 else D
            tnn.init.trunc_normal_(w[:, :ncols], 0.0, std, -2.0 * std, 2.0 * std)
            if padding_idx is not None:
                w[padding_idx].zero_()
        self.weight = tnn.Parameter(w, requires_grad=False)
        self._tag()

    def _tag(self):
        self.weight.is_sparse_table = True
        self.weight.fused_D = self.embedding_dim
        self.weight.fused_names = self._names
        self.weight.inslot_moments = self.moment_cols
        if not hasattr(self.weight, "grad_rows"):
            self.weight.grad_rows = None

    def _apply(self, fn, *a, **kw):
        out = super()._apply(fn, *a, **kw)
        self._tag()
        return out

    @property
    def pad(self) -> int:
        return -1 if self.padding_idx is None else int(self.padding_idx)

    def views(self):
        """One view per name: (embedding [V,D], embedding_one [V,1]) or (embedding,)."""
        w = self.weight.detach()
        D = self.embedding_dim
        return (w[:, :D], w[:, D:D + 1])[:len(self._names)]

    # ---- gradient sink protocol used by ops._EmbedFM -----------------------------------------
    def groups_for(self, ids, V, pad):
        return ops.raw_group_ids(ids, V, pad)

    def accept_fused(self, sr: ops.SelectedRows) -> None:
        sr.ncols = self.grad_cols
        if self.weight.grad_rows is not None:   # second use in one step: merge-add like Paddle
            sr = ops.merge_selected_rows(self.weight.grad_rows, sr)
            sr.ncols = self.grad_cols
        self.weight.grad_rows = sr

    @property
    def grad_rows(self):
        return self.weight.grad_rows

    def grad_dense(self):
        """(dW [V,D], dW1 [V,1]), or (dW,) with one name, as dense tensors (tests / small tables)."""
        D = self.embedding_dim
        if self.weight.grad_rows is None:
            z = torch.zeros(self.num_embeddings, D + 1, device=self.weight.device)
        else:
            z = self.weight.grad_rows.to_dense()
        return (z[:, :D], z[:, D:D + 1])[:len(self._names)]

    # ---- reference-compatible checkpoint keys -------------------------------------------------
    def _parent_prefix(self, prefix: str) -> str:
        return prefix[:-(len(self._attr) + 1)]

    def _save_to_state_dict(self, destination, prefix, keep_vars):
        parent = self._parent_prefix(prefix)
        for name, view in zip(self._names, self.views()):
            destination[parent + name] = view

    def _load_from_state_dict(self, *args, **kwargs):
        pass  # the owning module routes the reference-named keys here (load_views)

    def load_views(self, state_dict, parent_prefix, strict, missing_keys):
        """Copy `<parent>embedding.weight` / `<parent>embedding_one.weight` into the slot array and
        return the state_dict without those keys (torch only hands a child the keys under ITS
        prefix, so the parent module calls this from its own _load_from_state_dict)."""
        rest = dict(state_dict)
        for name, view in zip(self._names, self.views()):
            key = parent_prefix + name
            if key in rest:
                with torch.no_grad():
                    view.copy_(rest.pop(key).reshape(view.shape))
            elif strict:
                missing_keys.append(key)
        return rest


class FusedTableOwner(tnn.Module):
    """Mixin for a module that holds a FusedTable in `self._fused` (may be absent)."""

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys,
                              unexpected_keys, error_msgs):
        fused = self._modules.get("_fused")
        if fused is not None:
            state_dict = fused.load_views(state_dict, prefix, strict, missing_keys)
        super()._load_from_state_dict(state_dict, prefix, local_metadata, strict, missing_keys,
                                      unexpected_keys, error_msgs)


class EmbeddingPair:
    """Grad sink for the fused DeepFM kernel, which reads TWO tables ([V,1] and [V,D]) with the
    same ids: one grouping pass serves both SelectedRows."""

    def __init__(self, emb: Embedding, emb_one: Embedding):
        self.emb, self.emb_one = emb, emb_one

    def groups_for(self, ids, V, pad):
        return ops.raw_group_ids(ids, V, pad)

    def accept(self, sr_w: ops.SelectedRows, sr_w1: ops.SelectedRows) -> None:
        self.emb.accept(sr_w)
        self.emb_one.accept(sr_w1)


def sparse_tables(model: tnn.Module) -> List[Embedding]:
    return [m for m in model.modules() if isinstance(m, Embedding)]
