"""The dense MLP tower (Linear -> ReLU chain of models/rank/deepfm/net.py:142-174, also
wide_deep/net.py:55-71 and the DIN / DCN-V2 MLPs) as ONE autograd node in 'bf16x3' precision.

Tensor cores are reserved for exactly this part of the path (BASELINE north star).  Each fp32 GEMM
a@b is evaluated as a_hi@b_hi + a_lo@b_hi + a_hi@b_lo with bf16 operands and fp32 accumulation
(cuBLASLt via torch.mm(out_dtype=float32)); everything between two GEMMs — bias, ReLU, the hi/lo
split, the ReLU mask and bias column-sum in backward — is one hand-written streaming kernel per
layer (csrc/tower.cuh).  Activations are kept ONLY in their split bf16 form (what the backward GEMM
consumes), never as fp32.

    forward, layer i :  y = [a_hi|a_lo] @ [W_hi;W_hi]  (+)= a_hi @ W_lo         2 GEMMs
                        a_next = split(relu(y + b))                            1 kernel
    backward, layer i:  dz = split(dy * mask), db = colsum(dz)                 1 kernel
                        dW = fold([a_hi|a_lo]^T @ [dz_hi|dz_lo])               1 GEMM + 1 kernel
                        dx = [dz_hi|dz_lo] @ [W_hi|W_hi]^T (+)= dz_hi @ W_lo^T   2 GEMMs

Two back ends with the same arithmetic (three bf16 products per fp32 product, fp32 accumulation):
  'tcgen05' (default; the name predates the Hopper port)  hand-written wgmma / TMA GEMMs (csrc/tc_gemm.cuh) whose
                       epilogues apply bias + ReLU and emit the NEXT layer's hi/lo operand directly
                       (forward), or the ReLU mask + split + bias column-sum (backward); dW is a
                       batch-split GEMM on MN-major operands.  No elementwise kernel runs between
                       two GEMMs of the tower.
  'cublas'             round-1 path, kept for head-to-head timing (B200REC_TOWER=cublas).
"""
from __future__ import annotations

import os
from typing import List, Optional, Sequence

import torch

from . import ops

F32 = torch.float32
BACKEND = os.environ.get("B200REC_TOWER", "tcgen05")


# The weight-gradient GEMMs do not feed the rest of the backward pass (only the optimizer needs
# them), so they can run on a side stream while the main stream continues with the embedding
# backward, the gradient exchange and the row-wise table update — tensor-core / L2-bound work beside
# HBM- and NVLink-bound work.  Whoever consumes the gradients must call wait_pending() first: the
# optimizers of this package do.  Off by default (ad-hoc code that reads .grad right after
# backward() is then safe without it); runner.train and bench.py switch it on.
OVERLAP_DW = False
_PENDING: List["torch.cuda.Event"] = []
_SIDE = {}


def set_overlap_dw(on: bool) -> None:
    global OVERLAP_DW
    OVERLAP_DW = bool(on)


def wait_pending() -> None:
    """Make the current stream wait for the weight-gradient GEMMs still running on the side stream."""
    if _PENDING:
        cur = torch.cuda.current_stream()
        for ev in _PENDING:
            cur.wait_event(ev)
        _PENDING.clear()


def _side_stream(device) -> "torch.cuda.Stream":
    key = device.index
    if key not in _SIDE:
        _SIDE[key] = torch.cuda.Stream(device=device)
    return _SIDE[key]


def set_backend(name: str) -> None:
    global BACKEND
    if name not in ("tcgen05", "cublas"):
        raise ValueError("tower backend must be wgmma or cublas")
    BACKEND = name


class _TowerTcFn(torch.autograd.Function):
    """The whole Linear/ReLU chain on the wgmma kernels.  Saved for backward: the split
    activations of every layer (they are the dW operands and the ReLU masks) and planes(W)."""

    @staticmethod
    def forward(ctx, x, n_layers, last_act, *params):
        Ws, bs = params[:n_layers], params[n_layers:]
        # Layer i's bias gradient is colsum(g_i).  If its input width is not a multiple of the
        # 128-row dW tile, a column of ones rides in the input planes and the dW GEMM delivers the
        # column sum as an extra output row for free; otherwise the dX epilogue sums columns.
        ones = [b is not None and W.shape[0] % 128 != 0 for W, b in zip(Ws, bs)]
        # A width-1 last layer (the CTR logit) is two streaming kernels, not GEMM tiles
        head = (n_layers >= 2 and Ws[-1].shape[1] == 1 and not last_act and
                Ws[-1].shape[0] % 8 == 0 and Ws[-1].shape[0] <= 2048)
        if head:
            ones[-1] = False
        a = ops.raw_tc_split(x, ones_col=ones[0])
        acts, wps = [a], []
        y = None
        for i in range(n_layers):
            K, N = Ws[i].shape
            last = i == n_layers - 1
            if last and head:
                y = ops.raw_tc_head_fwd(a, K, Ws[i], bs[i])
                wps.append(None)
                break
            Wp, WTp = ops.raw_tc_prep_weight(Ws[i])
            wps.append(Wp)
            relu = (not last) or last_act
            y, a = ops.raw_tc_linear_fwd(a, K, WTp, N, bs[i], relu, want_f32=last,
                                         want_planes=(not last) or last_act,
                                         ones_col=(not last) and ones[i + 1])
            if a is not None:
                acts.append(a)
        ctx.n_layers, ctx.last_act, ctx.ones, ctx.head = n_layers, last_act, ones, head
        ctx.acts, ctx.wps = acts, wps
        ctx.w_last = Ws[-1].detach() if head else None
        ctx.shapes = [tuple(W.shape) for W in Ws]
        ctx.has_bias = [b is not None for b in bs]
        return y

    @staticmethod
    def backward(ctx, dy):
        n, ones = ctx.n_layers, ctx.ones
        acts, wps = ctx.acts, ctx.wps
        dWs, dbs = [None] * n, [None] * n
        top = n - 1
        if ctx.head:
            # g of the layer below, dW and db of the head in one pass over its input activations
            K = ctx.shapes[top][0]
            g, dWs[top], db_head = ops.raw_tc_head_bwd(acts[top], K, ctx.w_last, dy.contiguous())
            dbs[top] = db_head if ctx.has_bias[top] else None
            top -= 1
            db = None
            if ctx.has_bias[top] and not ones[top]:
                # rare (input width of that layer a multiple of 128): column sums of g
                ld = g.shape[1] // 2
                N_top = ctx.shapes[top][1]
                db = (g[:, :N_top].float() + g[:, ld:ld + N_top].float()).sum(0)
        else:
            g, db = ops.raw_tc_split_bwd(dy.contiguous(), acts[n] if ctx.last_act else None)
        dx0 = None
        overlap = OVERLAP_DW and dy.is_cuda
        deferred = []
        for i in range(top, -1, -1):
            K, N = ctx.shapes[i]
            if overlap:
                deferred.append((i, acts[i], K, g, N, db))
            elif ones[i]:
                dWs[i], dbs[i] = ops.raw_tc_linear_bwd_dw(acts[i], K, g, N, bias_row=True)
            else:
                dWs[i] = ops.raw_tc_linear_bwd_dw(acts[i], K, g, N)
                dbs[i] = db if ctx.has_bias[i] else None
            if i > 0:
                # dx of layer i, masked by layer i's input (= ReLU output of layer i-1) and split
                # into the next GEMM's operand, all in the GEMM epilogue
                want_db = ctx.has_bias[i - 1] and not ones[i - 1]
                _, g, db = ops.raw_tc_linear_bwd_dx(g, N, wps[i], K, acts[i], want_f32=False,
                                                    want_planes=True, want_dbias=want_db)
            elif ctx.needs_input_grad[0]:
                dx0, _, _ = ops.raw_tc_linear_bwd_dx(g, N, wps[i], K, None, want_f32=True,
                                                     want_planes=False, want_dbias=False)
        if deferred:
            # the dX chain is enqueued; the dW GEMMs follow on the side stream and overlap whatever
            # the main stream does next (embedding backward, exchange, table update)
            cur = torch.cuda.current_stream()
            side = _side_stream(dy.device)
            side.wait_stream(cur)
            with torch.cuda.stream(side):
                for i, a_i, K, g_i, N, db_i in deferred:
                    if ones[i]:
                        dWs[i], dbs[i] = ops.raw_tc_linear_bwd_dw(a_i, K, g_i, N, bias_row=True,
                                                                  ws_tag="tc_bwd_side")
                    else:
                        dWs[i] = ops.raw_tc_linear_bwd_dw(a_i, K, g_i, N, ws_tag="tc_bwd_side")
                        dbs[i] = db_i if ctx.has_bias[i] else None
                    a_i.record_stream(side)      # allocated on the main stream, read on the side
                    g_i.record_stream(side)
                ev = torch.cuda.Event()
                ev.record(side)
            _PENDING.append(ev)
        ctx.acts = ctx.wps = None
        return (dx0, None, None, *dWs, *dbs)


class _GatedTowerTcFn(torch.autograd.Function):
    """GateNet's tower (gatenet/net.py:112-119) on the wgmma kernels: every hidden layer is
    y = relu(x @ W + b) followed by the hidden gate z = y * tanh(y @ G), the last layer is a plain
    Linear.  The gate GEMM reads planes(y), which the Linear's epilogue emitted, and applies the gate
    in its own epilogue (b200rec_tc_gate_fwd).  Saved for backward: planes of every layer input,
    planes(y), a = y @ G (fp32), planes(W) and planes(G).

    z can be negative, so no layer input here is a ReLU output: the dX GEMM that produces dz runs
    without a mask, and a width-1 last layer takes the generic GEMMs (tc_head_bwd always masks).
    Per hidden layer, from dz:  (g, r) = tc_gate_bwd(dz, y, a);  dG = y^T g;
    du = mask_{y>0}(g @ G^T + r) (with db = colsum(du) in the same epilogue);  dW = x^T du;
    dz_prev = du @ W^T.  The dW GEMMs stay on the current stream."""

    @staticmethod
    def forward(ctx, x, n_layers, *params):
        Ws, bs, Gs = params[:n_layers], params[n_layers:2 * n_layers], params[2 * n_layers:]
        ones = [b is not None and W.shape[0] % 128 != 0 for W, b in zip(Ws, bs)]
        keep = any(ctx.needs_input_grad)
        xs = [ops.raw_tc_split(x, ones_col=ones[0])]
        ys, gate_a, wps, gps = [], [], [], []
        out = None
        for i in range(n_layers):
            K, N = Ws[i].shape
            Wp, WTp = ops.raw_tc_prep_weight(Ws[i], want_w=keep)
            wps.append(Wp)
            if i == n_layers - 1:
                out, _ = ops.raw_tc_linear_fwd(xs[i], K, WTp, N, bs[i], False, want_f32=True,
                                               want_planes=False)
                break
            _, y = ops.raw_tc_linear_fwd(xs[i], K, WTp, N, bs[i], True, want_f32=False,
                                         want_planes=True)
            Gp, GTp = ops.raw_tc_prep_weight(Gs[i], want_w=keep)
            _, z, a = ops.raw_tc_gate_fwd(y, GTp, N, want_a=keep, want_f32=False, want_planes=True,
                                          ones_col=ones[i + 1])
            ys.append(y)
            gate_a.append(a)
            gps.append(Gp)
            xs.append(z)
        ctx.n_layers, ctx.ones = n_layers, ones
        ctx.xs, ctx.ys, ctx.gate_a, ctx.wps, ctx.gps = xs, ys, gate_a, wps, gps
        ctx.shapes = [tuple(W.shape) for W in Ws]
        ctx.has_bias = [b is not None for b in bs]
        return out

    @staticmethod
    def backward(ctx, dy):
        n, ones, shapes = ctx.n_layers, ctx.ones, ctx.shapes
        xs, ys, gate_a, wps, gps = ctx.xs, ctx.ys, ctx.gate_a, ctx.wps, ctx.gps
        dWs, dbs, dGs = [None] * n, [None] * n, [None] * (n - 1)

        def linear_dw(i, g, db_epilogue):
            K, N = shapes[i]
            if ones[i]:
                dWs[i], dbs[i] = ops.raw_tc_linear_bwd_dw(xs[i], K, g, N, bias_row=True)
            else:
                dWs[i] = ops.raw_tc_linear_bwd_dw(xs[i], K, g, N)
                dbs[i] = db_epilogue if ctx.has_bias[i] else None

        top = n - 1
        K, N = shapes[top]
        g, db = ops.raw_tc_split_bwd(dy.contiguous(), None)        # no mask: z is not a ReLU output
        linear_dw(top, g, db)
        dx0 = None
        if top > 0 or ctx.needs_input_grad[0]:
            dx0, _, _ = ops.raw_tc_linear_bwd_dx(g, N, wps[top], K, None, want_f32=True,
                                                 want_planes=False, want_dbias=False)
        for i in range(n - 2, -1, -1):
            K, N = shapes[i]
            dz, dx0 = dx0, None
            ga, r = ops.raw_tc_gate_bwd(dz, ys[i], gate_a[i])
            dGs[i] = ops.raw_tc_linear_bwd_dw(ys[i], N, ga, N)
            want_db = ctx.has_bias[i] and not ones[i]
            _, du, db = ops.raw_tc_linear_bwd_dx(ga, N, gps[i], N, ys[i], want_f32=False,
                                                 want_planes=True, want_dbias=want_db, addend=r)
            linear_dw(i, du, db)
            if i > 0 or ctx.needs_input_grad[0]:
                dx0, _, _ = ops.raw_tc_linear_bwd_dx(du, N, wps[i], K, None, want_f32=True,
                                                     want_planes=False, want_dbias=False)
        ctx.xs = ctx.ys = ctx.gate_a = ctx.wps = ctx.gps = None
        return (dx0 if ctx.needs_input_grad[0] else None, None, *dWs, *dbs, *dGs)


class _TowerFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, n_layers, last_act, *params):
        Ws, bs = params[:n_layers], params[n_layers:]
        a = ops.raw_tower_split(x, None, False)             # [M, 2K0] bf16
        acts, preps = [a], []
        y = None
        for i in range(n_layers):
            W = Ws[i]
            K, N = W.shape
            W2r, W2c, Wlo = ops.raw_tower_prep_weight(W)
            preps.append((W2c, Wlo))
            y = torch.mm(a, W2r, out_dtype=F32)
            torch.addmm(y, a[:, :K], Wlo, out_dtype=F32, out=y)
            relu = (i < n_layers - 1) or last_act
            if i < n_layers - 1:
                a = ops.raw_tower_split(y, bs[i], relu)
                acts.append(a)
            else:
                if relu:
                    a = ops.raw_tower_split(y, bs[i], True)   # keep the mask source
                    acts.append(a)
                    y = torch.relu_(y.add_(bs[i])) if bs[i] is not None else torch.relu_(y)
                elif bs[i] is not None:
                    y = y.add_(bs[i])
        ctx.n_layers, ctx.last_act = n_layers, last_act
        ctx.acts, ctx.preps = acts, preps
        ctx.shapes = [tuple(W.shape) for W in Ws]
        ctx.has_bias = [b is not None for b in bs]
        return y

    @staticmethod
    def backward(ctx, dy):
        n = ctx.n_layers
        acts, preps = ctx.acts, ctx.preps
        dy = dy.contiguous()
        dWs, dbs = [None] * n, [None] * n
        for i in range(n - 1, -1, -1):
            K, N = ctx.shapes[i]
            masked = (i < n - 1) or ctx.last_act
            mask_src = acts[i + 1] if masked else None
            dz, db = ops.raw_tower_relu_bwd_split(dy, mask_src)      # [M, 2N] bf16
            a = acts[i]                                              # [M, 2K] bf16
            Mx = torch.mm(a.t(), dz, out_dtype=F32)                  # [2K, 2N]
            dWs[i] = ops.raw_tower_fold_dw(Mx, K, N)
            dbs[i] = db if ctx.has_bias[i] else None
            if i > 0 or ctx.needs_input_grad[0]:
                W2c, Wlo = preps[i]
                dx = torch.mm(dz, W2c.t(), out_dtype=F32)            # [M, K]
                torch.addmm(dx, dz[:, :N], Wlo.t(), out_dtype=F32, out=dx)
                dy = dx
        dx0 = dy if ctx.needs_input_grad[0] else None
        ctx.acts = ctx.preps = None
        return (dx0, None, None, *dWs, *dbs)


def mlp(x: torch.Tensor, weights: Sequence[torch.Tensor], biases: Sequence[torch.Tensor],
        last_act: bool = False, gates: Optional[Sequence[torch.Tensor]] = None) -> torch.Tensor:
    """relu(...relu(x@W0+b0)...)@W_last+b_last  (ReLU after the last layer iff last_act).

    With `gates` (one [N_i, N_i] matrix per hidden layer) every hidden layer is followed by
    GateNet's hidden gate y * tanh(y @ G_i) (gatenet/net.py:112-119); the last layer has no
    activation.  Only the wgmma back end implements it."""
    lead = x.shape[:-1]
    if gates is not None:
        if BACKEND != "tcgen05":
            raise ValueError("the gated tower runs on the wgmma back end only")
        if last_act or len(gates) != len(weights) - 1:
            raise ValueError("gated tower: one gate per hidden layer and no last activation")
        y = _GatedTowerTcFn.apply(x.reshape(-1, x.shape[-1]).contiguous(), len(weights), *weights,
                                  *biases, *gates)
        return y.reshape(*lead, y.shape[-1])
    fn = _TowerTcFn if BACKEND == "tcgen05" else _TowerFn
    y = fn.apply(x.reshape(-1, x.shape[-1]).contiguous(), len(weights), last_act, *weights, *biases)
    return y.reshape(*lead, y.shape[-1])
