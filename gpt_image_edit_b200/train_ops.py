"""Tensor-level wrappers over the training entry points of the C ABI (include/b2f.h, "Stage-2 training step").

Same rules as `ops.py`: torch owns storage, libb2f does the arithmetic, nothing here computes in torch and
every function raises if the tensors are not CUDA tensors of the expected dtype.
The reference reaches these ops through `accelerator.backward(loss)` / `optimizer.step()`
(train_denoiser.py:1172-1181).
"""
from __future__ import annotations

import torch

from . import _lib
from ._lib import check, ptr, stream_ptr
from .ops import _as3, _qkv_views, _req, _row_pitch, _rows, _shape, _token_rows

EPI_STORE, EPI_RESID, EPI_DGELU, EPI_DSILU = 0, 4, 8, 9


def _f32(t, name):
    _req(t, name, torch.float32)


def linear_dgrad(dy, weight, *, epilogue: int = EPI_STORE, aux=None, out=None) -> torch.Tensor:
    """dx = epi(dy @ weight) for weight [out_features, in_features] as nn.Linear stores it.
    dy: [M, out] or [B, M, out] view; aux: saved pre-activation (DGELU/DSILU) or the gradient to add to (RESID)."""
    _req(dy, "dy")
    _req(weight, "weight")
    d3 = _as3(dy)
    B, M, K = d3.shape
    if weight.shape[0] != K:
        raise _lib.B2FError(f"linear_dgrad: dy has {K} columns, weight has {weight.shape[0]} rows")
    N = weight.shape[1]
    if out is None:
        out = torch.empty((*dy.shape[:-1], N), device=dy.device, dtype=torch.bfloat16)
    o3 = _rows(out, "out", B, M, N)
    ld_aux = aux_bs = 0
    if epilogue != EPI_STORE:
        a3 = _rows(aux, "aux", B, M, N)
        ld_aux, aux_bs = a3.stride(1), a3.stride(0)
    check(_lib.lib.b2f_gemm_dgrad(ptr(d3), d3.stride(1), d3.stride(0), ptr(weight), weight.stride(0), ptr(o3),
                                  o3.stride(1), o3.stride(0), B, M, N, K, epilogue, ptr(aux), ld_aux, aux_bs, stream_ptr()),
          "b2f_gemm_dgrad")
    return out


def linear_wgrad(dy, x, *, out=None, accumulate: bool = False) -> torch.Tensor:
    """dW[out_features, in_features] (+)= sum over tokens dy^T x, fp32.  dy [B, rows, out], x [B, rows, in] views."""
    _req(dy, "dy")
    _req(x, "x")
    d3, x3 = _as3(dy), _as3(x)
    B, rows, M = d3.shape
    if x3.shape[0] != B or x3.shape[1] != rows:
        raise _lib.B2FError(f"linear_wgrad: token layouts differ: {tuple(d3.shape)} vs {tuple(x3.shape)}")
    N = x3.shape[2]
    if out is None:
        if accumulate:
            raise _lib.B2FError("linear_wgrad: accumulate needs an existing gradient tensor")
        out = torch.empty((M, N), device=dy.device, dtype=torch.float32)
    _f32(out, "out")
    _shape(out, "out", (M, N))
    check(_lib.lib.b2f_gemm_wgrad(ptr(d3), d3.stride(1), d3.stride(0), ptr(x3), x3.stride(1), x3.stride(0), ptr(out),
                                  out.stride(0), B, rows, M, N, int(accumulate), stream_ptr()), "b2f_gemm_wgrad")
    return out


def s_pad(S: int) -> int:
    return (S + 127) // 128 * 128


def attention_fwd_lse(q, k, v, *, out=None, scale: float | None = None):
    """(out [B,S,H*128], lse2 fp32 [B,H,S_pad]) — forward that keeps the base-2 log-sum-exp rows."""
    B, Sq, H, dh = _qkv_views(q, k, v)
    Skv, Hkv = k.shape[1], k.shape[2]
    if out is None:
        out = torch.empty((B, Sq, H * dh), device=q.device, dtype=torch.bfloat16)
    ldo = _token_rows(out, "out", B, Sq, H * dh)
    lse = torch.empty((B, H, s_pad(Sq)), device=q.device, dtype=torch.float32)
    if scale is None:
        scale = dh ** -0.5
    check(_lib.lib.b2f_attention_fwd_lse(ptr(q), _row_pitch(q), ptr(k), _row_pitch(k), ptr(v), _row_pitch(v), ptr(out),
                                         ldo, B, H, Hkv, Sq, Skv, dh, float(scale), 0, ptr(lse), lse.stride(1),
                                         stream_ptr()), "b2f_attention_fwd_lse")
    return out, lse


def attention_bwd(q, k, v, o, dout, lse, *, dq=None, dk=None, dv=None, scale: float | None = None):
    """dq, dk, dv ([B,S,H,128] views or new tensors) of softmax attention; o / dout: [B,S,H*128] views."""
    B, S, H, dh = _qkv_views(q, k, v)
    if k.shape != q.shape:
        raise _lib.B2FError("attention_bwd: the joint FLUX attention only (Sq == Skv, H == Hkv)")
    ldo, lddo = _token_rows(o, "o", B, S, H * dh), _token_rows(dout, "dout", B, S, H * dh)
    _f32(lse, "lse")
    sp = lse.shape[-1]
    if lse.dim() != 3 or tuple(lse.shape[:2]) != (B, H) or sp < S or sp % 128 or not lse.is_contiguous():
        raise _lib.B2FError(f"lse: expected a contiguous [B={B}, H={H}, S_pad] with S_pad >= {S} a multiple of 128, "
                            f"got {tuple(lse.shape)}")
    mk = lambda: torch.empty((B, S, H, dh), device=q.device, dtype=torch.bfloat16)
    dq = mk() if dq is None else dq
    dk = mk() if dk is None else dk
    dv = mk() if dv is None else dv
    if _qkv_views(dq, dk, dv, "d") != q.shape or dk.shape != q.shape:
        raise _lib.B2FError(f"dq, dk, dv: expected q's shape {tuple(q.shape)}, got {tuple(dq.shape)}, {tuple(dk.shape)}")
    delta = torch.empty((B, H, sp), device=q.device, dtype=torch.float32)
    if scale is None:
        scale = dh ** -0.5
    check(_lib.lib.b2f_attn_delta(ptr(o), ldo, ptr(dout), lddo, ptr(delta), ptr(lse), B, H, S, sp,
                                  stream_ptr()), "b2f_attn_delta")
    check(_lib.lib.b2f_attention_bwd(ptr(q), _row_pitch(q), ptr(k), _row_pitch(k), ptr(v), _row_pitch(v), ptr(dout),
                                     lddo, ptr(lse), ptr(delta), sp, ptr(dq), _row_pitch(dq), ptr(dk), _row_pitch(dk),
                                     ptr(dv), _row_pitch(dv), B, H, S, dh, float(scale), stream_ptr()), "b2f_attention_bwd")
    return dq, dk, dv


def gate_resid(x, y, gate, *, gate_b=None, split_row: int = 0, out=None):
    """out = x + gate[b] * y over [B, rows, D]; rows >= split_row use gate_b."""
    for t, n in ((x, "x"), (y, "y"), (gate, "gate")):
        _req(t, n)
    B, rows, D = x.shape
    if out is None:
        out = torch.empty_like(x)
    check(_lib.lib.b2f_gate_resid_fwd(ptr(x), x.stride(1), x.stride(0), ptr(y), y.stride(1), y.stride(0), ptr(gate),
                                      ptr(gate_b), gate.stride(0), ptr(out), out.stride(1), out.stride(0), B, rows, D,
                                      split_row, stream_ptr()), "b2f_gate_resid_fwd")
    return out


def _col_reduce(partial, nchunks, D, B, out, accumulate):
    check(_lib.lib.b2f_col_reduce(ptr(partial), nchunks, D, ptr(out), out.stride(0), B, int(accumulate), stream_ptr()),
          "b2f_col_reduce")


def gate_bwd(dout, *, y=None, gate=None, gate_b=None, split_row: int = 0, part_row0: int = 0, want_dy: bool = True,
             want_sum: bool = True, dy=None, col_out=None, accumulate: bool = False):
    """dy = gate[b] * dout and col[b, :] = sum_{rows >= part_row0} dout * y  (y None: column sum of dout).
    Returns (dy or None, col fp32 [B, D] or None)."""
    _req(dout, "dout")
    B, rows, D = dout.shape
    if want_dy:
        _req(gate, "gate")
        if dy is None:
            dy = torch.empty_like(dout)
    else:
        dy = None
    partial = None
    nch = int(_lib.lib.b2f_train_chunks(rows))
    if want_sum:
        partial = torch.empty((B, nch, D), device=dout.device, dtype=torch.float32)
    check(_lib.lib.b2f_gate_bwd(ptr(dout), dout.stride(1), dout.stride(0), ptr(y), 0 if y is None else y.stride(1),
                                0 if y is None else y.stride(0), ptr(gate) if want_dy else None,
                                ptr(gate_b) if want_dy else None, 0 if gate is None else gate.stride(0), ptr(dy),
                                0 if dy is None else dy.stride(1), 0 if dy is None else dy.stride(0), ptr(partial), B, rows,
                                D, split_row if want_dy else 0, part_row0, stream_ptr()), "b2f_gate_bwd")
    if want_sum:
        if col_out is None:
            col_out = torch.empty((B, D), device=dout.device, dtype=torch.float32)
        _col_reduce(partial, nch, D, B, col_out, accumulate)
    return dy, col_out


def ln_modulate_bwd(x, dy, scale, *, scale_b=None, split_row: int = 0, part_row0: int = 0, dres=None, out=None,
                    want_mod_grads: bool = True, eps: float = 1e-6):
    """(dres_out, dscale fp32 [B,D] | None, dshift | None): backward of ops.ln_modulate joined with the residual
    gradient `dres` (None: start a fresh gradient)."""
    for t, n in ((x, "x"), (dy, "dy"), (scale, "scale")):
        _req(t, n)
    B, rows, D = x.shape
    if out is None:
        out = torch.empty_like(x)
    nch = int(_lib.lib.b2f_train_ln_chunks(rows))
    partial = torch.empty((B, nch, 2 * D), device=x.device, dtype=torch.float32) if want_mod_grads else None
    check(_lib.lib.b2f_ln_modulate_bwd(ptr(x), x.stride(1), x.stride(0), ptr(dy), dy.stride(1), dy.stride(0), ptr(scale),
                                       ptr(scale_b), scale.stride(0), ptr(dres), 0 if dres is None else dres.stride(1),
                                       0 if dres is None else dres.stride(0), ptr(out), out.stride(1), out.stride(0),
                                       ptr(partial), B, rows, D, eps, split_row, part_row0, stream_ptr()),
          "b2f_ln_modulate_bwd")
    if not want_mod_grads:
        return out, None, None
    both = torch.empty((B, 2 * D), device=x.device, dtype=torch.float32)
    _col_reduce(partial, nch, 2 * D, B, both, False)
    return out, both[:, :D], both[:, D:]


def rmsnorm_rope(qkv_pre, H: int, wq, wk, cos, sin, *, wq_added=None, wk_added=None, n_added: int = 0, out=None,
                 eps: float = 1e-6):
    """Out-of-place per-head RMSNorm + RoPE of the Q and K blocks of qkv_pre [B,S,3*H*128]; the V block is copied by
    the caller's GEMM layout (out[:, :, 2d:] is left untouched)."""
    _req(qkv_pre, "qkv_pre")
    B, S, _ = qkv_pre.shape
    d = H * 128
    if out is None:
        out = torch.empty_like(qkv_pre)
    check(_lib.lib.b2f_rmsnorm_rope_out(ptr(qkv_pre), ptr(qkv_pre[:, :, d:]), qkv_pre.stride(1), qkv_pre.stride(0),
                                        ptr(out), ptr(out[:, :, d:]), out.stride(1), out.stride(0), ptr(wq_added),
                                        ptr(wk_added), ptr(wq), ptr(wk), ptr(cos), ptr(sin), B, S, H, n_added, eps,
                                        stream_ptr()), "b2f_rmsnorm_rope_out")
    return out


def rmsnorm_rope_bwd_(dqkv, qkv_pre, H: int, wq, wk, cos, sin, *, wq_added=None, wk_added=None, n_added: int = 0,
                      want_wgrads: bool = True, eps: float = 1e-6):
    """In place on the Q and K blocks of dqkv [B,S,3*H*128]; returns fp32 [4,128] weight gradients
    (norm_added_q, norm_added_k, norm_q, norm_k) or None."""
    _req(dqkv, "dqkv")
    _req(qkv_pre, "qkv_pre")
    B, S, _ = dqkv.shape
    d = H * 128
    nblk = (B * S + 7) // 8
    partial = torch.empty((1, nblk, 512), device=dqkv.device, dtype=torch.float32) if want_wgrads else None
    check(_lib.lib.b2f_rmsnorm_rope_bwd(ptr(dqkv), ptr(dqkv[:, :, d:]), dqkv.stride(1), dqkv.stride(0), ptr(qkv_pre),
                                        ptr(qkv_pre[:, :, d:]), qkv_pre.stride(1), qkv_pre.stride(0), ptr(wq_added),
                                        ptr(wk_added), ptr(wq), ptr(wk), ptr(cos), ptr(sin), ptr(partial), B, S, H, n_added,
                                        eps, stream_ptr()), "b2f_rmsnorm_rope_bwd")
    if not want_wgrads:
        return None
    out = torch.empty((1, 512), device=dqkv.device, dtype=torch.float32)
    _col_reduce(partial, nblk, 512, 1, out, False)
    return out.view(4, 128)


def gelu(x, *, out=None):
    _req(x, "x")
    x2 = x.reshape(-1, x.shape[-1]) if x.is_contiguous() else x
    if x2.dim() != 2:
        raise _lib.B2FError("gelu: expected a [rows, D] view")
    if out is None:
        out = torch.empty(x.shape, device=x.device, dtype=torch.bfloat16)
    o2 = out.reshape(-1, out.shape[-1]) if out.is_contiguous() else out
    check(_lib.lib.b2f_gelu_rows(ptr(x2), x2.stride(0), ptr(o2), o2.stride(0), x2.shape[0], x2.shape[1], stream_ptr()),
          "b2f_gelu_rows")
    return out


def outer_acc(dmod, act, *, out=None, accumulate: bool = False):
    """dW[N, K] (+)= dmod[B, N]^T act[B, K] (fp32)."""
    _f32(dmod, "dmod")
    _req(act, "act")
    B, N = dmod.shape
    K = act.shape[1]
    if out is None:
        out = torch.empty((N, K), device=dmod.device, dtype=torch.float32)
    check(_lib.lib.b2f_outer_acc(ptr(dmod), dmod.stride(0), ptr(act), act.stride(0), ptr(out), out.stride(0), B, N, K,
                                 int(accumulate), stream_ptr()), "b2f_outer_acc")
    return out


def mse_loss(pred, target, *, weight=None, grad_scale: float = 1.0, want_grad: bool = True):
    """(loss fp32 scalar tensor, dpred bf16 | None) of mean(weight * (pred - target)^2)."""
    _req(pred, "pred")
    _f32(target, "target")
    if not pred.is_contiguous() or not target.is_contiguous() or pred.shape != target.shape:
        raise _lib.B2FError("mse_loss: pred / target must be contiguous and of equal shape")
    loss = torch.empty((1,), device=pred.device, dtype=torch.float32)
    ws = torch.empty((1024,), device=pred.device, dtype=torch.float32)
    dpred = torch.empty_like(pred) if want_grad else None
    check(_lib.lib.b2f_mse_loss(ptr(pred), ptr(target), ptr(weight), ptr(dpred), ptr(loss), ptr(ws), pred.numel(),
                                float(grad_scale), stream_ptr()), "b2f_mse_loss")
    return loss, dpred


def grad_sumsq(g, *, out=None, accumulate: bool = False):
    _f32(g, "g")
    if out is None:
        out = torch.zeros((1,), device=g.device, dtype=torch.float32)
    ws = torch.empty((1024,), device=g.device, dtype=torch.float32)
    check(_lib.lib.b2f_grad_sumsq(ptr(g), g.numel(), ptr(out), ptr(ws), int(accumulate), stream_ptr()), "b2f_grad_sumsq")
    return out


def clip_coef(sumsq, max_norm: float, pre_scale: float = 1.0):
    """(coef, norm): coef = min(1, max_norm / (norm + 1e-6)) * pre_scale with norm = pre_scale * sqrt(sumsq)."""
    _f32(sumsq, "sumsq")
    coef = torch.empty((1,), device=sumsq.device, dtype=torch.float32)
    norm = torch.empty((1,), device=sumsq.device, dtype=torch.float32)
    check(_lib.lib.b2f_clip_coef(ptr(sumsq), float(max_norm), float(pre_scale), ptr(coef), ptr(norm), stream_ptr()),
          "b2f_clip_coef")
    return coef, norm


def adamw_step_(p32, m, v, g, *, p16=None, lr: float, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0.01,
                step: int, gscale=None):
    for t, n in ((p32, "p32"), (m, "m"), (v, "v"), (g, "g")):
        _f32(t, n)
        if not t.is_contiguous():
            raise _lib.B2FError(f"adamw_step_: {n} must be contiguous")
    if p16 is not None:
        _req(p16, "p16")
        if not p16.is_contiguous() or p16.numel() != p32.numel():
            raise _lib.B2FError("adamw_step_: p16 must be a contiguous bf16 tensor of the shard's size")
    check(_lib.lib.b2f_adamw_step(ptr(p32), ptr(m), ptr(v), ptr(g), ptr(p16), p32.numel(), float(lr), float(betas[0]),
                                  float(betas[1]), float(eps), float(weight_decay), int(step), ptr(gscale), stream_ptr()),
          "b2f_adamw_step")


def cast(src, dtype):
    """bf16 <-> fp32 copy of a contiguous tensor."""
    if not src.is_cuda or not src.is_contiguous():
        raise _lib.B2FError("cast: contiguous CUDA tensor expected")
    to_f32 = dtype == torch.float32
    _req(src, "src", torch.bfloat16 if to_f32 else torch.float32)
    dst = torch.empty(src.shape, device=src.device, dtype=dtype)
    check(_lib.lib.b2f_cast_bf16_f32(ptr(src), ptr(dst), src.numel(), int(to_f32), stream_ptr()), "b2f_cast_bf16_f32")
    return dst
