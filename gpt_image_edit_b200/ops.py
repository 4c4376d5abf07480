"""Tensor-level wrappers over the C ABI (torch owns storage; libb2f does the work).

Each function validates dtype/device/contiguity on the host, then passes raw device pointers and
the current CUDA stream to libb2f.  No function here computes anything in torch.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from ._lib import check, ptr, stream_ptr

EPI_BIAS, EPI_GELU_TANH, EPI_SILU, EPI_GATE_RESID, EPI_RESID, EPI_GELU_ERF = 0, 1, 2, 3, 4, 5
EPI_QUICK_GELU = 7


def _req(t: torch.Tensor, name: str, dtype=torch.bfloat16) -> None:
    if not isinstance(t, torch.Tensor):
        raise _lib.B2FError(f"{name}: expected a tensor, got {type(t)}")
    if not t.is_cuda:
        raise _lib.B2FError(f"{name}: libb2f runs on CUDA tensors only (got {t.device}); there is no CPU path")
    if t.dtype != dtype:
        raise _lib.B2FError(f"{name}: expected {dtype}, got {t.dtype}")
    if t.stride(-1) != 1:
        raise _lib.B2FError(f"{name}: innermost dimension must be contiguous")


def _as3(t: torch.Tensor) -> torch.Tensor:
    return t if t.dim() == 3 else t.unsqueeze(0)


def linear(x, weight, bias=None, *, epilogue: int = EPI_BIAS, out=None, resid=None, gate=None) -> torch.Tensor:
    """out = epilogue(x @ weight^T + bias) via b2f_gemm_bf16 (wgmma).

    x: [M,K] or [B,M,K] (any batch/row pitch); weight [N,K]; gate [B,N] for EPI_GATE_RESID."""
    _req(x, "x")
    _req(weight, "weight")
    x3 = _as3(x)
    B, M, K = x3.shape
    N = weight.shape[0]
    if out is None:
        out = torch.empty((*x.shape[:-1], N), device=x.device, dtype=torch.bfloat16)
    _req(out, "out")
    o3 = _as3(out)
    ldr = rbs = gld = 0
    if epilogue in (EPI_GATE_RESID, EPI_RESID):
        _req(resid, "resid")
        r3 = _as3(resid)
        ldr, rbs = r3.stride(1), r3.stride(0)
        if epilogue == EPI_GATE_RESID:
            _req(gate, "gate")
            gld = gate.stride(0) if gate.dim() == 2 else 0
    check(
        _lib.lib.b2f_gemm_bf16(
            ptr(x3), x3.stride(1), x3.stride(0), ptr(weight), weight.stride(0), ptr(bias),
            ptr(o3), o3.stride(1), o3.stride(0), B, M, N, K, epilogue,
            ptr(resid), ldr, rbs, ptr(gate), gld, stream_ptr(),
        ),
        "b2f_gemm_bf16",
    )
    return out


def attention(q, k, v, *, out=None, causal: bool = False, scale: float | None = None, bias=None) -> torch.Tensor:
    """softmax(q k^T * scale [+ bias]) v via b2f_attention_fwd / b2f_attention_bias_fwd.  q [B,Sq,H,128],
    k/v [B,Skv,Hkv,128] as (possibly strided) views whose last two dims are contiguous; out [B,Sq,H*128];
    bias [H,Sq,Skv] bf16 (shared by the batch; T5 relative position bias)."""
    for t, n in ((q, "q"), (k, "k"), (v, "v")):
        _req(t, n)
        if t.dim() != 4 or t.stride(2) != t.shape[3] or (t.shape[0] > 1 and t.stride(0) != t.shape[1] * _row_pitch(t)):
            raise _lib.B2FError(f"{n}: expected a [B,S,H,dh] view with contiguous heads and batch stride S*ld")
    B, Sq, H, dh = q.shape
    Skv, Hkv = k.shape[1], k.shape[2]
    if out is None:
        out = torch.empty((B, Sq, H * dh), device=q.device, dtype=torch.bfloat16)
    _req(out, "out")
    if scale is None:
        scale = dh ** -0.5
    if bias is not None:
        _req(bias, "bias")
        if bias.shape != (H, Sq, Skv) or bias.stride(2) != 1:
            raise _lib.B2FError(f"bias: expected [H={H},Sq={Sq},Skv={Skv}] with unit inner stride, got {tuple(bias.shape)}")
        check(
            _lib.lib.b2f_attention_bias_fwd(
                ptr(q), _row_pitch(q), ptr(k), _row_pitch(k), ptr(v), _row_pitch(v), ptr(out), _row_pitch(out),
                B, H, Hkv, Sq, Skv, dh, float(scale), int(causal), ptr(bias), bias.stride(0), bias.stride(1), stream_ptr(),
            ),
            "b2f_attention_bias_fwd",
        )
        return out
    check(
        _lib.lib.b2f_attention_fwd(
            ptr(q), _row_pitch(q), ptr(k), _row_pitch(k), ptr(v), _row_pitch(v), ptr(out), _row_pitch(out),
            B, H, Hkv, Sq, Skv, dh, float(scale), int(causal), stream_ptr(),
        ),
        "b2f_attention_fwd",
    )
    return out


def ln_modulate(x, scale, shift, *, out=None, eps: float = 1e-6, split_row: int = 0, scale_b=None, shift_b=None) -> torch.Tensor:
    """LayerNorm(x)*(1+scale[b])+shift[b]; x [B,rows,D] view, scale/shift [B,D] views.  With split_row,
    rows >= split_row use (scale_b, shift_b) instead (same pitch)."""
    _req(x, "x")
    _req(scale, "scale")
    _req(shift, "shift")
    x3 = _as3(x)
    B, rows, D = x3.shape
    if out is None:
        out = torch.empty(x.shape, device=x.device, dtype=torch.bfloat16)
    o3 = _as3(out)
    if scale.dim() != 2 or shift.stride(0) != scale.stride(0):
        raise _lib.B2FError("scale/shift must be [B,D] views with equal pitch")
    check(
        _lib.lib.b2f_ln_modulate(ptr(x3), x3.stride(1), x3.stride(0), ptr(scale), ptr(shift), scale.stride(0),
                                 ptr(o3), o3.stride(1), o3.stride(0), B, rows, D, eps, split_row, ptr(scale_b),
                                 ptr(shift_b), stream_ptr()),
        "b2f_ln_modulate",
    )
    return out


def rmsnorm_rope_(qkv, H: int, wq, wk, cos, sin, *, wq_added=None, wk_added=None, n_added: int = 0, eps: float = 1e-6):
    """In place on qkv [B,S,>=2*H*128] (Q block then K block): per-head RMSNorm + RoPE."""
    _req(qkv, "qkv")
    _req(cos, "cos", torch.float32)
    _req(sin, "sin", torch.float32)
    B, S, _ = qkv.shape
    k = qkv[:, :, H * 128:]
    check(
        _lib.lib.b2f_rmsnorm_rope(ptr(qkv), ptr(k), qkv.stride(1), qkv.stride(0), ptr(wq_added), ptr(wk_added),
                                  ptr(wq), ptr(wk), ptr(cos), ptr(sin), B, S, H, 128, n_added, eps, stream_ptr()),
        "b2f_rmsnorm_rope",
    )
    return qkv


def euler_step_(x, v, dt: float):
    """x <- bf16(float(x) + bf16(bf16(dt)*v)) in place; x, v [..., rows, cols] row views of equal shape."""
    _req(x, "x")
    _req(v, "v")
    if x.shape != v.shape:
        raise _lib.B2FError(f"euler_step_: shape mismatch {tuple(x.shape)} vs {tuple(v.shape)}")
    if x.dim() == 3:
        collapsible = all(t.stride(0) == t.shape[1] * t.stride(1) for t in (x, v))
        if not collapsible:
            for b in range(x.shape[0]):
                euler_step_(x[b], v[b], dt)
            return x
        rows, ldx, ldv = x.shape[0] * x.shape[1], x.stride(1), v.stride(1)
    else:
        rows, ldx, ldv = x.shape[0], x.stride(0), v.stride(0)
    check(_lib.lib.b2f_euler_step(ptr(x), ldx, ptr(v), ldv, rows, x.shape[-1], float(dt), stream_ptr()), "b2f_euler_step")
    return x


def rope_tables(ids: torch.Tensor, axes_dim=(16, 56, 56), theta: float = 10000.0):
    """FluxPosEmbed: ids fp32 [S,3] -> (cos, sin) fp32 [S,128]."""
    _req(ids, "ids", torch.float32)
    ids = ids.contiguous()
    S = ids.shape[0]
    cos = torch.empty((S, 128), device=ids.device, dtype=torch.float32)
    sin = torch.empty_like(cos)
    axes = (C.c_int * 3)(*axes_dim)
    check(_lib.lib.b2f_rope_tables(ptr(ids), S, axes, float(theta), ptr(cos), ptr(sin), stream_ptr()), "b2f_rope_tables")
    return cos, sin


def rmsnorm(x, weight, *, out=None, eps: float = 1e-6) -> torch.Tensor:
    """Qwen2RMSNorm over the last dim of x [..., D] (rows must be uniformly pitched)."""
    _req(x, "x")
    _req(weight, "weight")
    x2 = x.reshape(-1, x.shape[-1])
    if out is None:
        out = torch.empty(x.shape, device=x.device, dtype=torch.bfloat16)
    o2 = out.reshape(-1, out.shape[-1])
    check(_lib.lib.b2f_rmsnorm(ptr(x2), x2.stride(0), ptr(weight), ptr(o2), o2.stride(0), x2.shape[0], x2.shape[1], eps,
                               stream_ptr()), "b2f_rmsnorm")
    return out


def rope_half_(x, heads: int, head_pitch: int, cos, sin, *, fp32_math: bool):
    """In-place rotate-half RoPE on x [tokens, >= heads*head_pitch] (row view)."""
    _req(x, "x")
    _req(cos, "cos", torch.float32)
    _req(sin, "sin", torch.float32)
    check(_lib.lib.b2f_rope_half(ptr(x), x.stride(0), heads, head_pitch, ptr(cos), ptr(sin), cos.shape[-1], x.shape[0],
                                 int(fp32_math), stream_ptr()), "b2f_rope_half")
    return x


def swiglu(gu, inter: int, *, out=None) -> torch.Tensor:
    _req(gu, "gu")
    rows = gu.shape[0]
    if out is None:
        out = torch.empty((rows, inter), device=gu.device, dtype=torch.bfloat16)
    check(_lib.lib.b2f_swiglu(ptr(gu), gu.stride(0), ptr(out), out.stride(0), rows, inter, stream_ptr()), "b2f_swiglu")
    return out


def geglu(gu, inter: int, *, out=None) -> torch.Tensor:
    """T5 gated-GELU combine: bf16(bf16(gelu_tanh(gu[:, :inter])) * gu[:, inter:])."""
    _req(gu, "gu")
    rows = gu.shape[0]
    if out is None:
        out = torch.empty((rows, inter), device=gu.device, dtype=torch.bfloat16)
    check(_lib.lib.b2f_geglu(ptr(gu), gu.stride(0), ptr(out), out.stride(0), rows, inter, stream_ptr()), "b2f_geglu")
    return out


def layernorm(x, weight, bias, *, out=None, eps: float = 1e-5) -> torch.Tensor:
    """nn.LayerNorm (affine) over the last dim of x [..., D]."""
    _req(x, "x")
    _req(weight, "weight")
    _req(bias, "bias")
    x2 = x.reshape(-1, x.shape[-1])
    if out is None:
        out = torch.empty(x.shape, device=x.device, dtype=torch.bfloat16)
    o2 = out.reshape(-1, out.shape[-1])
    check(_lib.lib.b2f_layernorm(ptr(x2), x2.stride(0), ptr(weight), ptr(bias), ptr(o2), o2.stride(0), x2.shape[0], x2.shape[1],
                                 eps, stream_ptr()), "b2f_layernorm")
    return out


def embed(table, ids, pos=None, *, period: int = 0, out=None) -> torch.Tensor:
    """out[i] = table[ids[i]] (+ pos[i % period])."""
    _req(table, "table")
    _req(ids, "ids", torch.int64)
    n, D = ids.numel(), table.shape[1]
    if out is None:
        out = torch.empty((n, D), device=table.device, dtype=torch.bfloat16)
    if pos is not None:
        _req(pos, "pos")
    check(_lib.lib.b2f_embed(ptr(table), table.stride(0), ptr(ids), ptr(pos) if pos is not None else None,
                             pos.stride(0) if pos is not None else 0, period, ptr(out), out.stride(0), n, D, stream_ptr()),
          "b2f_embed")
    return out


def gather_rows(table, idx, *, out=None) -> torch.Tensor:
    _req(table, "table")
    _req(idx, "idx", torch.int64)
    n, D = idx.numel(), table.shape[1]
    if out is None:
        out = torch.empty((n, D), device=table.device, dtype=torch.bfloat16)
    check(_lib.lib.b2f_move_rows(ptr(table), table.stride(0), ptr(out), out.stride(0), ptr(idx), n, D, 0, stream_ptr()),
          "b2f_move_rows(gather)")
    return out


def scatter_rows_(dst, idx, src):
    _req(dst, "dst")
    _req(src, "src")
    _req(idx, "idx", torch.int64)
    check(_lib.lib.b2f_move_rows(ptr(src), src.stride(0), ptr(dst), dst.stride(0), ptr(idx), idx.numel(), dst.shape[1], 1,
                                 stream_ptr()), "b2f_move_rows(scatter)")
    return dst


def linear_qkv_norm_rope(x, weight, bias, wq, wk, cos, sin, *, rope_row0: int = 0, out=None, eps: float = 1e-6,
                         out_extra=None, epi_extra: int = EPI_BIAS):
    """[Q|K|V] = x @ weight^T + bias with per-head RMSNorm + RoPE on Q, K fused in the GEMM epilogue.
    With `out_extra` [.., n_extra]: weight has 3d + n_extra rows, the extra columns go there via epi_extra."""
    _req(x, "x")
    _req(weight, "weight")
    _req(cos, "cos", torch.float32)
    _req(sin, "sin", torch.float32)
    x3 = _as3(x)
    B, M, K = x3.shape
    n_extra = 0 if out_extra is None else out_extra.shape[-1]
    N = weight.shape[0] - n_extra
    if out is None:
        out = torch.empty((*x.shape[:-1], N), device=x.device, dtype=torch.bfloat16)
    o3 = _as3(out)
    e3 = None if out_extra is None else _as3(out_extra)
    check(_lib.lib.b2f_gemm_qkv_norm_rope(ptr(x3), x3.stride(1), x3.stride(0), ptr(weight), weight.stride(0), ptr(bias),
                                          ptr(o3), o3.stride(1), o3.stride(0), B, M, N // 3, K, ptr(wq), ptr(wk),
                                          ptr(cos), ptr(sin), rope_row0, eps, n_extra, ptr(e3),
                                          0 if e3 is None else e3.stride(1), 0 if e3 is None else e3.stride(0),
                                          epi_extra, stream_ptr()), "b2f_gemm_qkv_norm_rope")
    return out


def blend(a, b, wa: float, wb: float, *, out=None) -> torch.Tensor:
    """out = a * wa + b * wb in torch's bf16 evaluation order (each product and the sum rounded to bf16)."""
    _req(a, "a")
    _req(b, "b")
    if a.shape != b.shape or not a.is_contiguous() or not b.is_contiguous():
        raise _lib.B2FError("blend: contiguous tensors of equal shape expected")
    if out is None:
        out = torch.empty_like(a)
    check(_lib.lib.b2f_blend_bf16(ptr(a), ptr(b), float(wa), float(wb), ptr(out), a.numel(), stream_ptr()), "b2f_blend_bf16")
    return out


# ------------------------------------------------------------------------------------------------ LoRA
def lora_down(x, acat, colscale, *, cs_mul: float = 1.0, out=None) -> torch.Tensor:
    """T = bf16(fp32(x @ acat^T) * fp32(colscale * cs_mul)) via b2f_gemm_colscale.  x [.., K], acat [r_pad, K],
    colscale fp32 [r_pad]."""
    _req(x, "x")
    _req(acat, "acat")
    _req(colscale, "colscale", torch.float32)
    x3 = _as3(x)
    B, M, K = x3.shape
    N = acat.shape[0]
    if out is None:
        out = torch.empty((*x.shape[:-1], N), device=x.device, dtype=torch.bfloat16)
    o3 = _as3(out)
    check(_lib.lib.b2f_gemm_colscale(ptr(x3), x3.stride(1), x3.stride(0), ptr(acat), acat.stride(0), ptr(o3),
                                     o3.stride(1), o3.stride(0), B, M, N, K, ptr(colscale), float(cs_mul), stream_ptr()),
          "b2f_gemm_colscale")
    return out


def linear_lora(x, weight, bias, t, bcat, *, epilogue: int = EPI_BIAS, out=None, resid=None, gate=None) -> torch.Tensor:
    """out = epilogue(x @ weight^T + t @ bcat^T + bias) via b2f_gemm_bf16_lora (one fp32 accumulation).
    t [.., r_pad] (rows as x), bcat [N, r_pad]."""
    _req(x, "x")
    _req(weight, "weight")
    _req(t, "t")
    _req(bcat, "bcat")
    x3, t3 = _as3(x), _as3(t)
    B, M, K = x3.shape
    N = weight.shape[0]
    if out is None:
        out = torch.empty((*x.shape[:-1], N), device=x.device, dtype=torch.bfloat16)
    o3 = _as3(out)
    ldr = rbs = gld = 0
    if epilogue in (EPI_GATE_RESID, EPI_RESID):
        r3 = _as3(resid)
        ldr, rbs = r3.stride(1), r3.stride(0)
        if epilogue == EPI_GATE_RESID:
            gld = gate.stride(0) if gate.dim() == 2 else 0
    check(_lib.lib.b2f_gemm_bf16_lora(ptr(x3), x3.stride(1), x3.stride(0), ptr(weight), weight.stride(0), ptr(bias),
                                      ptr(o3), o3.stride(1), o3.stride(0), B, M, N, K, epilogue, ptr(resid), ldr, rbs,
                                      ptr(gate), gld, ptr(t3), t3.stride(1), t3.stride(0), ptr(bcat), bcat.stride(0),
                                      bcat.shape[1], stream_ptr()), "b2f_gemm_bf16_lora")
    return out


def linear_qkv_norm_rope_lora(x, weight, bias, wq, wk, cos, sin, t, bcat, *, rope_row0: int = 0, out=None,
                              eps: float = 1e-6, out_extra=None, epi_extra: int = EPI_BIAS):
    """linear_qkv_norm_rope with the LoRA K-extension (t, bcat) of linear_lora."""
    _req(x, "x")
    _req(t, "t")
    _req(bcat, "bcat")
    x3, t3 = _as3(x), _as3(t)
    B, M, K = x3.shape
    n_extra = 0 if out_extra is None else out_extra.shape[-1]
    N = weight.shape[0] - n_extra
    if out is None:
        out = torch.empty((*x.shape[:-1], N), device=x.device, dtype=torch.bfloat16)
    o3 = _as3(out)
    e3 = None if out_extra is None else _as3(out_extra)
    check(_lib.lib.b2f_gemm_qkv_norm_rope_lora(
        ptr(x3), x3.stride(1), x3.stride(0), ptr(weight), weight.stride(0), ptr(bias), ptr(o3), o3.stride(1),
        o3.stride(0), B, M, N // 3, K, ptr(wq), ptr(wk), ptr(cos), ptr(sin), rope_row0, eps, n_extra, ptr(e3),
        0 if e3 is None else e3.stride(1), 0 if e3 is None else e3.stride(0), epi_extra, ptr(t3), t3.stride(1),
        t3.stride(0), ptr(bcat), bcat.stride(0), bcat.shape[1], stream_ptr()), "b2f_gemm_qkv_norm_rope_lora")
    return out


def lora_fuse_(weight, bcat, acat, colscale, *, cs_mul: float = 1.0) -> torch.Tensor:
    """In place: weight <- bf16(weight + sum_k fp32(bcat[:, k] * colscale[k] * cs_mul) acat[k]) (b2f_lora_fuse)."""
    for t, n in ((weight, "weight"), (bcat, "bcat"), (acat, "acat")):
        _req(t, n)
    _req(colscale, "colscale", torch.float32)
    check(_lib.lib.b2f_lora_fuse(ptr(weight), weight.stride(0), weight.shape[0], weight.shape[1], ptr(bcat),
                                 bcat.stride(0), ptr(acat), acat.stride(0), ptr(colscale), float(cs_mul), acat.shape[0],
                                 stream_ptr()), "b2f_lora_fuse")
    return weight


# ---------------------------------------------------------------------------------------------------- FP8 (e4m3)
FP8 = torch.float8_e4m3fn


def _shape(t: torch.Tensor, name: str, want) -> None:
    if tuple(t.shape) != tuple(want):
        raise _lib.B2FError(f"{name}: expected shape {tuple(want)}, got {tuple(t.shape)}")


def _scales(s: torch.Tensor, name: str, B: int, rows: int) -> torch.Tensor:
    """a per-row fp32 scale vector as [B, rows] (any batch pitch, unit row pitch); [rows] when B == 1."""
    _req(s, name, torch.float32)
    s2 = s if s.dim() == 2 else s.unsqueeze(0)
    _shape(s2, name, (B, rows))
    return s2


def quant_fp8_rows(x, *, out=None, scale=None):
    """(q, scale): the FP8 row rule of include/b2f.h (b2f_quant_fp8_rows) on every row of x [rows, K] or [B, rows, K]
    (any pitches): q e4m3 like x, scale fp32 [rows] / [B, rows]."""
    _req(x, "x")
    x3 = _as3(x)
    B, rows, K = x3.shape
    if out is None:
        out = torch.empty(x.shape, device=x.device, dtype=FP8)
    if scale is None:
        scale = torch.empty(x.shape[:-1], device=x.device, dtype=torch.float32)
    _req(out, "out", FP8)
    q3, s2 = _as3(out), _scales(scale, "scale", B, rows)
    _shape(q3, "out", (B, rows, K))
    check(_lib.lib.b2f_quant_fp8_rows(ptr(x3), x3.stride(1), x3.stride(0), ptr(q3), q3.stride(1), q3.stride(0), ptr(s2),
                                      s2.stride(0), B, rows, K, stream_ptr()), "b2f_quant_fp8_rows")
    return out, scale


def ln_modulate_fp8(x, scale, shift, *, out=None, row_scale=None, eps: float = 1e-6, split_row: int = 0, scale_b=None,
                    shift_b=None):
    """(q, row_scale): ln_modulate's bf16 result quantized by the FP8 row rule (b2f_ln_modulate_fp8)."""
    _req(x, "x")
    _req(scale, "scale")
    _req(shift, "shift")
    x3 = _as3(x)
    B, rows, D = x3.shape
    if out is None:
        out = torch.empty(x.shape, device=x.device, dtype=FP8)
    if row_scale is None:
        row_scale = torch.empty(x.shape[:-1], device=x.device, dtype=torch.float32)
    _req(out, "out", FP8)
    o3, s2 = _as3(out), _scales(row_scale, "row_scale", B, rows)
    _shape(o3, "out", (B, rows, D))
    if scale.dim() != 2 or shift.stride(0) != scale.stride(0):
        raise _lib.B2FError("scale/shift must be [B,D] views with equal pitch")
    for t, n in ((scale, "scale"), (shift, "shift"), (scale_b, "scale_b"), (shift_b, "shift_b")):
        if t is not None:
            _shape(t, n, (B, D))
    check(_lib.lib.b2f_ln_modulate_fp8(ptr(x3), x3.stride(1), x3.stride(0), ptr(scale), ptr(shift), scale.stride(0),
                                       ptr(o3), o3.stride(1), o3.stride(0), ptr(s2), s2.stride(0), B, rows, D, eps,
                                       split_row, ptr(scale_b), ptr(shift_b), stream_ptr()), "b2f_ln_modulate_fp8")
    return out, row_scale


def _fp8_weight_checks(wq, w_scale, bias, N, K):
    _shape(wq, "wq", (N, K))
    _shape(w_scale, "w_scale", (N,))
    if bias is not None:
        _req(bias, "bias")
        _shape(bias, "bias", (N,))


def linear_fp8(xq, x_scale, wq, w_scale, bias=None, *, epilogue: int = EPI_BIAS, out=None, resid=None,
               gate=None) -> torch.Tensor:
    """out = epilogue(fp32(x_scale[m] * w_scale[n]) * (xq @ wq^T) + bias) via b2f_gemm_fp8.  xq e4m3 [M,K] / [B,M,K],
    x_scale fp32 [M] / [B,M], wq e4m3 [N,K], w_scale fp32 [N]."""
    _req(xq, "xq", FP8)
    _req(wq, "wq", FP8)
    _req(w_scale, "w_scale", torch.float32)
    x3 = _as3(xq)
    B, M, K = x3.shape
    s2 = _scales(x_scale, "x_scale", B, M)
    N = wq.shape[0]
    _fp8_weight_checks(wq, w_scale, bias, N, K)
    if out is None:
        out = torch.empty((*xq.shape[:-1], N), device=xq.device, dtype=torch.bfloat16)
    _req(out, "out")
    o3 = _as3(out)
    _shape(o3, "out", (B, M, N))
    ldr = rbs = gld = 0
    if epilogue in (EPI_GATE_RESID, EPI_RESID):
        _req(resid, "resid")
        r3 = _as3(resid)
        _shape(r3, "resid", (B, M, N))
        ldr, rbs = r3.stride(1), r3.stride(0)
        if epilogue == EPI_GATE_RESID:
            _req(gate, "gate")
            _shape(gate, "gate", (B, N) if gate.dim() == 2 else (N,))
            gld = gate.stride(0) if gate.dim() == 2 else 0
    check(_lib.lib.b2f_gemm_fp8(ptr(x3), x3.stride(1), x3.stride(0), ptr(s2), s2.stride(0), ptr(wq), wq.stride(0),
                                ptr(w_scale), ptr(bias), ptr(o3), o3.stride(1), o3.stride(0), B, M, N, K, epilogue,
                                ptr(resid), ldr, rbs, ptr(gate), gld, stream_ptr()), "b2f_gemm_fp8")
    return out


def linear_qkv_norm_rope_fp8(xq, x_scale, wq, w_scale, bias, nq, nk, cos, sin, *, rope_row0: int = 0, out=None,
                             eps: float = 1e-6, out_extra=None, epi_extra: int = EPI_BIAS):
    """linear_qkv_norm_rope with the FP8 operands of linear_fp8 (b2f_gemm_qkv_norm_rope_fp8)."""
    _req(xq, "xq", FP8)
    _req(wq, "wq", FP8)
    _req(w_scale, "w_scale", torch.float32)
    _req(cos, "cos", torch.float32)
    _req(sin, "sin", torch.float32)
    x3 = _as3(xq)
    B, M, K = x3.shape
    s2 = _scales(x_scale, "x_scale", B, M)
    n_extra = 0 if out_extra is None else out_extra.shape[-1]
    N = wq.shape[0] - n_extra
    _fp8_weight_checks(wq, w_scale, bias, N + n_extra, K)
    _shape(nq, "nq", (128,))
    _shape(nk, "nk", (128,))
    if cos.dim() != 2 or cos.shape[0] < rope_row0 + M or cos.shape[1] != 128 or cos.shape != sin.shape:
        raise _lib.B2FError(f"cos/sin: expected [>= {rope_row0 + M}, 128] tables, got {tuple(cos.shape)} / "
                            f"{tuple(sin.shape)}")
    if out is None:
        out = torch.empty((*xq.shape[:-1], N), device=xq.device, dtype=torch.bfloat16)
    _req(out, "out")
    o3 = _as3(out)
    _shape(o3, "out", (B, M, N))
    e3 = None
    if out_extra is not None:
        _req(out_extra, "out_extra")
        e3 = _as3(out_extra)
        _shape(e3, "out_extra", (B, M, n_extra))
    check(_lib.lib.b2f_gemm_qkv_norm_rope_fp8(ptr(x3), x3.stride(1), x3.stride(0), ptr(s2), s2.stride(0), ptr(wq),
                                              wq.stride(0), ptr(w_scale), ptr(bias), ptr(o3), o3.stride(1), o3.stride(0),
                                              B, M, N // 3, K, ptr(nq), ptr(nk), ptr(cos), ptr(sin), rope_row0, eps,
                                              n_extra, ptr(e3), 0 if e3 is None else e3.stride(1),
                                              0 if e3 is None else e3.stride(0), epi_extra, stream_ptr()),
          "b2f_gemm_qkv_norm_rope_fp8")
    return out


def _lora_ext(t, bcat, B, M, N):
    """(t3, r_pad) of a LoRA K-extension t [.., M, r_pad] / bcat [N, r_pad] checked against the launch."""
    _req(t, "t")
    _req(bcat, "bcat")
    t3 = _as3(t)
    r_pad = bcat.shape[1]
    _shape(t3, "t", (B, M, r_pad))
    _shape(bcat, "bcat", (N, r_pad))
    return t3, r_pad


def linear_fp8_lora(xq, x_scale, wq, w_scale, bias, t, bcat, *, epilogue: int = EPI_BIAS, out=None, resid=None,
                    gate=None) -> torch.Tensor:
    """out = epilogue(fp32(x_scale[m] * w_scale[n]) * (xq @ wq^T) + t @ bcat^T + bias) via b2f_gemm_fp8_lora: linear_fp8
    with the bf16 LoRA K-extension (t, bcat) of linear_lora accumulated onto the scaled FP8 accumulators."""
    _req(xq, "xq", FP8)
    _req(wq, "wq", FP8)
    _req(w_scale, "w_scale", torch.float32)
    x3 = _as3(xq)
    B, M, K = x3.shape
    s2 = _scales(x_scale, "x_scale", B, M)
    N = wq.shape[0]
    _fp8_weight_checks(wq, w_scale, bias, N, K)
    t3, r_pad = _lora_ext(t, bcat, B, M, N)
    if out is None:
        out = torch.empty((*xq.shape[:-1], N), device=xq.device, dtype=torch.bfloat16)
    _req(out, "out")
    o3 = _as3(out)
    _shape(o3, "out", (B, M, N))
    ldr = rbs = gld = 0
    if epilogue in (EPI_GATE_RESID, EPI_RESID):
        _req(resid, "resid")
        r3 = _as3(resid)
        _shape(r3, "resid", (B, M, N))
        ldr, rbs = r3.stride(1), r3.stride(0)
        if epilogue == EPI_GATE_RESID:
            _req(gate, "gate")
            _shape(gate, "gate", (B, N) if gate.dim() == 2 else (N,))
            gld = gate.stride(0) if gate.dim() == 2 else 0
    check(_lib.lib.b2f_gemm_fp8_lora(ptr(x3), x3.stride(1), x3.stride(0), ptr(s2), s2.stride(0), ptr(wq), wq.stride(0),
                                     ptr(w_scale), ptr(bias), ptr(o3), o3.stride(1), o3.stride(0), B, M, N, K, epilogue,
                                     ptr(resid), ldr, rbs, ptr(gate), gld, ptr(t3), t3.stride(1), t3.stride(0),
                                     ptr(bcat), bcat.stride(0), r_pad, stream_ptr()), "b2f_gemm_fp8_lora")
    return out


def linear_qkv_norm_rope_fp8_lora(xq, x_scale, wq, w_scale, bias, nq, nk, cos, sin, t, bcat, *, rope_row0: int = 0,
                                  out=None, eps: float = 1e-6, out_extra=None, epi_extra: int = EPI_BIAS):
    """linear_qkv_norm_rope_fp8 with the LoRA K-extension of linear_fp8_lora (b2f_gemm_qkv_norm_rope_fp8_lora)."""
    _req(xq, "xq", FP8)
    _req(wq, "wq", FP8)
    _req(w_scale, "w_scale", torch.float32)
    _req(cos, "cos", torch.float32)
    _req(sin, "sin", torch.float32)
    x3 = _as3(xq)
    B, M, K = x3.shape
    s2 = _scales(x_scale, "x_scale", B, M)
    n_extra = 0 if out_extra is None else out_extra.shape[-1]
    N = wq.shape[0] - n_extra
    _fp8_weight_checks(wq, w_scale, bias, N + n_extra, K)
    t3, r_pad = _lora_ext(t, bcat, B, M, N + n_extra)
    _shape(nq, "nq", (128,))
    _shape(nk, "nk", (128,))
    if cos.dim() != 2 or cos.shape[0] < rope_row0 + M or cos.shape[1] != 128 or cos.shape != sin.shape:
        raise _lib.B2FError(f"cos/sin: expected [>= {rope_row0 + M}, 128] tables, got {tuple(cos.shape)} / "
                            f"{tuple(sin.shape)}")
    if out is None:
        out = torch.empty((*xq.shape[:-1], N), device=xq.device, dtype=torch.bfloat16)
    _req(out, "out")
    o3 = _as3(out)
    _shape(o3, "out", (B, M, N))
    e3 = None
    if out_extra is not None:
        _req(out_extra, "out_extra")
        e3 = _as3(out_extra)
        _shape(e3, "out_extra", (B, M, n_extra))
    check(_lib.lib.b2f_gemm_qkv_norm_rope_fp8_lora(
        ptr(x3), x3.stride(1), x3.stride(0), ptr(s2), s2.stride(0), ptr(wq), wq.stride(0), ptr(w_scale), ptr(bias),
        ptr(o3), o3.stride(1), o3.stride(0), B, M, N // 3, K, ptr(nq), ptr(nk), ptr(cos), ptr(sin), rope_row0, eps,
        n_extra, ptr(e3), 0 if e3 is None else e3.stride(1), 0 if e3 is None else e3.stride(0), epi_extra, ptr(t3),
        t3.stride(1), t3.stride(0), ptr(bcat), bcat.stride(0), r_pad, stream_ptr()), "b2f_gemm_qkv_norm_rope_fp8_lora")
    return out


def _row_pitch(t: torch.Tensor) -> int:
    """Token pitch of a [B,S,H,dh] (or [B,S,n]) view; with S = 1 the stride of that dimension is arbitrary and the batch
    pitch is it."""
    B, S = t.shape[:2]
    return t.stride(1) if S > 1 else t.stride(0) if B > 1 else t[0, 0].numel()


def _qkv_views(q, k, v):
    """(B, S, H, dh) of bf16 [B,S,H,dh] views as attention() takes them, with one shape for all three."""
    for t, n in ((q, "q"), (k, "k"), (v, "v")):
        _req(t, n)
        if t.dim() != 4 or t.stride(2) != t.shape[3] or (t.shape[0] > 1 and t.stride(0) != t.shape[1] * _row_pitch(t)):
            raise _lib.B2FError(f"{n}: expected a [B,S,H,dh] view with contiguous heads and batch stride S*ld")
    if not (q.shape == k.shape == v.shape):
        raise _lib.B2FError(f"q, k, v: expected one shape, got {tuple(q.shape)}, {tuple(k.shape)}, {tuple(v.shape)}")
    return tuple(q.shape)


def _fp8_attn_buffers(B, S, H, dh, q8, k8, sq, sk, v8t, sv, device):
    """The operand buffers of b2f_attention_fp8 (include/b2f.h, "FP8 attention"), allocated where None, checked
    (dtype, shape, contiguity) where given."""
    S_pad = (S + 127) // 128 * 128
    want = (("q8", q8, FP8, (B, S, H, dh)), ("k8", k8, FP8, (B, S, H, dh)), ("sq", sq, torch.float32, (B, H)),
            ("sk", sk, torch.float32, (B, H)), ("v8t", v8t, FP8, (B, H, dh, S_pad)),
            ("sv", sv, torch.float32, (B, H, dh)))
    out = []
    for n, t, dt, shp in want:
        if t is None:
            t = torch.empty(shp, device=device, dtype=dt)
        _req(t, n, dt)
        _shape(t, n, shp)
        if not t.is_contiguous():
            raise _lib.B2FError(f"{n}: must be contiguous")
        out.append(t)
    return out


def attn_quant_fp8(q, k, v, *, q8=None, k8=None, sq=None, sk=None, v8t=None, sv=None):
    """(q8, k8, sq, sk, v8t, sv) of b2f_attn_quant_fp8: q, k, v bf16 [B,S,H,dh] views as attention() takes them ->
    q8 / k8 e4m3 [B,S,H,dh] with per-head scales sq / sk fp32 [B,H], v8t e4m3 [B,H,dh,S_pad] (tokens contiguous, in the
    P-fragment order of include/b2f.h, padding +0) with per-channel scales sv fp32 [B,H,dh]."""
    B, S, H, dh = _qkv_views(q, k, v)
    bufs = _fp8_attn_buffers(B, S, H, dh, q8, k8, sq, sk, v8t, sv, q.device)
    q8, k8, sq, sk, v8t, sv = bufs
    check(_lib.lib.b2f_attn_quant_fp8(ptr(q), _row_pitch(q), ptr(k), _row_pitch(k), ptr(v), _row_pitch(v), ptr(q8), ptr(k8),
                                      ptr(sq), ptr(sk), ptr(v8t), ptr(sv), B, H, S, dh, stream_ptr()),
          "b2f_attn_quant_fp8")
    return tuple(bufs)


def attention_fp8(q8, k8, sq, sk, v8t, sv, *, out=None, scale: float | None = None, causal: bool = False,
                  bias=None) -> torch.Tensor:
    """softmax(q k^T * scale) v via b2f_attention_fp8 from the buffers of attn_quant_fp8; out [B,S,H*dh] bf16 (any row
    pitch).  Non-causal, without a bias: anything else raises."""
    if bias is not None:
        raise _lib.B2FError("attention_fp8: a score bias is not supported")
    _req(q8, "q8", FP8)
    if q8.dim() != 4:
        raise _lib.B2FError(f"q8: expected [B,S,H,dh], got {tuple(q8.shape)}")
    B, S, H, dh = q8.shape
    q8, k8, sq, sk, v8t, sv = _fp8_attn_buffers(B, S, H, dh, q8, k8, sq, sk, v8t, sv, q8.device)
    if out is None:
        out = torch.empty((B, S, H * dh), device=q8.device, dtype=torch.bfloat16)
    _req(out, "out")
    _shape(out, "out", (B, S, H * dh))
    if B > 1 and out.stride(0) != S * out.stride(1):
        raise _lib.B2FError("out: expected batch stride S * row pitch")
    check(_lib.lib.b2f_attention_fp8(ptr(q8), ptr(k8), ptr(sq), ptr(sk), ptr(v8t), ptr(sv), ptr(out), out.stride(1), B,
                                     H, S, dh, float(dh ** -0.5 if scale is None else scale), int(causal), stream_ptr()),
          "b2f_attention_fp8")
    return out
