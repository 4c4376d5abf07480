"""References of the FP8 attention path (include/b2f.h, "FP8 attention").

  quant_attn         b2f_attn_quant_fp8, bit-exact: fp8_ref.quant_rows over one (batch item, head) of Q / K and one
                     (batch item, head, channel) of V, and v8t's token order (V8T_TOKEN) and +0 padding;
  attention_fp8_emu  b2f_attention_fp8: kernel_ref.attention_emu with the FP8 quantization points (Q8 K8^T in fp64,
                     P8 = e4m3(256 p), O += P8 V8, out = bf16(O sv / 256 / l)) and the floor of fp8_ref's accumulation
                     (on P8 V8, and on Q8 K8^T carried through the softmax) plus one e4m3 step of the largest P8 |V|
                     term plus bf16 output rounding;
  fp8_attention()    a context in which oracle.flux_oracle.attention quantizes as the engine does (combines with
                     fp8_linears()).
"""
from __future__ import annotations

import contextlib
import math

import torch

import fp8_ref as Q
import kernel_ref as R
from oracle import flux_oracle as fo

F64 = torch.float64
BLOCK = 128


def v8t_token(p: int) -> int:
    """The token (within its 32-token group) at k-position p of v8t."""
    return (p & 16) + 2 * ((p & 15) >> 2) + (p & 1) + 8 * ((p >> 1) & 1)


V8T_TOKEN = torch.tensor([v8t_token(p) for p in range(32)])


def v8t_order(S_pad: int) -> torch.Tensor:
    """idx [S_pad]: v8t[..., p] holds token idx[p]."""
    p = torch.arange(S_pad)
    return (p & ~31) + V8T_TOKEN[p & 31]


def s_pad(S: int) -> int:
    return (S + 127) // 128 * 128


def quant_attn(q, k, v):
    """(q8, k8, sq, sk, v8t, sv) of b2f_attn_quant_fp8 for q, k, v [B, S, H, D] (any float dtype; quantized from
    x.float()): q8 / k8 e4m3 [B, S, H, D], sq / sk fp32 [B, H], v8t e4m3 [B, H, D, S_pad], sv fp32 [B, H, D]."""
    B, S, H, D = q.shape

    def per_head(x):
        x8, s = Q.quant_rows(x.permute(0, 2, 1, 3).reshape(B, H, S * D))
        return x8.view(torch.uint8).reshape(B, H, S, D).permute(0, 2, 1, 3).contiguous().view(Q.E4M3), s

    q8, sq = per_head(q)
    k8, sk = per_head(k)
    v8, sv = Q.quant_rows(v.permute(0, 2, 3, 1))                         # rows: (b, h, channel) over S tokens
    P = s_pad(S)
    vt = torch.zeros(B, H, D, P, dtype=torch.uint8, device=v.device)   # +0 padding
    vt[..., :S] = v8.view(torch.uint8)
    v8t = vt[..., v8t_order(P).to(v.device)].contiguous().view(Q.E4M3)
    return q8, k8, sq, sk, v8t, sv


def v8t_tokens(v8t: torch.Tensor, S: int) -> torch.Tensor:
    """v8t [..., S_pad] back in token order, [..., S]."""
    P = v8t.shape[-1]
    inv = torch.empty(P, dtype=torch.long)
    inv[v8t_order(P)] = torch.arange(P)
    u = v8t.view(torch.uint8)[..., inv.to(v8t.device)]
    return u[..., :S].contiguous().view(Q.E4M3)


def score_scale(sq, sk, scale):
    """c = fp32(fp32(sq * sk) * fp32(scale * log2 e)) per (batch item, head), as fp64 [B, H]; scale is rounded to fp32
    (the kernel's argument) and multiplied by log2 e in double, as the host does."""
    s32 = torch.tensor(scale, dtype=torch.float32).item()
    return ((sq.float() * sk.float()) * torch.tensor(s32 * R.LOG2E, dtype=torch.float32)).to(F64)


def _online(t, v8, *, quant_p=True, block=BLOCK):
    """The kernel's online softmax on base-2 scores t [B, H, Sq, Skv] (fp64) and V values v8 [B, H, Skv, D] (fp64):
    (O, l, m) with P~ = e4m3(256 p) (or 256 p unrounded when not quant_p)."""
    B, H, Sq, Skv = t.shape
    m = torch.full((B, H, Sq, 1), -math.inf, dtype=F64, device=t.device)
    l = torch.zeros_like(m)
    o = torch.zeros(B, H, Sq, v8.shape[-1], dtype=F64, device=t.device)
    for j0 in range(0, Skv, block):
        tj = t[..., j0:j0 + block]
        m_new = torch.maximum(m, tj.amax(-1, keepdim=True))
        alpha = torch.where(m == -math.inf, torch.zeros_like(m), torch.exp2(m - m_new))
        p = torch.exp2(tj - torch.where(m_new == -math.inf, torch.zeros_like(m_new), m_new))
        l = l * alpha + p.sum(-1, keepdim=True)
        p8 = (p * 256).float().to(Q.E4M3).to(F64) if quant_p else p * 256
        o = o * alpha + p8 @ v8[..., j0:j0 + block, :]
        m = m_new
    return o, l, m


def attention_fp8_core(q8, k8, sq, sk, v8, sv, scale, *, quant_p=True, block=BLOCK):
    """out [B, H, S, D] fp64 (unrounded) of the kernel arithmetic on e4m3 operands in head-major layout: q8 / k8 / v8
    [B, H, S, D] e4m3 (or any float: the identity quantization), sq / sk [B, H], sv [B, H, D]."""
    c = score_scale(sq, sk, scale)[..., None, None]
    t = (q8.to(F64) @ k8.to(F64).transpose(-1, -2)) * c
    o, l, _ = _online(t, v8.to(F64), quant_p=quant_p, block=block)
    return o * (sv.to(F64)[..., None, :] / 256) / l


def attention_fp8_emu(q, k, v, *, scale=None, p_acc: float = 11.0, block=BLOCK):
    """(out, floor, math) for b2f_attn_quant_fp8 + b2f_attention_fp8 on bf16 q, k, v [B, S, H, D]: out [B, S, H*D] is
    the bf16-rounded emulation, floor its per-element allowance, math the fp64 unquantized attention.

    floor = max(Skv 2^-24, 2^-p_acc) * (P @ |V~|)          the FP8 tensor cores' accumulation of P8 V8 (fp8_ref)
            + ln 2 * (W @ |V~| + rowsum(W) * |out|)         the same accumulation allowance on Q8 K8^T, dt = c 2^-p_acc
                                                            (|Q8| |K8|^T) in base-2 score units, carried through the
                                                            softmax to first order (W = P * dt)
            + 2^-3 * max_j P_j |V~_j|                       one e4m3 step of the largest term: p carries the error of
                                                            its score and of ex2.approx, so where 256 p lies that close
                                                            to an e4m3 tie, P8 rounds the other way
    with P the normalized probabilities and V~ the dequantized V; bf16 output rounding is the unit of ulp_diff."""
    B, S, H, D = q.shape
    scale = D ** -0.5 if scale is None else scale
    q8, k8, sq, sk, v8t, sv = quant_attn(q, k, v)
    hm = lambda x: x.permute(0, 2, 1, 3)
    v8 = v8t_tokens(v8t, S).transpose(-1, -2)                          # [B, H, S, D]
    o = attention_fp8_core(hm(q8), hm(k8), sq, sk, v8, sv, scale, block=block)
    vd = v8.to(F64) * sv.to(F64)[..., None, :]
    qd, kd = hm(q8).to(F64), hm(k8).to(F64)
    c = score_scale(sq, sk, scale)[..., None, None]
    P = torch.softmax(qd @ kd.transpose(-1, -2) * c * math.log(2), -1)
    W = P * (c * 2.0 ** -p_acc * (qd.abs() @ kd.abs().transpose(-1, -2)))
    floor = (max(S * R.U32, 2.0 ** -p_acc) * (P @ vd.abs())
             + math.log(2) * (W @ vd.abs() + W.sum(-1, keepdim=True) * o.abs())
             + 2.0 ** -3 * R.max_outer(P, vd.abs()))
    flat = lambda a: a.permute(0, 2, 1, 3).reshape(B, S, H * D)
    mth, _ = R.attention_math(q, k, v, scale=scale)
    return flat(R.bf16r(o)), flat(floor), mth


def attention_fp8_reference(q, k, v, scale=None):
    """fp64 out [B, H, S, D] of the FP8 attention on head-major q, k, v [B, H, S, D] of any dtype: the quantization of
    b2f_attn_quant_fp8 and the kernel arithmetic, unrounded."""
    qt, kt, vt = (x.transpose(1, 2) for x in (q, k, v))
    B, S, H, D = qt.shape
    q8, k8, sq, sk, v8t, sv = quant_attn(qt, kt, vt)
    hm = lambda x: x.permute(0, 2, 1, 3)
    v8 = v8t_tokens(v8t, S).transpose(-1, -2)
    return attention_fp8_core(hm(q8), hm(k8), sq, sk, v8, sv, D ** -0.5 if scale is None else scale)


@contextlib.contextmanager
def fp8_attention():
    """The oracle with its joint attention in FP8: Q / K quantized per head, V per channel, P to e4m3(256 p) in the
    kernel's 128-token online softmax; the result in q's dtype."""
    old = fo.attention

    def attn(q, k, v, attn_mask=None):
        assert attn_mask is None
        return attention_fp8_reference(q, k, v).to(q.dtype)

    fo.attention = attn
    try:
        yield
    finally:
        fo.attention = old
