"""fp64 references of the HBM-bound row kernels (elementwise.cu, train_kernels.cu, llm_kernels.cu, vae_kernels.cu).

Same conventions as kernel_ref.py: every function takes the kernel's bf16 / fp32 inputs and returns
(emu, floor, math), all float64:

  emu    the rounding chain documented above the kernel, evaluated exactly (the kernel's fp32 statistics, sums and
         transcendental values are exact here; its bf16 roundings are not skipped);
  floor  the fp32 allowance: K * 2^-24 * (the same reduction over |inputs|) for a reduction of depth K, a few fp32
         ulps per transcendental, plus the first-order effect of one flip at each intermediate bf16 rounding;
  math   the exact operation, no rounding.

bf16 outputs are checked with Checker.bf16 (ulps of emu, never in units below floor), fp32 outputs with
Checker.within_floor against emu.  K is the length of the longest sequential fp32 accumulation chain of the kernel
(per-thread loop + shuffle tree + the cross-block sum), not the number of terms, so it follows the launch formulas.
"""
from __future__ import annotations

import math

import torch

from kernel_ref import F64, LOG2E, U32, _rot_pairs, bf16r, d64, gelu_tanh, silu, ulp_bf16

f32 = lambda v: float(torch.tensor(v, dtype=torch.float32))   # a host scalar as the kernel receives it


def warp_depth(D: int) -> int:
    """Accumulation depth of a warp-per-row reduction: D / 32 sequential terms per lane, then 5 shuffle levels."""
    return D // 32 + 5


def per_row(a, b, rows: int, split_row: int):
    """[B, D] parameter rows -> [B, rows, D]: rows < split_row take `a`, the others `b` (split_row = 0: all `a`)."""
    a = d64(a)[:, None, :].expand(-1, rows, -1)
    if split_row <= 0:
        return a
    b = d64(b)[:, None, :].expand(-1, rows, -1)
    r = torch.arange(rows, device=a.device)[None, :, None]
    return torch.where(r < split_row, a, b)


# ---------------------------------------------------------------------------------------------------- AdaLN modulate
def _ln_stats(x, eps):
    D = x.shape[-1]
    mean = x.mean(-1, keepdim=True)
    rstd = torch.rsqrt(((x - mean) ** 2).mean(-1, keepdim=True) + eps)
    xh = (x - mean) * rstd
    K = warp_depth(D)
    # fp32 error of xhat: the mean (K-deep sum of x), the centred sum of squares, the final products
    f_xh = K * U32 * (rstd * x.abs().mean(-1, keepdim=True) + xh.abs()) + 4 * U32 * xh.abs()
    return mean, rstd, xh, f_xh


def ln_modulate_emu(x, scale, shift, *, eps=1e-6, split_row=0, scale_b=None, shift_b=None):
    """ln_modulate: bf16(bf16(bf16(LN(x)) * bf16(1 + scale)) + shift), fp32 two-pass statistics; x [B, rows, D]."""
    xd = d64(x)
    rows = xd.shape[1]
    sc = per_row(scale, scale_b, rows, split_row)
    sh = per_row(shift, shift_b, rows, split_row)
    _, _, xh, f_xh = _ln_stats(xd, eps)
    y = bf16r(xh)
    t = bf16r(1 + sc)
    z = bf16r(y * t)
    emu = bf16r(z + sh)
    # y = bf16(xhat) may flip where the fp32 xhat lies within f_xh of a tie; z = bf16(y t) is then off by the flip
    # and its own rounding.  Elsewhere y and z are exact and only the fp32 error of xhat is allowed.
    near = _near_tie(xh, f_xh)
    floor = t.abs() * f_xh + near * (t.abs() * ulp_bf16(y) + ulp_bf16(z))
    return emu, floor, xh * (1 + sc) + sh


def ln_modulate_bwd_emu(x, dy, scale, *, eps=1e-6, split_row=0, scale_b=None, dres=None, part_row0=0):
    """ln_modulate_bwd.  Returns ((emu, floor, math) of dres_out, (ref, floor) of dscale, (ref, floor) of dshift):

      g = dy * bf16(1 + scale);  dx = rstd (g - mean g - xhat mean(g xhat));  dres_out = bf16(dres + bf16(dx))
      dscale[b] = sum_{rows >= part_row0} dy * bf16(xhat);  dshift[b] = sum_{rows >= part_row0} dy"""
    xd, d = d64(x), d64(dy)
    B, rows, D = xd.shape
    _, rstd, xh, f_xh = _ln_stats(xd, eps)
    t = bf16r(1 + per_row(scale, scale_b, rows, split_row))
    g = d * t
    c1 = g.mean(-1, keepdim=True)
    c2 = (g * xh).mean(-1, keepdim=True)
    dx = rstd * (g - c1 - xh * c2)
    K = warp_depth(D)
    f_dx = rstd * (K * U32 * ((g.abs().mean(-1, keepdim=True) + (g * xh).abs().mean(-1, keepdim=True))
                              + xh.abs() * (g * xh).abs().mean(-1, keepdim=True))
                   + c2.abs() * f_xh) + K * U32 * dx.abs() + 4 * U32 * rstd * (g.abs() + c1.abs() + (xh * c2).abs())
    r0 = torch.zeros_like(xd) if dres is None else d64(dres)
    dxb = bf16r(dx)
    if dres is None:
        emu, floor = dxb, f_dx
    else:
        emu, floor = bf16r(r0 + dxb), f_dx + ulp_bf16(dxb) * _near_tie(dx, f_dx)
    # exact math: autograd-free closed form of the same gradient with exact (1 + scale)
    tm = 1 + per_row(scale, scale_b, rows, split_row)
    gm = d * tm
    dx_m = rstd * (gm - gm.mean(-1, keepdim=True) - xh * (gm * xh).mean(-1, keepdim=True))
    part = d[:, part_row0:]
    xhb = bf16r(xh)[:, part_row0:]
    n = max(rows - part_row0, 1)
    # the fp32 xhat that the kernel rounds may sit on the other side of a bf16 tie: one flip per term
    ds = (part * xhb).sum(1)
    f_ds = (n + 4) * U32 * (part * xhb).abs().sum(1) + (part.abs() * (ulp_bf16(xhb) * _near_tie(xh, f_xh)[:, part_row0:])).sum(1)
    dh = part.sum(1)
    f_dh = (n + 4) * U32 * part.abs().sum(1)
    return (emu, floor, r0 + dx_m), (ds, f_ds), (dh, f_dh)


def _near_tie(v, f):
    """1 where the value v, known to within f, may round to bf16 on either side of a tie; else 0."""
    r = bf16r(v)
    u = ulp_bf16(r)
    return ((u / 2 - (v - r).abs()).abs() <= f + 1e-300).to(F64)


# ---------------------------------------------------------------------------------------------------- gates
def gate_resid_emu(x, y, gate, *, split_row=0, gate_b=None):
    """gate_resid_fwd: bf16(x + bf16(gate[b] * y)) — exact products / sums of bf16 values, bit-exact."""
    g = per_row(gate, gate_b, x.shape[1], split_row)
    return bf16r(d64(x) + bf16r(g * d64(y)))


def gate_bwd_emu(dout, *, y=None, gate=None, gate_b=None, split_row=0, part_row0=0):
    """gate_bwd: (dy = bf16(gate[b] * dout), bit-exact or None;  (ref, floor) of col[b] = sum_{rows >= part_row0}
    dout * y, or the plain column sum of dout when y is None)."""
    d = d64(dout)
    B, rows, D = d.shape
    dy = None if gate is None else bf16r(per_row(gate, gate_b, rows, split_row) * d)
    terms = d[:, part_row0:] * (1.0 if y is None else d64(y)[:, part_row0:])
    # per thread: the rows of one 32-row chunk; then col_reduce over the chunks
    K = 32 + (rows + 31) // 32
    return dy, (terms.sum(1), K * U32 * terms.abs().sum(1))


def col_reduce_emu(partial, out_old=None):
    """col_reduce: out[b, c] (+)= sum_k partial[b, k, c] (fixed order).  partial [B, nchunks, D]."""
    p = d64(partial)
    s = p.sum(1)
    fl = p.shape[1] * U32 * p.abs().sum(1)
    if out_old is None:
        return s, fl
    o = d64(out_old)
    return o + s, fl + U32 * (o + s).abs()


# ---------------------------------------------------------------------------------------------------- QKV RMSNorm + RoPE
def rmsnorm_rope_emu(x, wq_b, wk_b, cos, sin, *, wq_a=None, wk_a=None, n_a=0, eps=1e-6):
    """rmsnorm_rope_ / rmsnorm_rope_out on x = (xq, xk), each [B, S, H, 128]:
    y = bf16(x r), z = bf16(y w), out = bf16(z cos + rot(z) sin); tokens s < n_a use weight set A."""
    outs = []
    S = x[0].shape[1]
    c = d64(cos)[None, :S, None, :]
    s_ = d64(sin)[None, :S, None, :]
    for xi, wa, wb in ((x[0], wq_a, wq_b), (x[1], wk_a, wk_b)):
        xd = d64(xi)
        w = _wset(wa, wb, S, n_a)
        r = torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + eps)
        y = bf16r(xd * r)
        z = bf16r(y * w)
        emu = bf16r(z * c + _rot_pairs(z) * s_)
        zm = xd * r * w
        mth = zm * c + _rot_pairs(zm) * s_
        f_y = 12 * U32 * xd.abs() * r                  # fp32 error of x r (the 16-lane sum of squares, rsqrtf)
        sl = w.abs() * f_y + _near_tie(xd * r, f_y) * (w.abs() * ulp_bf16(y) + ulp_bf16(z))
        slp = torch.maximum(sl, _rot_pairs(sl).abs())
        floor = slp * (c.abs() + s_.abs()) + 2 * U32 * (z.abs() * c.abs() + _rot_pairs(z).abs() * s_.abs())
        outs.append((emu, floor, mth))
    return outs


def _wset(wa, wb, S, n_a):
    """[1, S, 1, 128] per-token norm weights: set A for s < n_a, set B after."""
    b = d64(wb)[None, None, None, :].expand(1, S, 1, -1)
    if n_a <= 0:
        return b
    a = d64(wa)[None, None, None, :].expand(1, S, 1, -1)
    s = torch.arange(S, device=b.device)[None, :, None, None]
    return torch.where(s < n_a, a, b)


def rmsnorm_rope_bwd_emu(x, do, wq_b, wk_b, cos, sin, *, wq_a=None, wk_a=None, n_a=0, eps=1e-6):
    """rmsnorm_rope_bwd_ on (xq, xk) / (dq, dk), each [B, S, H, 128] (the comment above the kernel):

      dy = rope^T(do): dy0 = do0 c0 + do1 s1, dy1 = do1 c1 - do0 s0
      dx = bf16(r (dy w - x r^2 mean(dy w x)));   dw[set] = sum over tokens of the set and heads of dy bf16(x r)

    Returns ([(emu, floor, math) of dq, of dk], (ref [4, 128], floor) of the weight gradients in the order
    (set A q, set A k, set B q, set B k))."""
    B, S, H, _ = x[0].shape
    c = d64(cos)[None, :S, None, :]
    s_ = d64(sin)[None, :S, None, :]
    sa = (torch.arange(S, device=c.device) < n_a)[None, :, None, None]
    grads, wg, wf = [], [], []
    for xi, di, wa, wb in ((x[0], do[0], wq_a, wq_b), (x[1], do[1], wk_a, wk_b)):
        xd, dd = d64(xi), d64(di)
        w = _wset(wa, wb, S, n_a)
        r = torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + eps)
        d2 = dd.unflatten(-1, (-1, 2))
        c2, s2 = c.unflatten(-1, (-1, 2)), s_.unflatten(-1, (-1, 2))
        dy = torch.stack([d2[..., 0] * c2[..., 0] + d2[..., 1] * s2[..., 1],
                          d2[..., 1] * c2[..., 1] - d2[..., 0] * s2[..., 0]], -1).flatten(-2)
        dya = torch.stack([d2[..., 0].abs() * c2[..., 0].abs() + d2[..., 1].abs() * s2[..., 1].abs(),
                           d2[..., 1].abs() * c2[..., 1].abs() + d2[..., 0].abs() * s2[..., 0].abs()], -1).flatten(-2)
        gx = (dy * w * xd).mean(-1, keepdim=True)
        dx = r * (dy * w - xd * r * r * gx)
        f_dx = 24 * U32 * r * (dya * w.abs() + xd.abs() * r * r * (dya * w.abs() * xd.abs()).mean(-1, keepdim=True))
        grads.append((bf16r(dx), f_dx, dx))
        xr = xd * r
        t = dy * bf16r(xr)
        # per warp: H heads; 8 warps per block; col_reduce over the blocks
        K = H + 8 + (B * S + 7) // 8 + 2
        fl_t = K * U32 * (dya * bf16r(xr).abs()) + dya * ulp_bf16(bf16r(xr)) * _near_tie(xr, 12 * U32 * xr.abs())
        for m in (sa, ~sa):
            wg.append((t * m).sum((0, 1, 2)))
            wf.append((fl_t * m).sum((0, 1, 2)))
    order = [0, 2, 1, 3]     # (q A, q B, k A, k B) -> (q A, k A, q B, k B)
    return grads, (torch.stack([wg[i] for i in order]), torch.stack([wf[i] for i in order]))


# ---------------------------------------------------------------------------------------------------- timestep embedding
def silu_emu(x):
    """silu (and the SiLU of temb_combine): bf16(x / (1 + __expf(-x))).  __expf carries an argument error of |x|
    fp32 ulps."""
    xd = d64(x)
    v = silu(xd)
    return bf16r(v), (xd.abs() + 8) * U32 * v.abs(), v


def temb_sinusoid_emu(t):
    """temb_sinusoid: out[r] = [cos(t f) | sin(t f)], f_j = exp(-ln(1e4) j / 128), fp32 math, bf16 output.
    The fp32 angle t f is off by (2 |ln(1e4) j / 128| + 6) fp32 ulps of itself (exponent, expf, the product), which
    moves cos / sin by that much times sin / cos; cosf / sinf add 2 ulps."""
    td = d64(t)[:, None]
    arg = -math.log(10000.0) * torch.arange(128, device=td.device, dtype=F64) / 128
    a = td * torch.exp(arg)[None]
    ea = a.abs() * (2 * arg.abs() + 6)[None] * U32
    c, s = torch.cos(a), torch.sin(a)
    mth = torch.cat([c, s], 1)
    floor = torch.cat([s.abs() * ea + 2 * U32 * c.abs(), c.abs() * ea + 2 * U32 * s.abs()], 1)
    return bf16r(mth), floor, mth


def temb_combine_emu(t, g, txt):
    """temb_combine: temb = bf16(bf16(t + g) + txt) (g None: bf16(t + txt)), bit-exact; silu_temb = silu_emu(temb).
    Returns (temb, (emu, floor, math) of silu_temb)."""
    a = d64(t)
    if g is not None:
        a = bf16r(a + d64(g))
    temb = bf16r(a + d64(txt))
    return temb, silu_emu(temb)


def rope_tables_emu(ids, axes=(16, 56, 56), theta=10000.0):
    """rope_tables (FluxPosEmbed): fp64 angle ids[:, axis] * theta^(-2i / dim) and cos / sin, each value repeated
    twice, cast to fp32.  Returns (cos, sin, floor): fp64 values and one fp32 ulp of each."""
    cols = []
    for a, dim in enumerate(axes):
        w = 1.0 / theta ** (torch.arange(0, dim, 2, device=ids.device, dtype=F64) / dim)
        cols.append(d64(ids[:, a:a + 1]) * w[None])
    ang = torch.cat(cols, 1).repeat_interleave(2, 1)
    c, s = torch.cos(ang), torch.sin(ang)
    ulp32 = lambda v: torch.ldexp(torch.ones_like(v), torch.frexp(v.abs())[1] - 24).clamp_min(2.0 ** -149)
    return c, s, (ulp32(c), ulp32(s))


def cast_emu(x, to_f32):
    """cast_bf16_f32: bf16 -> fp32 is exact, fp32 -> bf16 one round-to-nearest-even; bit-exact either way."""
    return d64(x) if to_f32 else bf16r(x)


# ---------------------------------------------------------------------------------------------------- small training kernels
def gelu_rows_emu(x):
    """gelu_rows: bf16(0.5 u (1 + tanhf(k0 (u + k1 u^3)))) — one rounding of an fp32 transcendental."""
    u = d64(x)
    v = gelu_tanh(u)
    return bf16r(v), 8 * U32 * (u.abs() + v.abs()), v


def outer_acc_emu(dmod, act, out_old=None):
    """outer_acc: dW[n, k] (+)= sum_b dmod[b, n] act[b, k] (fp32)."""
    a, g = d64(act), d64(dmod)
    ref = g.T @ a
    fl = (g.shape[0] + 1) * U32 * (g.abs().T @ a.abs())
    if out_old is not None:
        ref = ref + d64(out_old)
        fl = fl + U32 * ref.abs()
    return ref, fl


def attn_delta_emu(o, dout, B, H, S):
    """attn_delta: delta[b, h, s] = sum_c dO o over the 128 columns of head h ([B*S, >= H*128] row views)."""
    t = (d64(o)[:, :H * 128] * d64(dout)[:, :H * 128]).reshape(B, S, H, 128)
    return t.sum(-1).permute(0, 2, 1), 20 * U32 * t.abs().sum(-1).permute(0, 2, 1)


def mse_loss_emu(pred, target, weight=None, grad_scale=1.0):
    """mse_loss: (loss ref, floor), (dpred emu, floor, math).  loss = sum(w d^2) / n as the sum of per-block
    partials; dpred = bf16(2 w d * fp32(grad_scale / n))."""
    p, t = d64(pred).flatten(), d64(target).flatten()
    n = p.numel()
    w = torch.ones_like(p) if weight is None else d64(weight).flatten()
    d = p - t
    loss = (w * d * d).sum() / n
    blocks = max(1, min(n // 256, 1024))
    K = -(-n // (blocks * 256)) + 13 + blocks
    f_d = U32 * (p.abs() + t.abs())                 # fp32 rounding of pred - target
    f_loss = (K * U32 * (w * d * d).sum() + 2 * (w * d.abs() * f_d).sum()) / n + U32 * loss.abs()
    gs = f32(f32(grad_scale) / f32(float(n)))
    v = 2 * w * d * gs
    emu = bf16r(v)
    floor = 2 * w * gs * f_d + 4 * U32 * v.abs()
    return (loss, f_loss), (emu.reshape(pred.shape), floor.reshape(pred.shape), (2 * w * d * grad_scale / n).reshape(pred.shape))


def sumsq_blocks(n: int) -> int:
    """Grid of grad_sumsq (train_kernels.cu): n / 1024 blocks, at least 1, at most 1024."""
    return max(1, min(n // 1024, 1024))


def grad_sumsq_emu(g, old=None):
    """grad_sumsq: (sum g^2 (+ old), floor).  Depth: the per-thread loop, the block tree, col_reduce over blocks."""
    x = d64(g).flatten()
    n = x.numel()
    blocks = sumsq_blocks(n)
    K = -(-n // (blocks * 256)) + 13 + blocks + 1
    s = (x * x).sum()
    if old is not None:
        s = s + d64(old).flatten()[0]
    return s, K * U32 * s.abs()


def clip_coef_emu(sumsq, max_norm, pre_scale=1.0):
    """clip_coef: norm = sqrt(sumsq) * pre_scale;  coef = min(1, max_norm / (norm + 1e-6)) * pre_scale (1 if
    max_norm <= 0).  Returns (coef, norm) in fp64 and the allowance of a few correctly rounded fp32 operations."""
    ss = d64(sumsq).flatten()[0]
    ps, mn = f32(pre_scale), f32(max_norm)
    nrm = torch.sqrt(ss) * ps
    c = mn / (nrm + f32(1e-6)) if mn > 0 else torch.ones_like(nrm)
    coef = torch.clamp(c, max=1.0) * ps
    return coef, 4 * U32 * coef.abs(), nrm, 4 * U32 * nrm.abs()


def adamw_emu(p32, m, v, g, *, lr, betas, eps, wd, step, gscale=None):
    """adamw_step_ (train_kernels.cu adamw_one), fp64 with the kernel's fp32 constants:

      g *= gs;  m = b1 m + (1 - b1) g;  v = b2 v + (1 - b2) g^2;  p *= 1 - lr wd;
      p -= (lr / bc1) m / (sqrt(v) / sqrt(bc2) + eps),  bc = 1 - powf(beta, step) in fp32

    Returns ((p, floor), (m, floor), (v, floor))."""
    b1, b2 = f32(betas[0]), f32(betas[1])
    lr_, eps_, wd_ = f32(lr), f32(eps), f32(wd)
    bc1 = f32(1.0 - f32(b1 ** step))
    bc2 = f32(1.0 - f32(b2 ** step))
    gs = 1.0 if gscale is None else d64(gscale).flatten()[0]
    gg = d64(g) * gs
    m1 = b1 * d64(m) + f32(1 - b1) * gg
    v1 = b2 * d64(v) + f32(1 - b2) * gg * gg
    fm = 4 * U32 * (b1 * d64(m).abs() + f32(1 - b1) * gg.abs())
    fv = 4 * U32 * (b2 * d64(v).abs() + f32(1 - b2) * gg * gg)
    p = d64(p32) * f32(1 - lr_ * wd_)
    den = torch.sqrt(v1) / math.sqrt(bc2) + eps_
    upd = f32(lr_ / bc1) * m1 / den
    p1 = p - upd
    # fp32 ops of the update (incl. the error of m, v carried through) and of the decayed parameter
    fp = 3 * U32 * p.abs() + upd.abs() * (8 * U32 + fm / m1.abs().clamp_min(1e-300)
                                          + 0.5 * fv / v1.clamp_min(1e-300)) + U32 * p1.abs()
    return (p1, fp), (m1, fm), (v1, fv)


# ---------------------------------------------------------------------------------------------------- LLM / text encoders
def rmsnorm_emu(x, w, eps=1e-6):
    """rmsnorm (Qwen2RMSNorm): bf16(w * bf16(x rs)), rs = rsqrt(mean(x^2) + eps); x [rows, D]."""
    xd = d64(x)
    D = xd.shape[-1]
    rs = torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + eps)
    y = bf16r(xd * rs)
    wd = d64(w)
    emu = bf16r(wd * y)
    f_y = (warp_depth(D) + 4) * U32 * (xd * rs).abs()
    floor = wd.abs() * (f_y + ulp_bf16(y) * _near_tie(xd * rs, f_y))
    return emu, floor, wd * xd * rs


def layernorm_emu(x, w, b, eps=1e-5):
    """layernorm (nn.LayerNorm, affine): bf16((x - mean) rs w + b), fp32 two-pass statistics, one rounding."""
    xd = d64(x)
    _, _, xh, f_xh = _ln_stats(xd, eps)
    wd, bd = d64(w), d64(b)
    v = xh * wd + bd
    return bf16r(v), wd.abs() * f_xh + 4 * U32 * ((xh * wd).abs() + bd.abs()), v


def rope_half_emu(x, heads, head_pitch, cos, sin, *, fp32_math):
    """rope_half_ on x [tokens, >= heads * head_pitch], rotating the first rot = cos.shape[-1] columns of each head:
      vision (fp32_math): bf16(a c0 - b s0), bf16(b c1 + a s1)             ulp, floor of the fp32 products
      text:               bf16(bf16(a c0) + bf16(-b s0)), ...              bit-exact (bf16-valued cos / sin)
    Columns outside the rotated parts are returned unchanged."""
    xd = d64(x).clone()
    rot = cos.shape[-1]
    half = rot // 2
    c, s = d64(cos), d64(sin)
    emu, floor, mth = xd.clone(), torch.zeros_like(xd), xd.clone()
    for h in range(heads):
        lo = slice(h * head_pitch, h * head_pitch + half)
        hi = slice(h * head_pitch + half, h * head_pitch + rot)
        a, b = xd[:, lo], xd[:, hi]
        c0, c1, s0, s1 = c[:, :half], c[:, half:], s[:, :half], s[:, half:]
        mth[:, lo], mth[:, hi] = a * c0 - b * s0, b * c1 + a * s1
        if fp32_math:
            emu[:, lo], emu[:, hi] = bf16r(mth[:, lo]), bf16r(mth[:, hi])
            floor[:, lo] = 2 * U32 * (a.abs() * c0.abs() + b.abs() * s0.abs())
            floor[:, hi] = 2 * U32 * (b.abs() * c1.abs() + a.abs() * s1.abs())
        else:
            emu[:, lo] = bf16r(bf16r(a * c0) + bf16r(-b * s0))
            emu[:, hi] = bf16r(bf16r(b * c1) + bf16r(a * s1))
    return emu, floor, mth


def _gated(gu, inter, act, f_act):
    g, u = d64(gu)[:, :inter], d64(gu)[:, inter:2 * inter]
    a = act(g)
    ab = bf16r(a)
    fa = f_act(g, a)
    return bf16r(ab * u), u.abs() * (fa + ulp_bf16(ab) * _near_tie(a, fa)), a * u


def swiglu_emu(gu, inter):
    """swiglu: bf16(bf16(g / (1 + __expf(-g))) u).  __expf carries an argument error of |g| fp32 ulps."""
    return _gated(gu, inter, silu, lambda g, a: (g.abs() + 8) * U32 * a.abs())


def geglu_emu(gu, inter):
    """geglu: bf16(bf16(0.5 g (1 + tanhf(.))) u)."""
    return _gated(gu, inter, gelu_tanh, lambda g, a: 8 * U32 * (g.abs() + a.abs()))


# ---------------------------------------------------------------------------------------------------- VAE
GN_THREADS, GN_PIX_PER_BLOCK = 256, 512


def groupnorm_silu_emu(x, gamma, beta, *, eps=1e-6, silu_on=True, groups=32):
    """groupnorm_silu on x [N, P, C] (NHWC): per (item, group) mean / var = E[x^2] - mean^2,
    v = bf16((x - mean) rstd gamma + beta), out = bf16(silu(v)) (SiLU with __expf) or v.

    The statistics are double sums of per-thread fp32 partials over up to GN_PIX_PER_BLOCK / (256 / (C / 8))
    pixels of one channel: the floor carries that partial-sum error into E[x^2] - mean^2."""
    xd = d64(x)
    N, P, C = xd.shape
    cpg = C // groups
    xg = xd.reshape(N, P, groups, cpg)
    cnt = P * cpg
    mean = xg.sum((1, 3), keepdim=True) / cnt
    ex2 = (xg * xg).sum((1, 3), keepdim=True) / cnt
    var = (ex2 - mean * mean).clamp_min(0)
    rstd = torch.rsqrt(var + eps)
    xh = (xg - mean) * rstd
    m_thr = -(-min(P, GN_PIX_PER_BLOCK) // (GN_THREADS // (C // 8)))     # pixels per thread partial
    e_mean = m_thr * U32 * xg.abs().mean((1, 3), keepdim=True)
    e_var = m_thr * U32 * ex2 + 2 * mean.abs() * e_mean
    f_xh = rstd * (e_mean + U32 * xg.abs()) + xh.abs() * (0.5 * e_var / (var + eps) + 2 * U32)
    ga = d64(gamma).reshape(groups, cpg)
    be = d64(beta).reshape(groups, cpg)
    pre = xh * ga + be
    f_pre = ga.abs() * f_xh + 4 * U32 * ((xh * ga).abs() + be.abs())
    v = bf16r(pre)
    if silu_on:
        s = silu(v)
        ds = (torch.sigmoid(v) * (1 + v * (1 - torch.sigmoid(v)))).abs()
        flip = ulp_bf16(v) * _near_tie(pre, f_pre)
        emu, floor, mth = bf16r(s), ds * (f_pre + flip) + (v.abs() + 8) * U32 * s.abs(), silu(pre)
    else:
        emu, floor, mth = v, f_pre, pre
    shp = (N, P, C)
    return emu.reshape(shp), floor.reshape(shp), mth.reshape(shp)


def softmax_rows_emu(s, scale):
    """softmax_rows: bf16(exp2((s - max) k) / sum), k = fp32(scale log2 e); s [rows, L]."""
    sd = d64(s)
    L = sd.shape[-1]
    k = f32(f32(scale) * f32(LOG2E))
    t = (sd - sd.amax(-1, keepdim=True)) * k
    e = torch.exp2(t)
    p = e / e.sum(-1, keepdim=True)
    # fp32 argument (|t| ulps), exp2f (2 ulps), the L-term sum (8 terms per vector, one vector per thread every 2048
    # columns, then a 13-level tree), the reciprocal and the product
    floor = p * U32 * (t.abs() * math.log(2) + 8 * -(-L // 2048) + 20)
    return bf16r(p), floor, torch.softmax(sd * scale, -1)
