"""fp64 references of the tensor-core ops and element-wise checks against them.

Every op has two references, both evaluated in float64 on the bf16 inputs:

  *math*       the operation itself (linear, conv, softmax attention and their gradients);
  *emulation*  the same arithmetic with bf16 rounding applied exactly where include/b2f.h documents it
               (epilogue chains, the QKV RMSNorm/RoPE chain, conv residual, the online softmax over 128-column
               K/V blocks, the bf16 P~ / dS~ operands of the attention backward).

A correct kernel differs from its emulation only by fp32 accumulation and by the occasional rounding flip where the
fp32 value lies within that accumulation error of a bf16 rounding boundary.  `ulp_diff` measures the difference in
bf16 ulps of the emulated value, with a floor for outputs that cancel to near zero:

    ulp_diff = |out - emu| / max(ulp_bf16(emu), floor)

`floor` is the fp32 accumulation allowance K * 2^-24 * absref (absref: the same op on |inputs|), widened by the first-
order effect of one flip at an intermediate rounding point.  The math reference backs a whole-tensor rel-L2 sanity gate.

Everything here is plain torch on whatever device the tensors live on; the CPU tests run it at small sizes.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

F64 = torch.float64
LOG2E = math.log2(math.e)
U32 = 2.0 ** -24        # fp32 unit roundoff

# epilogue ids (include/b2f.h)
EPI_BIAS, EPI_GELU_TANH, EPI_SILU, EPI_GATE_RESID, EPI_RESID, EPI_GELU_ERF = 0, 1, 2, 3, 4, 5
EPI_QUICK_GELU, EPI_DGELU, EPI_DSILU = 7, 8, 9

_K0, _K1 = 0.7978845608028654, 0.044715


# ---------------------------------------------------------------------------------------------------- rounding
def d64(t: torch.Tensor) -> torch.Tensor:
    return t.to(F64)


def bf16r(x: torch.Tensor) -> torch.Tensor:
    """Round to bf16 (round-to-nearest-even, through fp32 as the kernels round fp32 values) and return fp64."""
    return x.float().bfloat16().to(F64)


def ulp_bf16(x: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 numbers at |x|: 2^(e - 8) for |x| in [2^(e-1), 2^e); subnormal spacing at zero."""
    a = d64(x).abs()
    _, e = torch.frexp(a)
    ulp = torch.ldexp(torch.ones_like(a), (e - 8).clamp_min(-133))
    return torch.where(a == 0, torch.full_like(a, 2.0 ** -133), ulp)


def acc_floor(K: int, absref: torch.Tensor) -> torch.Tensor:
    """fp32 accumulation allowance of a K-term dot product whose absolute-value counterpart is `absref`."""
    return K * U32 * d64(absref)


def ulp_diff(out: torch.Tensor, emu: torch.Tensor, floor: torch.Tensor | float = 0.0) -> torch.Tensor:
    """|out - emu| in bf16 ulps of emu, never in units smaller than `floor`; NaN / inf in `out` count as inf."""
    o = d64(out)
    unit = torch.maximum(ulp_bf16(emu), torch.as_tensor(floor, dtype=F64, device=o.device))
    d = (o - emu).abs() / unit
    return torch.where(torch.isfinite(o), d, torch.full_like(d, math.inf))


def rel_l2(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = d64(a), d64(b)
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


# ---------------------------------------------------------------------------------------------------- checks
class Checker:
    """Collects the checks of one test case, prints every observed statistic (so margins can be read from the log)
    and raises once at the end with all failures, each naming the worst element and its margin."""

    def __init__(self, case: str):
        self.case = case
        self.fails: list[str] = []

    def _where(self, d: torch.Tensor, dims) -> str:
        idx = torch.unravel_index(torch.argmax(torch.nan_to_num(d, nan=math.inf)), d.shape)
        names = dims if dims is not None and len(dims) == d.dim() else [f"d{i}" for i in range(d.dim())]
        return "(" + ", ".join(f"{n}={int(i)}" for n, i in zip(names, idx)) + ")"

    def bf16(self, name, out, emu, floor=0.0, *, max_ulp, share_gt1, mean_ulp, math_ref=None, rel_l2_max=None,
             dims=None):
        """bf16 output against its emulation: max / share above 1 ulp / mean of ulp_diff, plus rel-L2 vs math."""
        d = ulp_diff(out, emu, floor)
        mx, share, mean = d.max().item(), (d > 1).double().mean().item(), d.mean().item()
        line = f"{self.case} {name}: max_ulp={mx:.3g} share>1ulp={share:.3g} mean_ulp={mean:.4g}"
        rl = None
        if math_ref is not None:
            rl = rel_l2(out, math_ref)
            line += f" relL2={rl:.3g}"
        print("KREF", line)
        where = self._where(d, dims)
        if not mx <= max_ulp:
            i = torch.unravel_index(torch.argmax(torch.nan_to_num(d, nan=math.inf)), d.shape)
            self.fails.append(f"{self.case} {name}: max ulp_diff {mx:.3g} > {max_ulp} at {where}: "
                              f"out={d64(out)[i].item():.6g} emu={emu[i].item():.6g}")
        if not share <= share_gt1:
            self.fails.append(f"{self.case} {name}: {share:.3g} of elements > 1 ulp (bound {share_gt1}); worst {where}")
        if not mean <= mean_ulp:
            self.fails.append(f"{self.case} {name}: mean ulp_diff {mean:.4g} > {mean_ulp}")
        if rel_l2_max is not None and not rl <= rel_l2_max:
            self.fails.append(f"{self.case} {name}: rel-L2 vs fp64 math {rl:.3g} > {rel_l2_max}")

    def within_floor(self, name, out, ref, floor, *, max_ratio, rel_l2_max=None, dims=None):
        """fp32 output (no bf16 rounding) against the math reference: |out - ref| <= max_ratio * floor."""
        r = (d64(out) - ref).abs() / d64(floor).clamp_min(1e-300)
        r = torch.where(torch.isfinite(d64(out)), r, torch.full_like(r, math.inf))
        mx = r.max().item()
        rl = rel_l2(out, ref)
        print("KREF", f"{self.case} {name}: max_err/floor={mx:.3g} relL2={rl:.3g}")
        if not mx <= max_ratio:
            self.fails.append(f"{self.case} {name}: error {mx:.3g} x the fp32 floor (bound {max_ratio}) at "
                              f"{self._where(r, dims)}")
        if rel_l2_max is not None and not rl <= rel_l2_max:
            self.fails.append(f"{self.case} {name}: rel-L2 vs fp64 math {rl:.3g} > {rel_l2_max}")

    def abs_err(self, name, out, ref, tol, dims=None):
        """per-element absolute error (the base-2 lse rows)."""
        d = (d64(out) - d64(ref)).abs()
        d = torch.where(torch.isfinite(d64(out)), d, torch.full_like(d, math.inf))
        mx = d.max().item()
        print("KREF", f"{self.case} {name}: max_abs={mx:.3g}")
        if not mx <= tol:
            self.fails.append(f"{self.case} {name}: abs error {mx:.3g} > {tol} at {self._where(d, dims)}")

    def equal(self, name, a, b):
        n = (a != b).sum().item()
        print("KREF", f"{self.case} {name}: mismatches={n}")
        if n:
            self.fails.append(f"{self.case} {name}: {n} elements differ")

    def finish(self):
        if self.fails:
            raise AssertionError("\n".join(self.fails))


# ---------------------------------------------------------------------------------------------------- activations
def gelu_tanh(x):
    # 0.5 x (1 + tanh(u)) = x * sigmoid(2u): the same function without the cancellation of 1 + tanh(u) for x << 0
    return x * torch.sigmoid(2.0 * _K0 * (x + _K1 * x ** 3))


def dgelu_tanh(x):
    t = torch.tanh(_K0 * (x + _K1 * x ** 3))
    return 0.5 * (1.0 + t) + 0.5 * x * (1.0 - t * t) * _K0 * (1.0 + 3.0 * _K1 * x * x)


def gelu_erf(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def dgelu_erf(x):
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


def silu(x):
    return x * torch.sigmoid(x)


def dsilu(x):
    s = torch.sigmoid(x)
    return s * (1.0 + x * (1.0 - s))


# ---------------------------------------------------------------------------------------------------- linear
def linear_math(x, w, b=None):
    """x [..., K] @ w[N, K]^T + b in fp64."""
    y = d64(x) @ d64(w).T
    return y if b is None else y + d64(b)


def linear_absref(x, w, b=None):
    y = d64(x).abs() @ d64(w).abs().T
    return y if b is None else y + d64(b).abs()


def epilogue_emu(acc, epi, *, floor0, resid=None, gate=None, aux=None):
    """Epilogue chain of include/b2f.h on fp64 pre-activations `acc` (= A.W^T + bias, or the dgrad product).

    Returns (emu, floor): emu is the bf16 output of the documented chain, floor the allowance for the fp32
    accumulation error `floor0` of acc carried through the chain plus one flip at each intermediate rounding."""
    if epi == EPI_BIAS:
        return bf16r(acc), floor0
    # the activations are evaluated in fp32: an absolute allowance of a few fp32 ulps of |x| (erff(x) == -1 in fp32
    # below x = -3.9, so 0.5 x (1 + erf) is exactly 0 there; the fp64 value is not)
    if epi in (EPI_GELU_TANH, EPI_GELU_ERF, EPI_SILU):
        f, df = {EPI_GELU_TANH: (gelu_tanh, dgelu_tanh), EPI_GELU_ERF: (gelu_erf, dgelu_erf),
                 EPI_SILU: (silu, dsilu)}[epi]
        x = bf16r(acc)
        return bf16r(f(x)), df(x).abs() * (ulp_bf16(x) + floor0) + 4 * U32 * x.abs()
    if epi == EPI_QUICK_GELU:
        x = bf16r(acc)
        t = bf16r(1.702 * x)
        s = bf16r(torch.sigmoid(t))
        ds = s * (1 - s)
        fl = (s + 1.702 * x.abs() * ds) * (ulp_bf16(x) + floor0) + x.abs() * (ds * ulp_bf16(t) + ulp_bf16(s))
        return bf16r(x * s), fl + 4 * U32 * x.abs()
    if epi == EPI_GATE_RESID:
        g = d64(gate)
        y = bf16r(acc)
        z = bf16r(g * y)
        return bf16r(d64(resid) + z), g.abs() * (ulp_bf16(y) + floor0) + ulp_bf16(z)
    if epi == EPI_RESID:
        y = bf16r(acc)
        return bf16r(d64(resid) + y), ulp_bf16(y) + floor0
    if epi in (EPI_DGELU, EPI_DSILU):
        u = d64(aux)
        dact = (dgelu_tanh if epi == EPI_DGELU else dsilu)(u)
        y = bf16r(acc)
        # act'(u) in fp32: 1 + tanh and 1 - t^2 cancel for large |u|
        return bf16r(y * dact), dact.abs() * (ulp_bf16(y) + floor0) + 8 * U32 * (1 + u * u) * y.abs()
    raise ValueError(f"epilogue {epi}")


def linear_emu(x, w, b=None, epi=EPI_BIAS, *, resid=None, gate=None):
    """(emu, floor, math) of b2f_gemm_bf16: out = epi(x @ w^T + b).  gate [B, N] broadcasts over rows."""
    acc = linear_math(x, w, b)
    floor0 = acc_floor(x.shape[-1], linear_absref(x, w, b))
    if gate is not None:
        gate = gate[:, None, :] if acc.dim() == 3 else gate
    emu, fl = epilogue_emu(acc, epi, floor0=floor0, resid=resid, gate=gate)
    return emu, fl, acc


def dgrad_emu(dy, w, epi=EPI_BIAS, aux=None):
    """(emu, floor, math) of b2f_gemm_dgrad: dx = epi(dy @ w) with w [K, N] as nn.Linear stores it."""
    acc = d64(dy) @ d64(w)
    floor0 = acc_floor(dy.shape[-1], d64(dy).abs() @ d64(w).abs())
    if epi == EPI_BIAS:
        return bf16r(acc), floor0, acc
    if epi == EPI_RESID:
        emu, fl = epilogue_emu(acc, EPI_RESID, floor0=floor0, resid=aux)
        return emu, fl, d64(aux) + acc
    emu, fl = epilogue_emu(acc, epi, floor0=floor0, aux=aux)
    dact = (dgelu_tanh if epi == EPI_DGELU else dsilu)(d64(aux))
    return emu, fl, acc * dact


def wgrad_math(dy, x):
    """(math, floor) of b2f_gemm_wgrad: dW = sum over batch and rows of dy^T x, fp32 output."""
    ref = torch.einsum("brm,brn->mn", d64(dy), d64(x))
    absref = torch.einsum("brm,brn->mn", d64(dy).abs(), d64(x).abs())
    return ref, acc_floor(dy.shape[0] * dy.shape[1], absref)


def _rot_pairs(z):
    z2 = z.unflatten(-1, (-1, 2))
    return torch.stack([-z2[..., 1], z2[..., 0]], -1).flatten(-2)


def qkv_norm_rope_emu(x, w, b, nw_q, nw_k, cos, sin, *, rope_row0=0, eps=1e-6, n_extra=0, epi_extra=EPI_BIAS):
    """(emu, floor, math) of b2f_gemm_qkv_norm_rope over all 3d + n_extra columns.

    Per 128-column head of Q and K (include/b2f.h, gemm.cu epilogue_head_norm_rope):
      x = bf16(acc + bias); y = bf16(x * rsqrt(mean(x^2) + eps)); z = bf16(y * w); out = bf16(z*cos + rot(z)*sin)
    V: bf16(acc + bias); extra columns: epilogue epi_extra.  Token `row` uses table row rope_row0 + row."""
    acc = linear_math(x, w, b)
    floor0 = acc_floor(x.shape[-1], linear_absref(x, w, b))
    N = acc.shape[-1]
    d = (N - n_extra) // 3
    M = acc.shape[-2]
    c = d64(cos[rope_row0:rope_row0 + M])
    s = d64(sin[rope_row0:rope_row0 + M])
    emu = torch.empty_like(acc)
    fl = torch.empty_like(acc)
    mth = torch.empty_like(acc)
    for blk, nw in ((0, nw_q), (1, nw_k)):
        cols = slice(blk * d, (blk + 1) * d)
        a = acc[..., cols].unflatten(-1, (-1, 128))
        f0 = floor0[..., cols].unflatten(-1, (-1, 128))
        wv = d64(nw)
        cc, ss = c[:, None, :], s[:, None, :]
        # math: fp64 throughout
        r_m = torch.rsqrt(a.pow(2).mean(-1, keepdim=True) + eps)
        zm = a * r_m * wv
        mth[..., cols] = (zm * cc + _rot_pairs(zm) * ss).flatten(-2)
        # emulation
        xb = bf16r(a)
        r = torch.rsqrt(xb.pow(2).mean(-1, keepdim=True) + eps)
        y = bf16r(xb * r)
        z = bf16r(y * wv)
        emu[..., cols] = bf16r(z * cc + _rot_pairs(z) * ss).flatten(-2)
        sl = wv.abs() * (r * (ulp_bf16(xb) + f0) + ulp_bf16(y)) + ulp_bf16(z)
        slp = torch.maximum(sl, _rot_pairs(sl).abs())
        fl[..., cols] = (slp * (cc.abs() + ss.abs())).flatten(-2)
    v = slice(2 * d, 3 * d)
    emu[..., v], fl[..., v] = epilogue_emu(acc[..., v], EPI_BIAS, floor0=floor0[..., v])
    mth[..., v] = acc[..., v]
    if n_extra:
        e = slice(3 * d, N)
        emu[..., e], fl[..., e] = epilogue_emu(acc[..., e], epi_extra, floor0=floor0[..., e])
        mth[..., e] = {EPI_BIAS: lambda t: t, EPI_GELU_TANH: gelu_tanh, EPI_SILU: silu}[epi_extra](acc[..., e])
    return emu, fl, mth


# ---------------------------------------------------------------------------------------------------- conv 3x3
def conv_math(x_nhwc, w_ohwi, b=None, stride=1):
    """fp64 3x3 conv, NHWC in / out.  stride 1: padding 1; stride 2: Downsample2D (pad right/bottom by one)."""
    x = d64(x_nhwc).permute(0, 3, 1, 2)
    w = d64(w_ohwi).permute(0, 3, 1, 2)
    bb = None if b is None else d64(b)
    if stride == 1:
        y = F.conv2d(x, w, bb, padding=1)
    else:
        y = F.conv2d(F.pad(x, (0, 1, 0, 1)), w, bb, stride=2)
    return y.permute(0, 2, 3, 1)


def conv_emu(x_nhwc, w_ohwi, b=None, stride=1, resid=None):
    """(emu, floor, math) of b2f_conv3x3 with NHWC output: bf16(conv + bias), then bf16(resid + that)."""
    acc = conv_math(x_nhwc, w_ohwi, b, stride)
    absref = conv_math(d64(x_nhwc).abs(), d64(w_ohwi).abs(), None if b is None else d64(b).abs(), stride)
    floor0 = acc_floor(9 * x_nhwc.shape[-1], absref)
    if resid is None:
        emu, fl = epilogue_emu(acc, EPI_BIAS, floor0=floor0)
        return emu, fl, acc
    emu, fl = epilogue_emu(acc, EPI_RESID, floor0=floor0, resid=resid)
    return emu, fl, d64(resid) + acc


def u8_rule(img_bf16: torch.Tensor) -> torch.Tensor:
    """VaeImageProcessor.postprocess on a bf16 image, in fp32: round(clamp(x/2 + 0.5, 0, 1) * 255), half to even."""
    u = torch.clamp(img_bf16.float() / 2.0 + 0.5, 0.0, 1.0)
    return torch.round(u * 255.0).to(torch.uint8)


# ---------------------------------------------------------------------------------------------------- attention
def _heads(t, H):
    """[B, S, Hx, D] -> [B, H, S, D] fp64 with GQA expansion (query head h reads kv head h // (H / Hx))."""
    t = d64(t).permute(0, 2, 1, 3)
    return t.repeat_interleave(H // t.shape[1], dim=1)


def _scores(q, k, scale, bias, causal):
    """Scaled scores in natural-log units [B, H, Sq, Skv] with masked entries at -inf."""
    H = q.shape[2]
    s = _heads(q, H) @ _heads(k, H).transpose(-1, -2) * scale
    if bias is not None:
        s = s + d64(bias)[None]
    if causal:
        Sq, Skv = s.shape[-2:]
        mask = torch.ones(Sq, Skv, dtype=torch.bool, device=s.device).tril()
        s = s.masked_fill(~mask, -math.inf)
    return s


def max_outer(a, x, chunk=32):
    """out[..., i, c] = max_j a[..., i, j] * x[..., j, c] for nonnegative a, x (the largest single term of a @ x)."""
    out = torch.zeros(*a.shape[:-1], x.shape[-1], dtype=F64, device=a.device)
    for j0 in range(0, a.shape[-1], chunk):
        prod = a[..., j0:j0 + chunk, None] * x[..., None, j0:j0 + chunk, :]
        out = torch.maximum(out, prod.amax(-2))
    return out


def attention_math(q, k, v, *, scale=None, causal=False, bias=None):
    """(out [B, Sq, H*D], lse2 [B, H, Sq]) of softmax(q k^T * scale + bias) v in fp64; lse2 in base 2."""
    B, Sq, H, D = q.shape
    scale = D ** -0.5 if scale is None else scale
    s = _scores(q, k, scale, bias, causal)
    p = torch.softmax(s, -1)
    o = p @ _heads(v, H)
    return o.permute(0, 2, 1, 3).reshape(B, Sq, H * D), torch.logsumexp(s, -1) * LOG2E


def attention_emu(q, k, v, *, scale=None, causal=False, bias=None, block=128):
    """(out, lse2, floor) of the online softmax of attention.cu, in fp64 with its bf16 rounding points.

    K/V are streamed in `block`-column blocks.  Per block: m = running max of the base-2 scores t = s * c
    (c = scale * log2 e; with a bias, t = (s * scale + bias) * log2 e), p = 2^(t - m), P~ = bf16(p);
    l = l * 2^(m_old - m) + sum(p) (unrounded p), O = O * 2^(m_old - m) + P~ V.  out = bf16(O / l), lse2 = m + log2 l."""
    B, Sq, H, D = q.shape
    Skv = k.shape[1]
    scale = D ** -0.5 if scale is None else scale
    t = _scores(q, k, scale, bias, causal) * LOG2E
    vh = _heads(v, H)
    m = torch.full((B, H, Sq, 1), -math.inf, dtype=F64, device=t.device)
    l = torch.zeros_like(m)
    o = torch.zeros(B, H, Sq, D, dtype=F64, device=t.device)
    for j0 in range(0, Skv, block):
        tj = t[..., j0:j0 + block]
        m_new = torch.maximum(m, tj.amax(-1, keepdim=True))
        alpha = torch.where(m == -math.inf, torch.zeros_like(m), torch.exp2(m - m_new))
        p = torch.exp2(tj - torch.where(m_new == -math.inf, torch.zeros_like(m_new), m_new))
        l = l * alpha + p.sum(-1, keepdim=True)
        o = o * alpha + bf16r(p) @ vh[..., j0:j0 + block, :]
        m = m_new
    out = bf16r(o / l)
    # floor: Skv-term fp32 accumulation of the probability-weighted |V|, plus one flip of the largest P~ term: the
    # kernel's p carries the fp32 error of its scores and of ex2.approx, so where p lies that close to a bf16 tie its
    # P~ rounds the other way (a change of up to 2^-7 P_j |v_j| in every output of that row)
    P = torch.exp2(t - m) / l
    floor = acc_floor(Skv, P @ vh.abs()) + 2.0 ** -7 * max_outer(P, vh.abs())
    perm = lambda a: a.permute(0, 2, 1, 3).reshape(B, Sq, H * D)
    return perm(out), (m + torch.log2(l)).squeeze(-1), perm(floor)


def attention_bwd_math(q, k, v, dout, *, scale=None):
    """(dq, dk, dv) [B, S, H, D] of softmax attention by fp64 autograd."""
    B, S, H, D = q.shape
    scale = D ** -0.5 if scale is None else scale
    qf, kf, vf = (d64(t).detach().requires_grad_(True) for t in (q, k, v))
    s = torch.einsum("bqhd,bkhd->bhqk", qf, kf) * scale
    o = torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, -1), vf).reshape(B, S, H * D)
    o.backward(d64(dout))
    return qf.grad, kf.grad, vf.grad


def attention_bwd_emu(q, k, v, o, dout, lse2, *, scale=None):
    """(dq, dk, dv, floors) of attention_bwd.cu in fp64 with its rounding points, given the forward's own o and lse2:

      P = 2^(s*c - lse2), P~ = bf16(P);  dV = bf16(P~^T dO)
      delta = rowsum(dO * o);  dS = P * (dO V^T - delta), dS~ = bf16(dS)
      dK = bf16(scale * dS~^T Q);  dQ = bf16(scale * dS~ K)"""
    B, S, H, D = q.shape
    scale = D ** -0.5 if scale is None else scale
    c = scale * LOG2E
    qh, kh, vh = _heads(q, H), _heads(k, H), _heads(v, H)
    doh = d64(dout).reshape(B, S, H, D).permute(0, 2, 1, 3)
    oh = d64(o).reshape(B, S, H, D).permute(0, 2, 1, 3)
    lse = d64(lse2[..., :S])[..., None]
    P = torch.exp2(qh @ kh.transpose(-1, -2) * c - lse)
    Pb = bf16r(P)
    delta = (doh * oh).sum(-1, keepdim=True)
    dP = doh @ vh.transpose(-1, -2)
    dS = P * (dP - delta)
    dSb = bf16r(dS)
    dv = bf16r(Pb.transpose(-1, -2) @ doh)
    dk = bf16r(scale * (dSb.transpose(-1, -2) @ qh))
    dq = bf16r(scale * (dSb @ kh))
    dS_abs = P * (doh.abs() @ vh.abs().transpose(-1, -2) + delta.abs())
    Kt = S + D
    # plus one flip of the largest bf16 operand term: P~ (2^-7 P), and dS~, whose fp32 value also carries the
    # accumulation error of dP - delta
    es = 2.0 ** -7 * dS.abs() + 8 * Kt * U32 * dS_abs
    fl_dv = acc_floor(Kt, Pb.transpose(-1, -2) @ doh.abs()) + 2.0 ** -7 * max_outer(P.transpose(-1, -2), doh.abs())
    fl_dk = acc_floor(Kt, scale * (dS_abs.transpose(-1, -2) @ qh.abs())) + scale * max_outer(es.transpose(-1, -2),
                                                                                               qh.abs())
    fl_dq = acc_floor(Kt, scale * (dS_abs @ kh.abs())) + scale * max_outer(es, kh.abs())
    back = lambda a: a.permute(0, 2, 1, 3)
    return back(dq), back(dk), back(dv), (back(fl_dq), back(fl_dk), back(fl_dv))
