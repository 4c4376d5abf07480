"""Edge sweeps of the sm_90a tensor-core kernels, element by element, against the fp64 references of kernel_ref.py.

The shapes aim at the edges of the Hopper kernels:
  GEMM / conv (gemm_sm90.cuh)  128 x 128 x 64 tiles, two 64-row consumer halves, a 4-stage TMA ring (phase flips every
                               4 k-blocks), epilogue in 32-column chunks of 8-column groups, n-block panels of 16;
  attention forward            128 query rows (2 x 64), 128-row K/V blocks through 2 slots (phase flips at block 3),
                               tail masking only where kv0 + 128 > Skv or causal;
  attention backward           64-row streamed blocks in a 2-stage ring, lse = +inf / delta = 0 in the padding rows;
  conv                         8 x 16 spatial tiles, 9 * Cin / 64 k-blocks, a strided tensor map for stride 2.

Every check prints (max ulp, share > 1 ulp, mean ulp) of the output against its rounding-faithful emulation, and the
rel-L2 against the exact fp64 op.  Thresholds below were set from H100 runs of the unmodified kernels; each sits between
what the correct kernels produce (worst on an H100 80GB HBM3: max 1.01 ulp, share > 1 ulp 6e-5, mean 0.004 ulp) and
what deliberately broken kernels (one dropped bias group, a missing k16 MMA, an off-by-one mask, a missing rescale of
the softmax sum, a wrong RoPE row, a skipped residual column, a dropped fp32 accumulation) produce.
"""
import math

import pytest
import torch

import kernel_ref as R

pytestmark = pytest.mark.gpu

# (max ulp, share of elements above 1 ulp, mean ulp) for bf16 outputs against their emulation
TH_GEMM = dict(max_ulp=2, share_gt1=1e-3, mean_ulp=0.1)
TH_CONV = dict(max_ulp=2, share_gt1=1e-3, mean_ulp=0.1)
TH_ATTN = dict(max_ulp=2, share_gt1=1e-3, mean_ulp=0.05)
TH_BWD = dict(max_ulp=2, share_gt1=1e-3, mean_ulp=0.05)
LSE_TOL = 2e-4          # absolute, base 2
BHSD = ("b", "token", "head", "col")


def _g(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _bf(*shape, g, scale=1.0, shift=0.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale + shift).bfloat16()


# ---------------------------------------------------------------------------------------------------- GEMM forward
@pytest.mark.parametrize("M,N,K", [
    (1, 8, 8),          # one row, one column group, one partial k-block
    (63, 24, 56),       # inside one consumer half
    (64, 72, 64),       # exactly one half, one full k-block
    (65, 2056, 256),    # second half starts; 17 n-blocks (panel edge at 16/17); exactly one turn of the ring
    (129, 2176, 320),   # second m-block; 17 full n-blocks; the ring wraps (5 k-blocks)
    (64, 136, 520),     # 9 k-blocks with an 8-wide tail: the phase flips twice
    (129, 8, 64),
])
def test_gemm_edges(M, N, K):
    from gpt_image_edit_b200 import ops

    g = _g(M * 7 + N + K)
    x, w, b = _bf(M, K, g=g), _bf(N, K, g=g, scale=K ** -0.5), _bf(N, g=g, scale=0.5)
    out = ops.linear(x, w, b)
    emu, floor, acc = R.linear_emu(x, w, b)
    c = R.Checker(f"gemm M{M} N{N} K{K}")
    c.bf16("out", out, emu, floor, math_ref=acc, rel_l2_max=4e-3, dims=("row", "col"), **TH_GEMM)
    c.finish()


def test_gemm_batched_pitched_views():
    """B = 3, ragged M, A and out as slices of wider buffers: row pitch != width, batch stride != M * ld."""
    from gpt_image_edit_b200 import ops

    g = _g(31)
    B, M, N, K = 3, 65, 136, 80
    xa = _bf(B, 100, 96, g=g)
    x = xa[:, 10:10 + M, :K]
    w, b = _bf(N, K, g=g, scale=K ** -0.5), _bf(N, g=g, scale=0.5)
    oa = _bf(B, 90, 200, g=g)
    before = oa.clone()
    out = oa[:, 5:5 + M, 16:16 + N]
    ops.linear(x, w, b, out=out)
    emu, floor, acc = R.linear_emu(x, w, b)
    c = R.Checker("gemm batched B3 M65")
    c.bf16("out", out, emu, floor, math_ref=acc, rel_l2_max=4e-3, dims=("b", "row", "col"), **TH_GEMM)
    mask = torch.ones_like(oa, dtype=torch.bool)
    mask[:, 5:5 + M, 16:16 + N] = False
    c.equal("outside the view", oa[mask], before[mask])
    c.finish()


@pytest.mark.parametrize("epi", [R.EPI_BIAS, R.EPI_GELU_TANH, R.EPI_GELU_ERF, R.EPI_SILU, R.EPI_QUICK_GELU,
                                 R.EPI_GATE_RESID, R.EPI_RESID])
def test_gemm_epilogues_on_tails(epi):
    """Every forward epilogue on M / N / K tails, batched; the residual epilogues run in place (resid aliases out)."""
    from gpt_image_edit_b200 import ops

    g = _g(40 + epi)
    B, M, N, K = 2, 65, 136, 72
    x, w, b = _bf(B, M, K, g=g), _bf(N, K, g=g, scale=K ** -0.5 * 2), _bf(N, g=g, scale=0.5)
    resid, gate = _bf(B, M, N, g=g), _bf(B, N, g=g)
    if epi in (R.EPI_GATE_RESID, R.EPI_RESID):
        out = resid.clone()
        ops.linear(x, w, b, epilogue=epi, resid=out, gate=gate if epi == R.EPI_GATE_RESID else None, out=out)
    else:
        out = ops.linear(x, w, b, epilogue=epi)
    emu, floor, acc = R.linear_emu(x, w, b, epi, resid=resid, gate=gate)
    c = R.Checker(f"gemm epi{epi} B2 M65 N136 K72")
    c.bf16("out", out, emu, floor, dims=("b", "row", "col"), **TH_GEMM)
    c.finish()


def _rope(S, g):
    ang = torch.rand(S, 64, device="cuda", generator=g) * 6.28
    return torch.cos(ang).repeat_interleave(2, 1).contiguous(), torch.sin(ang).repeat_interleave(2, 1).contiguous()


@pytest.mark.parametrize("B,M,H,K,row0,extra", [
    (2, 65, 2, 320, 40, True),     # single-stream block: [Q|K|V|proj_mlp] in one launch, MLP GELU'd into [attn|mlp]
    (1, 129, 3, 64, 0, False),     # double-stream block QKV
])
def test_gemm_qkv_norm_rope(B, M, H, K, row0, extra):
    from gpt_image_edit_b200 import ops

    g = _g(50 + M)
    d = H * 128
    n_extra = 4 * d if extra else 0
    x = _bf(B, M, K, g=g)
    w, b = _bf(3 * d + n_extra, K, g=g, scale=K ** -0.5), _bf(3 * d + n_extra, g=g, scale=0.5)
    nq, nk = _bf(128, g=g, scale=0.1, shift=1.0), _bf(128, g=g, scale=0.1, shift=1.0)
    cos, sin = _rope(row0 + M + 7, g)
    cat = before = out_extra = None
    if extra:
        cat = _bf(B, M, d + n_extra, g=g)
        before = cat.clone()
        out_extra = cat[:, :, d:]
    out = ops.linear_qkv_norm_rope(x, w, b, nq, nk, cos, sin, rope_row0=row0, out_extra=out_extra,
                                   epi_extra=ops.EPI_GELU_TANH)
    emu, floor, mth = R.qkv_norm_rope_emu(x, w, b, nq, nk, cos, sin, rope_row0=row0, n_extra=n_extra,
                                          epi_extra=R.EPI_GELU_TANH)
    c = R.Checker(f"qkv_norm_rope B{B} M{M} H{H} row0={row0} extra={n_extra}")
    dims = ("b", "row", "col")
    c.bf16("Q", out[..., :d], emu[..., :d], floor[..., :d], math_ref=mth[..., :d], rel_l2_max=8e-3, dims=dims,
           **TH_GEMM)
    c.bf16("K", out[..., d:2 * d], emu[..., d:2 * d], floor[..., d:2 * d], math_ref=mth[..., d:2 * d],
           rel_l2_max=8e-3, dims=dims, **TH_GEMM)
    c.bf16("V", out[..., 2 * d:], emu[..., 2 * d:3 * d], floor[..., 2 * d:3 * d], dims=dims, **TH_GEMM)
    if extra:
        c.bf16("mlp", out_extra, emu[..., 3 * d:], floor[..., 3 * d:], math_ref=mth[..., 3 * d:], rel_l2_max=6e-3,
               dims=dims, **TH_GEMM)
        c.equal("attn columns of [attn|mlp]", cat[:, :, :d], before[:, :, :d])
    c.finish()


# ---------------------------------------------------------------------------------------------------- dgrad / wgrad
@pytest.mark.parametrize("B,M,N,K", [
    (1, 1, 8, 8),
    (1, 63, 24, 56),
    (1, 129, 2056, 320),    # 17 n-blocks, ring wrap
    (3, 65, 136, 520),      # batched ragged rows, 9 k-blocks with a tail
    (1, 64, 2176, 256),
])
def test_dgrad_edges(B, M, N, K):
    from gpt_image_edit_b200 import train_ops as T

    g = _g(60 + M + N)
    dy, w = _bf(B, M, K, g=g), _bf(K, N, g=g, scale=K ** -0.5)
    out = T.linear_dgrad(dy, w)
    emu, floor, mth = R.dgrad_emu(dy, w)
    c = R.Checker(f"dgrad B{B} M{M} N{N} K{K}")
    c.bf16("dx", out, emu, floor, math_ref=mth, rel_l2_max=4e-3, dims=("b", "row", "col"), **TH_GEMM)
    c.finish()


@pytest.mark.parametrize("epi", [R.EPI_BIAS, R.EPI_DGELU, R.EPI_DSILU, R.EPI_RESID])
def test_dgrad_epilogues_on_tails(epi):
    from gpt_image_edit_b200 import train_ops as T

    g = _g(70 + epi)
    B, M, N, K = 2, 65, 136, 72
    dy, w = _bf(B, M, K, g=g), _bf(K, N, g=g, scale=K ** -0.5)
    aux = _bf(B, M, N, g=g, scale=2.0)
    out = T.linear_dgrad(dy, w, epilogue=epi, aux=None if epi == R.EPI_BIAS else aux)
    emu, floor, mth = R.dgrad_emu(dy, w, epi, aux=aux)
    c = R.Checker(f"dgrad epi{epi} B2 M65 N136 K72")
    c.bf16("dx", out, emu, floor, math_ref=mth, rel_l2_max=6e-3, dims=("b", "row", "col"), **TH_GEMM)
    c.finish()


@pytest.mark.parametrize("B,rows,M,N", [
    (3, 1, 64, 136),        # one token per batch item: every k-block is a 1-row tail
    (3, 63, 136, 2056),     # 17 n-blocks
    (3, 65, 2176, 72),      # two k-blocks per batch item, the second a 1-row tail
])
def test_wgrad_edges(B, rows, M, N):
    from gpt_image_edit_b200 import train_ops as T

    g = _g(80 + rows)
    dy, x = _bf(B, rows, M, g=g), _bf(B, rows, N, g=g)
    ref, floor = R.wgrad_math(dy, x)
    dw = T.linear_wgrad(dy, x)
    prior = torch.randn(M, N, device="cuda", generator=g)
    dw2 = T.linear_wgrad(dy, x, out=prior.clone(), accumulate=True)
    c = R.Checker(f"wgrad B{B} rows{rows} M{M} N{N}")
    c.within_floor("dw", dw, ref, floor, max_ratio=1.0, rel_l2_max=1e-5, dims=("m", "n"))
    c.within_floor("dw accumulate", dw2, ref + prior.double(), floor + R.U32 * (prior.double().abs() + ref.abs()),
                   max_ratio=1.0, dims=("m", "n"))
    c.finish()


# ---------------------------------------------------------------------------------------------------- attention forward
def _attn_check(c, out, q, k, v, *, scale=None, causal=False, bias=None, lse=None):
    B, Sq, H, _ = q.shape
    emu, lse_emu, floor = R.attention_emu(q, k, v, scale=scale, causal=causal, bias=bias)
    mth, lse_m = R.attention_math(q, k, v, scale=scale, causal=causal, bias=bias)
    shp = (B, Sq, H, 128)
    c.bf16("o", out.view(shp), emu.view(shp), floor.view(shp), math_ref=mth.view(shp), rel_l2_max=8e-3, dims=BHSD,
           **TH_ATTN)
    if lse is not None:
        c.abs_err("lse2 vs emulation", lse[..., :Sq], lse_emu, LSE_TOL, dims=("b", "head", "token"))
        c.abs_err("lse2 vs math", lse[..., :Sq], lse_m, 2 * LSE_TOL, dims=("b", "head", "token"))


@pytest.mark.parametrize("B,H,Hkv,Sq,Skv,causal", [
    (1, 1, 1, 1, 1, False),
    (1, 2, 2, 63, 65, False),
    (1, 2, 1, 64, 127, False),
    (2, 2, 2, 65, 128, False),
    (1, 1, 1, 127, 129, False),     # second K/V block with one valid key
    (1, 7, 1, 128, 256, False),     # 7 query heads per K/V head
    (1, 2, 2, 129, 257, False),     # third K/V block reuses slot 0 (phase flip)
    (1, 2, 2, 256, 385, False),
    (2, 3, 3, 385, 64, False),
    (1, 2, 2, 1, 1, True),
    (1, 2, 2, 65, 65, True),
    (1, 4, 2, 129, 129, True),
    (2, 2, 2, 257, 257, True),
])
def test_attention_edges(B, H, Hkv, Sq, Skv, causal):
    from gpt_image_edit_b200 import ops, train_ops as T

    g = _g(Sq * 3 + Skv + H)
    q, k, v = _bf(B, Sq, H, 128, g=g), _bf(B, Skv, Hkv, 128, g=g), _bf(B, Skv, Hkv, 128, g=g)
    out = ops.attention(q, k, v, causal=causal)
    c = R.Checker(f"attn B{B} H{H}/{Hkv} Sq{Sq} Skv{Skv} causal={int(causal)}")
    lse = None
    if not causal:
        out2, lse = T.attention_fwd_lse(q, k, v)
        c.equal("attention_fwd_lse output", out2, out)
    _attn_check(c, out, q, k, v, causal=causal, lse=lse)
    c.finish()


@pytest.mark.parametrize("Skv", [129, 257, 1000])
def test_attention_decode_from_cache(Skv):
    """Sq = 1 against K/V slices of a longer cache buffer (the Qwen2.5-VL decode step), 28 query / 4 K/V heads."""
    from gpt_image_edit_b200 import ops

    g = _g(90 + Skv)
    lo, H, Hkv = 5, 28, 4
    cache = _bf(2, 1, 1100, Hkv, 128, g=g)
    k, v = cache[0, :, lo:lo + Skv], cache[1, :, lo:lo + Skv]
    q = _bf(1, 1, H, 128, g=g)
    out = ops.attention(q, k, v)
    c = R.Checker(f"decode Skv{Skv}")
    _attn_check(c, out, q, k, v)
    c.finish()


def test_attention_vit_windows():
    """Vision-tower layout: 16 windows of 64 tokens, head dim 80 zero-padded to 128, scale 80^-0.5, Q/K/V as column
    slices of one [tokens, 3 * H * 128] projection buffer."""
    from gpt_image_edit_b200 import ops

    g = _g(95)
    W, L, H = 16, 64, 4
    rows = torch.zeros(W * L, 3, H, 128, device="cuda", dtype=torch.bfloat16)
    rows[..., :80] = _bf(W * L, 3, H, 80, g=g)
    rows = rows.view(W * L, 3 * H * 128)
    q = rows[:, :H * 128].unflatten(1, (H, 128)).unflatten(0, (W, L))
    k = rows[:, H * 128:2 * H * 128].unflatten(1, (H, 128)).unflatten(0, (W, L))
    v = rows[:, 2 * H * 128:].unflatten(1, (H, 128)).unflatten(0, (W, L))
    out = ops.attention(q, k, v, scale=80 ** -0.5)
    c = R.Checker("vit windows 16x64 d80")
    _attn_check(c, out, q, k, v, scale=80 ** -0.5)
    c.finish()


@pytest.mark.parametrize("S", [1, 129, 257, 512])
def test_attention_bias_kernel(S):
    """T5 path: scale 1, additive bf16 bias shared by the batch, bias rows pitched wider than Skv."""
    from gpt_image_edit_b200 import ops

    g = _g(100 + S)
    B, H = 2, 2
    q, k, v = _bf(B, S, H, 128, g=g, scale=0.3), _bf(B, S, H, 128, g=g, scale=0.3), _bf(B, S, H, 128, g=g)
    big = _bf(H, S, S + 24, g=g, scale=2.0)
    bias = big[:, :, :S]
    out = ops.attention(q, k, v, scale=1.0, bias=bias)
    c = R.Checker(f"attn bias S{S}")
    _attn_check(c, out, q, k, v, scale=1.0, bias=bias)
    c.finish()


# ---------------------------------------------------------------------------------------------------- attention backward
def _bwd_check(c, q, k, v, do, *, scale=None, dq=None, dk=None, dv=None, dq_rel_l2=1.2e-2):
    from gpt_image_edit_b200 import train_ops as T

    o, lse = T.attention_fwd_lse(q, k, v, scale=scale)
    dq, dk, dv = T.attention_bwd(q, k, v, o, do, lse, dq=dq, dk=dk, dv=dv, scale=scale)
    eq, ek, ev, (fq, fk, fv) = R.attention_bwd_emu(q, k, v, o, do, lse, scale=scale)
    mq, mk, mv = R.attention_bwd_math(q, k, v, do, scale=scale)
    for name, out, emu, fl, mth, rl in (("dv", dv, ev, fv, mv, 1.2e-2), ("dk", dk, ek, fk, mk, 1.2e-2),
                                        ("dq", dq, eq, fq, mq, dq_rel_l2)):
        c.bf16(name, out, emu, fl, math_ref=mth, rel_l2_max=rl, dims=BHSD, **TH_BWD)
    return dq, dk, dv


@pytest.mark.parametrize("B,S,H", [
    (1, 1, 1), (2, 63, 1), (1, 64, 2), (2, 65, 1), (1, 127, 1), (2, 129, 2), (1, 192, 1), (1, 193, 2),
    (1, 65, 24),
])
def test_attention_bwd_edges(B, S, H):
    g = _g(110 + S + H)
    q, k, v = (_bf(B, S, H, 128, g=g) for _ in range(3))
    do = _bf(B, S, H * 128, g=g)
    c = R.Checker(f"attn bwd B{B} S{S} H{H}")
    _bwd_check(c, q, k, v, do)
    c.finish()


def test_attention_bwd_scale_and_very_negative_lse():
    """Every score of every row far below zero (lse2 < -128, so 2^-lse2 overflows fp32): a streamed padding column
    that escaped its mask would turn dq into NaN.  Non-default scale.  All keys point the same way, so dq = sum dS k
    cancels to the spread of k around its mean: the bf16 dS~ operand alone puts the exact fp64 dq ~3e-2 away (the
    rounding-faithful emulation is the tight check here)."""
    g = _g(120)
    B, S, H = 1, 65, 2
    k = _bf(B, S, H, 128, g=g, scale=0.1, shift=1.0)
    q = _bf(B, S, H, 128, g=g, scale=0.5, shift=-8.0)
    v = _bf(B, S, H, 128, g=g)
    do = _bf(B, S, H * 128, g=g)
    scale = 0.1
    c = R.Checker("attn bwd lse<-128 scale0.1")
    _bwd_check(c, q, k, v, do, scale=scale, dq_rel_l2=5e-2)
    c.finish()


def test_attention_bwd_training_layout():
    """flux_train.cu layout: q / k from a [B, S, 3d] buffer, v from a [B, S, 7d] buffer, dO [B, S, d], and dq / dk / dv
    written into a [B, S, 7d] gradient buffer whose other columns must not change."""
    g = _g(130)
    B, S, H = 2, 193, 2
    d = H * 128
    qk = _bf(B, S, 3 * d, g=g)
    vb = _bf(B, S, 7 * d, g=g)
    q, k = qk[:, :, :d].unflatten(-1, (H, 128)), qk[:, :, d:2 * d].unflatten(-1, (H, 128))
    v = vb[:, :, 2 * d:3 * d].unflatten(-1, (H, 128))
    do = _bf(B, S, d, g=g)
    gb = _bf(B, S, 7 * d, g=g)
    before = gb.clone()
    dq, dk, dv = (gb[:, :, i * d:(i + 1) * d].unflatten(-1, (H, 128)) for i in range(3))
    c = R.Checker("attn bwd training layout")
    _bwd_check(c, q, k, v, do, dq=dq, dk=dk, dv=dv)
    c.equal("other gradient columns", gb[:, :, 3 * d:], before[:, :, 3 * d:])
    c.finish()


# ---------------------------------------------------------------------------------------------------- conv 3x3
def _conv(x, w, b, out, resid, N, H, W, Cin, Cout, stride, mode):
    from gpt_image_edit_b200 import _lib as L

    L.check(L.lib.b2f_conv3x3(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(out), L.ptr(resid), N, H, W, Cin, Cout, stride, mode,
                              L.stream_ptr()), "b2f_conv3x3")


@pytest.mark.parametrize("N,H,W,Cin,Cout,stride", [
    (2, 5, 7, 64, 8, 1),         # one partial tile per image, one column group
    (1, 9, 17, 64, 136, 1),      # one-pixel corner tile (y = 8, x = 16); second n-block of 8 channels
    (3, 17, 33, 128, 128, 2),    # stride-2 tensor map, N = 3
    (1, 16, 16, 512, 512, 1),    # 72 k-blocks: the ring turns 18 times
])
def test_conv_edges(N, H, W, Cin, Cout, stride):
    g = _g(140 + H * W + Cout)
    x = _bf(N, H, W, Cin, g=g)
    w = _bf(Cout, 3, 3, Cin, g=g, scale=(9 * Cin) ** -0.5)
    b = _bf(Cout, g=g, scale=0.5)
    Ho, Wo = (H, W) if stride == 1 else ((H + 1 - 3) // 2 + 1, (W + 1 - 3) // 2 + 1)
    out = torch.empty(N, Ho, Wo, Cout, device="cuda", dtype=torch.bfloat16)
    _conv(x, w, b, out, None, N, H, W, Cin, Cout, stride, 0)
    resid = _bf(N, Ho, Wo, Cout, g=g)
    out_r = resid.clone()
    _conv(x, w, b, out_r, out_r, N, H, W, Cin, Cout, stride, 0)         # residual aliases out
    emu, floor, mth = R.conv_emu(x, w, b, stride)
    emu_r, floor_r, mth_r = R.conv_emu(x, w, b, stride, resid=resid)
    c = R.Checker(f"conv N{N} {H}x{W} {Cin}->{Cout} s{stride}")
    dims = ("n", "y", "x", "c")
    c.bf16("out", out, emu, floor, math_ref=mth, rel_l2_max=4e-3, dims=dims, **TH_CONV)
    c.bf16("out + resid", out_r, emu_r, floor_r, math_ref=mth_r, rel_l2_max=4e-3, dims=dims, **TH_CONV)
    c.finish()


def test_conv_rgb_planar_and_uint8_on_ragged_tiles():
    """decoder.conv_out: Cout = 3 with the bias zero-padded to 8; planar bf16 output, and uint8 pixels that must equal
    the host postprocess rule applied to the kernel's own bf16 image."""
    g = _g(150)
    N, H, W, Cin, Cout = 2, 9, 17, 128, 3
    x = _bf(N, H, W, Cin, g=g)
    w = _bf(Cout, 3, 3, Cin, g=g, scale=2 * (9 * Cin) ** -0.5)
    b = torch.zeros(8, device="cuda", dtype=torch.bfloat16)
    b[:3] = _bf(3, g=g, scale=0.3)
    planar = torch.empty(N, Cout, H, W, device="cuda", dtype=torch.bfloat16)
    _conv(x, w, b, planar, None, N, H, W, Cin, Cout, 1, 1)
    u8 = torch.empty(N, H, W, Cout, device="cuda", dtype=torch.uint8)
    _conv(x, w, b, u8, None, N, H, W, Cin, Cout, 1, 2)
    emu, floor, mth = R.conv_emu(x, w, b[:3], 1)
    c = R.Checker("conv rgb 9x17")
    nhwc = planar.permute(0, 2, 3, 1)
    c.bf16("planar", nhwc, emu, floor, math_ref=mth, rel_l2_max=4e-3, dims=("n", "y", "x", "c"), **TH_CONV)
    c.equal("uint8 == rule(bf16 image)", u8, R.u8_rule(nhwc))
    c.finish()
