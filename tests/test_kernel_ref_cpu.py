"""CPU tier for tests/kernel_ref.py: each fp64 emulation agrees with an independent math reference to bf16 level, and
the element-wise checks catch errors that the whole-tensor rel-L2 gates of the older GPU tests let through."""
import math

import pytest
import torch
import torch.nn.functional as F

import kernel_ref as R

F64 = torch.float64


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _bf(*shape, g, scale=1.0):
    return (torch.randn(*shape, generator=g, dtype=F64) * scale).bfloat16()


def test_bf16_helpers():
    x = torch.tensor([1.0, 1.5, -3.0, 0.0, 2.0 ** -130, 1000.0], dtype=F64)
    assert torch.equal(R.ulp_bf16(x), torch.tensor([2.0 ** -7, 2.0 ** -7, 2.0 ** -6, 2.0 ** -133, 2.0 ** -133, 4.0],
                                                   dtype=F64))
    # round to nearest even at bf16 precision
    assert R.bf16r(torch.tensor([1 + 2.0 ** -8], dtype=F64)).item() == 1.0
    assert R.bf16r(torch.tensor([1 + 3 * 2.0 ** -8], dtype=F64)).item() == 1 + 2.0 ** -6
    emu = torch.tensor([1.0, -2.0, 0.0], dtype=F64)
    out = torch.tensor([1.0 + 2.0 ** -6, -2.0, float("nan")], dtype=F64)
    d = R.ulp_diff(out, emu, floor=torch.tensor([0.0, 0.0, 1e-3], dtype=F64))
    assert d[0].item() == 2.0 and d[1].item() == 0.0 and math.isinf(d[2].item())


# ---------------------------------------------------------------------------------------------------- emulation vs math
def _sdpa64(q, k, v, *, scale, causal=False, bias=None):
    """F.scaled_dot_product_attention in fp64 on [B,S,H,D] views (GQA expanded by hand)."""
    B, Sq, H, D = q.shape
    rep = H // k.shape[2]
    qf = q.to(F64).transpose(1, 2)
    kf = k.to(F64).transpose(1, 2).repeat_interleave(rep, 1)
    vf = v.to(F64).transpose(1, 2).repeat_interleave(rep, 1)
    mask = None if bias is None else bias.to(F64)[None]
    o = F.scaled_dot_product_attention(qf, kf, vf, attn_mask=mask, is_causal=causal, scale=scale)
    return o.transpose(1, 2).reshape(B, Sq, H * D)


@pytest.mark.parametrize("B,H,Hkv,Sq,Skv,causal,bias", [
    (1, 2, 2, 65, 300, False, False),    # three K/V blocks, ragged tail
    (2, 4, 2, 129, 129, True, False),    # GQA, causal across a block edge
    (1, 3, 1, 40, 257, False, False),    # 3 query heads per kv head
    (1, 2, 2, 130, 130, False, True),    # additive bias, scale 1 (T5)
])
def test_attention_emulation_matches_sdpa(B, H, Hkv, Sq, Skv, causal, bias):
    g = _g(Sq + Skv)
    sc = 0.3 if bias else 1.0
    q, k, v = _bf(B, Sq, H, 128, g=g, scale=sc), _bf(B, Skv, Hkv, 128, g=g, scale=sc), _bf(B, Skv, Hkv, 128, g=g)
    bb = _bf(H, Sq, Skv, g=g) if bias else None
    scale = 1.0 if bias else 128 ** -0.5
    ref = _sdpa64(q, k, v, scale=scale, causal=causal, bias=bb)
    mth, lse_m = R.attention_math(q, k, v, scale=scale, causal=causal, bias=bb)
    assert R.rel_l2(mth, ref) < 1e-12
    emu, lse, floor = R.attention_emu(q, k, v, scale=scale, causal=causal, bias=bb)
    # P~ and the output are bf16: the emulation sits two bf16 roundings from the exact op, no further
    assert 5e-4 < R.rel_l2(emu, ref) < 6e-3
    assert ((emu - ref).abs() <= 4 * R.ulp_bf16(ref) + 4e-3 * ref.abs().max()).all()
    assert (lse - lse_m).abs().max().item() < 1e-8      # the online lse is exact to fp64 rounding


def test_attention_bwd_emulation_matches_autograd():
    g = _g(7)
    B, S, H = 2, 150, 2
    q, k, v = (_bf(B, S, H, 128, g=g) for _ in range(3))
    do = _bf(B, S, H * 128, g=g)
    o, lse, _ = R.attention_emu(q, k, v)
    dq, dk, dv, _ = R.attention_bwd_emu(q, k, v, o, do, lse)
    rq, rk, rv = R.attention_bwd_math(q, k, v, do)
    for a, b in ((dq, rq), (dk, rk), (dv, rv)):
        assert R.rel_l2(a, b) < 1.2e-2


@pytest.mark.parametrize("N,H,W,Cin,Cout,stride", [(2, 5, 7, 64, 8, 1), (1, 9, 6, 64, 16, 2)])
def test_conv_emulation_matches_tap_sum(N, H, W, Cin, Cout, stride):
    g = _g(H * W)
    x = _bf(N, H, W, Cin, g=g)
    w = _bf(Cout, 3, 3, Cin, g=g, scale=(9 * Cin) ** -0.5)
    b = _bf(Cout, g=g)
    # independent reference: explicit sum over the nine taps of the zero-padded input
    xp = F.pad(x.to(F64), (0, 0, 1, 1, 1, 1)) if stride == 1 else F.pad(x.to(F64), (0, 0, 0, 1, 0, 1))
    Ho, Wo = (H, W) if stride == 1 else (H // 2, W // 2)
    ref = b.to(F64).expand(N, Ho, Wo, Cout).clone()
    for ky in range(3):
        for kx in range(3):
            patch = xp[:, ky:ky + stride * Ho:stride, kx:kx + stride * Wo:stride, :]
            ref += patch @ w[:, ky, kx, :].to(F64).T
    resid = _bf(N, Ho, Wo, Cout, g=g)
    emu, floor, mth = R.conv_emu(x, w, b, stride)
    assert R.rel_l2(mth, ref) < 1e-12
    assert (R.ulp_diff(emu, ref) <= 0.5).all()
    emu_r, floor_r, mth_r = R.conv_emu(x, w, b, stride, resid=resid)
    # two roundings (conv + bias, then the residual sum): within one ulp of the output plus the inner rounding
    assert (R.ulp_diff(emu_r, resid.to(F64) + ref, floor_r) <= 1.0).all()


def test_dgrad_wgrad_emulation_matches_autograd():
    g = _g(3)
    B, M, N, K = 2, 37, 24, 40
    x = _bf(B, M, N, g=g)
    w = _bf(K, N, g=g, scale=0.2)
    dy = _bf(B, M, K, g=g)
    # the fused dgrad epilogue: dX = (dY @ W) * act'(u), u the saved pre-activation [B, M, N] of an activation that
    # follows the layer whose input gradient dX is
    u = _bf(B, M, N, g=g, scale=2.0)
    for epi, act in ((R.EPI_DGELU, lambda t: F.gelu(t, approximate="tanh")), (R.EPI_DSILU, F.silu)):
        uf = u.to(F64).requires_grad_(True)
        act(uf).backward(dy.to(F64) @ w.to(F64))
        emu, _, mth = R.dgrad_emu(dy, w, epi, aux=u)
        assert R.rel_l2(mth, uf.grad) < 1e-12
        assert R.rel_l2(emu, uf.grad) < 6e-3
    # wgrad: the gradient of W in y = x @ W^T with upstream dy
    W = torch.zeros(K, N, dtype=F64, requires_grad=True)
    (x.to(F64) @ W.T).backward(dy.to(F64))
    ref, floor = R.wgrad_math(dy, x)
    assert R.rel_l2(ref, W.grad) < 1e-12 and (floor > 0).all()


@pytest.mark.parametrize("epi", [R.EPI_BIAS, R.EPI_GELU_TANH, R.EPI_GELU_ERF, R.EPI_SILU, R.EPI_QUICK_GELU,
                                 R.EPI_GATE_RESID, R.EPI_RESID])
def test_linear_epilogue_emulation_matches_torch(epi):
    g = _g(epi)
    B, M, N, K = 2, 33, 40, 64
    x, w, b = _bf(B, M, K, g=g), _bf(N, K, g=g, scale=0.2), _bf(N, g=g)
    resid, gate = _bf(B, M, N, g=g), _bf(B, N, g=g)
    emu, floor, acc = R.linear_emu(x, w, b, epi, resid=resid, gate=gate)
    a = F.linear(x.to(F64), w.to(F64), b.to(F64))
    ref = {R.EPI_BIAS: lambda: a, R.EPI_GELU_TANH: lambda: F.gelu(a, approximate="tanh"),
           R.EPI_GELU_ERF: lambda: F.gelu(a), R.EPI_SILU: lambda: F.silu(a),
           R.EPI_QUICK_GELU: lambda: a * torch.sigmoid(1.702 * a),
           R.EPI_GATE_RESID: lambda: resid.to(F64) + gate.to(F64)[:, None] * a,
           R.EPI_RESID: lambda: resid.to(F64) + a}[epi]()
    assert R.rel_l2(emu, ref) < 6e-3
    assert (floor >= 0).all()


def test_qkv_norm_rope_emulation_matches_math():
    g = _g(11)
    B, M, H, K, row0, n_extra = 2, 20, 2, 64, 5, 256
    d = H * 128
    x = _bf(B, M, K, g=g)
    w = _bf(3 * d + n_extra, K, g=g, scale=0.1)
    b = _bf(3 * d + n_extra, g=g)
    nq, nk = (1 + 0.1 * torch.randn(128, generator=g, dtype=F64)).bfloat16(), (1 + 0.1 * torch.randn(128, generator=g,
                                                                                                        dtype=F64)).bfloat16()
    ang = torch.rand(row0 + M, 64, generator=g, dtype=F64) * 6.28
    cos = torch.cos(ang).repeat_interleave(2, 1).float()
    sin = torch.sin(ang).repeat_interleave(2, 1).float()
    emu, floor, mth = R.qkv_norm_rope_emu(x, w, b, nq, nk, cos, sin, rope_row0=row0, n_extra=n_extra,
                                          epi_extra=R.EPI_GELU_TANH)
    # independent restatement of diffusers RMSNorm + apply_rotary_emb on the fp64 projection
    a = F.linear(x.to(F64), w.to(F64), b.to(F64))
    for blk, nw in ((0, nq), (1, nk)):
        h = a[..., blk * d:(blk + 1) * d].unflatten(-1, (H, 128))
        y = h * torch.rsqrt(h.pow(2).mean(-1, keepdim=True) + 1e-6) * nw.to(F64)
        yr, yi = y.unflatten(-1, (64, 2)).unbind(-1)
        rot = torch.stack([-yi, yr], -1).flatten(-2)
        c, s = cos[row0:].to(F64)[:, None], sin[row0:].to(F64)[:, None]
        ref = (y * c + rot * s).flatten(-2)
        assert R.rel_l2(mth[..., blk * d:(blk + 1) * d], ref) < 1e-12
        assert R.rel_l2(emu[..., blk * d:(blk + 1) * d], ref) < 8e-3
    assert R.rel_l2(emu[..., 3 * d:], F.gelu(a[..., 3 * d:], approximate="tanh")) < 6e-3


# ---------------------------------------------------------------------------------------------------- the checks have teeth
def _fails(fn) -> str:
    with pytest.raises(AssertionError) as e:
        fn()
    return str(e.value)


# the attention thresholds of the GPU edge tests (tests/test_sm90_edges_gpu.py)
_TH = dict(max_ulp=2, share_gt1=1e-3, mean_ulp=0.05)


def test_checks_catch_three_ulp_element():
    g = _g(1)
    x, w, b = _bf(64, 64, g=g), _bf(72, 64, g=g, scale=0.1), _bf(72, g=g)
    emu, floor, acc = R.linear_emu(x, w, b)
    out = emu.clone()
    out[17, 41] += 3 * R.ulp_bf16(emu[17, 41])
    ok = R.Checker("clean")
    ok.bf16("out", emu, emu, floor, **_TH)
    ok.finish()
    c = R.Checker("3ulp")
    c.bf16("out", out, emu, floor, dims=("row", "col"), **_TH)
    msg = _fails(c.finish)
    assert "row=17, col=41" in msg


def test_checks_catch_replaced_token_head_row_that_rel_l2_misses():
    """Output of attention at (1, 4, 4, 8736) proportions: one (token, head) row of 128 values is never written (left
    at zero).  The old gate (rel-L2 < 8e-3 against the fp32 reference) passes; the element-wise check names the row."""
    g = _g(2)
    S, H = 8736, 4
    ref = torch.randn(1, S, H, 128, generator=g, dtype=F64) * 0.05
    emu = R.bf16r(ref)
    out = emu.clone()
    out[0, 5000, 2] = 0
    assert R.rel_l2(out, ref) < 8e-3
    c = R.Checker("row-replaced")
    c.bf16("o", out, emu, 0.0, dims=("b", "token", "head", "col"), **_TH)
    msg = _fails(c.finish)
    assert "token=5000, head=2" in msg


def test_checks_catch_extra_zero_key_that_rel_l2_misses():
    """A tail mask off by one lets the zero-filled key at column Skv into every softmax denominator (O shrinks by
    l / (l + 2^-m)).  At the proportions of the (2, 3, 3, 300, 300) attention test the old gate passes; the mean ulp
    shift does not."""
    g = _g(3)
    B, S, H = 1, 300, 3
    q, k, v = (_bf(B, S, H, 128, g=g) for _ in range(3))
    mth, _ = R.attention_math(q, k, v)
    emu, lse, floor = R.attention_emu(q, k, v)
    z = torch.zeros(B, 1, H, 128, dtype=torch.bfloat16)
    bad, bad_lse, _ = R.attention_emu(q, torch.cat([k, z], 1), torch.cat([v, z], 1))
    assert R.rel_l2(bad, mth) < 8e-3
    ok = R.Checker("clean")
    ok.bf16("o", emu, emu, floor, **_TH)
    ok.finish()
    c = R.Checker("extra-key")
    c.bf16("o", bad, emu, floor, **_TH)
    msg = _fails(c.finish)
    assert "mean ulp_diff" in msg
    assert (bad_lse - lse).min().item() > 0       # the lse rows move too


def test_checks_catch_missing_bias_in_one_column_group():
    g = _g(4)
    M, N, K = 256, 512, 64
    x, w, b = _bf(M, K, g=g), _bf(N, K, g=g, scale=0.1), _bf(N, g=g, scale=0.1)
    emu, floor, acc = R.linear_emu(x, w, b)
    b2 = b.clone()
    b2[24:32] = 0
    out, _, _ = R.linear_emu(x, w, b2)
    c = R.Checker("bias-group")
    c.bf16("out", out, emu, floor, dims=("row", "col"), **_TH)
    msg = _fails(c.finish)
    assert "col=2" in msg or "col=3" in msg


def test_fp32_check_catches_one_wrong_column_group():
    """wgrad output (fp32) with 3072 columns: one 8-column group 1.5 % off.  The old gate (rel-L2 < 1e-3) passes."""
    g = _g(5)
    dy, x = _bf(1, 64, 64, g=g), _bf(1, 64, 3072, g=g)
    ref, floor = R.wgrad_math(dy, x)
    out = ref.float()
    out[:, 96:104] *= 0.985
    assert R.rel_l2(out, ref) < 1e-3
    c = R.Checker("wgrad-group")
    c.within_floor("dw", out, ref, floor, max_ratio=1.0, dims=("m", "n"))
    _fails(c.finish)
