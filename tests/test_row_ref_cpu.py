"""CPU tier for tests/row_ref.py: each fp64 emulation of a row kernel agrees with an independent fp64 reference
(torch.nn.functional, autograd through the forward emulation, torch.optim.AdamW), and the element-wise checks catch
errors that the older whole-tensor gates of the row-kernel tests pass."""
import math

import pytest
import torch
import torch.nn.functional as F

import kernel_ref as R
import row_ref as RR

F64 = torch.float64


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _bf(*shape, g, scale=1.0, shift=0.0):
    return (torch.randn(*shape, generator=g, dtype=F64) * scale + shift).bfloat16()


def _fails(fn):
    with pytest.raises(AssertionError) as e:
        fn()
    return str(e.value)


def _bf16_close(emu, ref, n_ulp, mag=None):
    """emu (a chain of bf16 roundings of ref) within n_ulp bf16 ulps of `mag` (the magnitude of the chain's
    intermediates; default ref itself), or a small absolute amount near zero."""
    tol = n_ulp * R.ulp_bf16(ref.abs() if mag is None else mag) + 2 ** -12 * ref.abs().amax()
    assert ((emu - ref).abs() <= tol).all(), ((emu - ref).abs() / tol).max().item()


# ---------------------------------------------------------------------------------------------------- emulation vs math
def test_ln_modulate_emulation_matches_layer_norm():
    g = _g(1)
    B, rows, D, split = 2, 9, 256, 4
    x = _bf(B, rows, D, g=g, scale=2.0, shift=0.5)
    mod = _bf(B, 4 * D, g=g, scale=0.3)
    sc, sh, scb, shb = (mod[:, i * D:(i + 1) * D] for i in range(4))
    emu, floor, mth = RR.ln_modulate_emu(x, sc, sh, split_row=split, scale_b=scb, shift_b=shb)
    ln = F.layer_norm(x.to(F64), (D,), eps=1e-6)
    sel = lambda a, b: torch.cat([a.to(F64)[:, None].expand(B, split, D), b.to(F64)[:, None].expand(B, rows - split, D)], 1)
    ref = ln * (1 + sel(sc, scb)) + sel(sh, shb)
    assert R.rel_l2(mth, ref) < 1e-12
    _bf16_close(emu, ref, 3, mag=(ln * (1 + sel(sc, scb))).abs() + sel(sh, shb).abs())


def test_ln_modulate_bwd_emulation_matches_autograd():
    g = _g(2)
    B, rows, D, split = 2, 20, 256, 6
    x = _bf(B, rows, D, g=g, scale=2.0, shift=0.5)
    dy, dres = _bf(B, rows, D, g=g), _bf(B, rows, D, g=g)
    mod = _bf(B, 2 * D, g=g, scale=0.3)
    sc, scb = mod[:, :D], mod[:, D:]
    (dx, fl, mth), (ds, _), (dh, _) = RR.ln_modulate_bwd_emu(x, dy, sc, split_row=split, scale_b=scb, dres=dres,
                                                              part_row0=split)
    xf = x.to(F64).requires_grad_(True)
    s = RR.per_row(sc, scb, rows, split).clone().requires_grad_(True)
    h = torch.zeros_like(s).requires_grad_(True)
    (F.layer_norm(xf, (D,), eps=1e-6) * (1 + s) + h).backward(dy.to(F64))
    ref = dres.to(F64) + xf.grad
    assert R.rel_l2(mth, ref) < 1e-12
    # bf16(1 + scale) against the exact factor: 2^-9 of every term of the gradient
    gm = dy.to(F64) * (1 + s.detach())
    _bf16_close(dx, ref, 4, mag=dres.to(F64).abs() + 2 * xf.grad.abs() + gm.abs() * torch.rsqrt(xf.var(-1, True, keepdim=True)))
    assert R.rel_l2(ds, s.grad[:, split:].sum(1)) < 5e-3      # bf16(xhat), as in the forward
    assert R.rel_l2(dh, h.grad[:, split:].sum(1)) < 1e-12


def test_rmsnorm_rope_and_backward_emulations_match_autograd():
    g = _g(3)
    B, S, H, n_a = 2, 11, 3, 4
    xq, xk = _bf(B, S, H, 128, g=g), _bf(B, S, H, 128, g=g)
    dq, dk = _bf(B, S, H, 128, g=g), _bf(B, S, H, 128, g=g)
    ws = [(torch.rand(128, generator=g, dtype=F64) + 0.5).bfloat16() for _ in range(4)]   # q A, k A, q B, k B
    ang = torch.rand(S, 64, generator=g, dtype=F64) * 6.28
    cos, sin = (f(ang).repeat_interleave(2, 1).float() for f in (torch.cos, torch.sin))
    fw = RR.rmsnorm_rope_emu((xq, xk), ws[2], ws[3], cos, sin, wq_a=ws[0], wk_a=ws[1], n_a=n_a)
    grads, (wg, _) = RR.rmsnorm_rope_bwd_emu((xq, xk), (dq, dk), ws[2], ws[3], cos, sin, wq_a=ws[0], wk_a=ws[1], n_a=n_a)
    wf = [w.to(F64).requires_grad_(True) for w in ws]
    xs = [t.to(F64).requires_grad_(True) for t in (xq, xk)]
    c, s_ = cos.to(F64)[None, :, None], sin.to(F64)[None, :, None]
    for i, (x, d) in enumerate(zip(xs, (dq, dk))):
        w = torch.where(torch.arange(S)[None, :, None, None] < n_a, wf[i], wf[2 + i])
        y = x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-6) * w
        o = y * c + R._rot_pairs(y) * s_
        emu, _, mth = fw[i]
        assert R.rel_l2(mth, o) < 1e-12
        _bf16_close(emu, o.detach(), 4, mag=(y.abs() * c.abs() + R._rot_pairs(y).abs() * s_.abs()).detach())
        o.backward(d.to(F64))
    for i in range(2):
        assert R.rel_l2(grads[i][2], xs[i].grad) < 1e-12
        _bf16_close(grads[i][0], xs[i].grad, 2)
    for i in range(4):
        assert R.rel_l2(wg[i], wf[i].grad) < 5e-3                  # bf16(x r) in the weight gradient


def test_optimizer_chain_matches_torch_adamw_and_clip():
    g = _g(4)
    n = 1003
    p = torch.randn(n, generator=g, dtype=F64).float()
    m, v = torch.zeros(n), torch.zeros(n)
    ref = torch.nn.Parameter(p.to(F64).clone())
    opt = torch.optim.AdamW([ref], lr=1e-3, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.05)
    for step in range(1, 4):
        grad = (torch.randn(n, generator=g, dtype=F64) * 3).float()
        ss, _ = RR.grad_sumsq_emu(grad)
        coef, _, nrm, _ = RR.clip_coef_emu(ss, 1.0)
        ref.grad = grad.to(F64).clone()
        total = torch.nn.utils.clip_grad_norm_([ref], 1.0)
        assert abs(nrm.item() - total.item()) < 1e-12 * total.item()
        opt.step()
        (p1, fp), (m1, _), (v1, _) = RR.adamw_emu(p, m, v, grad, lr=1e-3, betas=(0.9, 0.95), eps=1e-8, wd=0.05,
                                                   step=step, gscale=coef)
        # the emulation uses the kernel's fp32 constants (betas, bias corrections): a few fp32 ulps of the update
        assert ((p1 - ref.data).abs() <= 1e-6 * (p1.abs() + 1e-3)).all()
        p, m, v = p1.float(), m1.float(), v1.float()
        ref.data.copy_(p.to(F64))


def test_loss_and_small_kernel_emulations():
    g = _g(5)
    pred, target, w = _bf(3, 257, g=g), torch.randn(3, 257, generator=g).float(), torch.rand(3, 257, generator=g).float()
    (loss, _), (dp, _, dpm) = RR.mse_loss_emu(pred, target, w, grad_scale=0.5)
    pf = pred.to(F64).requires_grad_(True)
    lr = (w.to(F64) * (pf - target.to(F64)) ** 2).mean()
    (lr * 0.5).backward()
    assert abs(loss.item() - lr.item()) < 1e-12 and R.rel_l2(dpm, pf.grad) < 1e-6
    _bf16_close(dp, pf.grad, 1)
    x = _bf(40, 64, g=g, scale=4.0)
    emu, _, mth = RR.gelu_rows_emu(x)
    assert R.rel_l2(mth, F.gelu(x.to(F64), approximate="tanh")) < 1e-12
    gu = _bf(5, 2 * 48, g=g, scale=3.0)
    _, _, sw = RR.swiglu_emu(gu, 48)
    _, _, ge = RR.geglu_emu(gu, 48)
    gd = gu.to(F64)
    assert R.rel_l2(sw, F.silu(gd[:, :48]) * gd[:, 48:]) < 1e-12
    assert R.rel_l2(ge, F.gelu(gd[:, :48], approximate="tanh") * gd[:, 48:]) < 1e-12
    s = _bf(6, 2056, g=g, scale=4.0)
    emu, _, mth = RR.softmax_rows_emu(s, 0.3)
    assert R.rel_l2(mth, F.softmax(s.to(F64) * 0.3, -1)) < 1e-12
    _bf16_close(emu, mth, 1)
    dmod, act = torch.randn(3, 16, generator=g).float(), _bf(3, 40, g=g)
    ref, _ = RR.outer_acc_emu(dmod, act)
    assert R.rel_l2(ref, torch.einsum("bn,bk->nk", dmod.to(F64), act.to(F64))) < 1e-12


def test_timestep_embedding_and_rope_table_emulations():
    g = _g(12)
    t = torch.tensor([0.0, 0.5, 999.75, 1000.0], dtype=torch.float32)
    emu, floor, mth = RR.temb_sinusoid_emu(t)
    # diffusers get_timestep_embedding(t, 256, flip_sin_to_cos=True, downscale_freq_shift=0), in fp64
    half = 128
    freqs = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=F64) / half)
    ang = t.to(F64)[:, None] * freqs[None]
    ref = torch.cat([torch.cos(ang), torch.sin(ang)], -1)
    assert R.rel_l2(mth, ref) < 1e-14
    _bf16_close(emu, ref, 1)
    assert (floor < 4 * R.ulp_bf16(torch.ones(1, dtype=F64))).all()      # below one bf16 ulp of 1 even at t = 1000
    x = _bf(64, g=g, scale=6.0)
    emu, _, mth = RR.silu_emu(x)
    assert R.rel_l2(mth, F.silu(x.to(F64))) < 1e-14
    tt, gg, txt = _bf(16, g=g), _bf(16, g=g), _bf(16, g=g)
    temb, (se, _, _) = RR.temb_combine_emu(tt, gg, txt)
    assert torch.equal(temb, ((tt + gg) + txt).to(F64))                   # torch's own bf16 chain
    assert torch.equal(se, F.silu(temb).bfloat16().to(F64))
    ids = torch.tensor([[0.0, 0.0, 0.0], [0.0, 17.0, 4096.0]])
    c, s, _ = RR.rope_tables_emu(ids)
    # FluxPosEmbed: per axis, pairs of dim / 2 frequencies theta^(-2i / dim), interleaved cos / sin
    w = torch.cat([10000.0 ** (-torch.arange(0, d, 2, dtype=F64) / d) for d in (16, 56, 56)])
    axis = torch.cat([torch.full((d // 2,), a) for a, d in enumerate((16, 56, 56))])
    ang = ids.to(F64)[:, axis] * w[None]
    assert (c - torch.cos(ang).repeat_interleave(2, 1)).abs().max() < 1e-12
    assert (s - torch.sin(ang).repeat_interleave(2, 1)).abs().max() < 1e-12


def test_llm_norm_and_rope_emulations():
    g = _g(6)
    x = _bf(7, 512, g=g, shift=3.0)
    w, b = _bf(512, g=g), _bf(512, g=g)
    emu, _, mth = RR.layernorm_emu(x, w, b)
    ref = F.layer_norm(x.to(F64), (512,), w.to(F64), b.to(F64), eps=1e-5)
    assert R.rel_l2(mth, ref) < 1e-12
    _bf16_close(emu, ref, 1)
    emu, _, mth = RR.rmsnorm_emu(x, w)
    xd = x.to(F64)
    ref = w.to(F64) * xd * torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + 1e-6)
    assert R.rel_l2(mth, ref) < 1e-12
    _bf16_close(emu, ref, 2, mag=ref.abs() * 2)
    # rotate-half: the text path's bf16 chain and the vision path's single rounding both sit near the exact rotation
    t = _bf(5, 2 * 128 + 64, g=g)
    ang = torch.rand(5, 64, generator=g, dtype=F64) * 6.28
    cos = torch.cat([torch.cos(ang)] * 2, -1).bfloat16().float()
    sin = torch.cat([torch.sin(ang)] * 2, -1).bfloat16().float()
    a, bb = t.to(F64)[:, :64], t.to(F64)[:, 64:128]
    for fp32 in (True, False):
        emu, _, mth = RR.rope_half_emu(t, 2, 128, cos, sin, fp32_math=fp32)
        assert R.rel_l2(mth[:, :64], a * cos[:, :64].double() - bb * sin[:, :64].double()) < 1e-12
        mag = torch.cat([a, bb], -1).abs() + torch.cat([bb, a], -1).abs()      # |cos|, |sin| <= 1
        _bf16_close(emu[:, :128], mth[:, :128], 3, mag=mag)
        assert torch.equal(emu[:, 256:], t.to(F64)[:, 256:])


@pytest.mark.parametrize("C,shift", [(128, 0.3), (256, 20.0)])
def test_groupnorm_emulation_matches_group_norm(C, shift):
    g = _g(7)
    N, P = 2, 300
    x = _bf(N, P, C, g=g, scale=2.0, shift=shift)
    ga, be = _bf(C, g=g, scale=0.1, shift=1.0), _bf(C, g=g, scale=0.1)
    emu, floor, mth = RR.groupnorm_silu_emu(x, ga, be)
    ref = F.silu(F.group_norm(x.to(F64).permute(0, 2, 1), 32, ga.to(F64), be.to(F64), eps=1e-6)).permute(0, 2, 1)
    assert R.rel_l2(mth, ref) < 1e-10
    _bf16_close(emu, ref, 3)


# ---------------------------------------------------------------------------------------------------- what old gates miss
TH = dict(max_ulp=2, share_gt1=1e-3, mean_ulp=0.05)


def test_adamw_tail_without_weight_decay_passes_old_gate():
    """n = 100 003: the last 3 elements (the scalar tail after 25 000 float4s) skip the decoupled weight decay.
    The old gate (rel-L2 < 1e-5 over the shard) passes; the per-element fp32 floor names the tail."""
    g = _g(8)
    n = 100_003
    p = torch.randn(n, generator=g).float()
    m, v = torch.randn(n, generator=g).float() * 0.01, torch.rand(n, generator=g).float() * 1e-4
    grad = torch.randn(n, generator=g).float()
    kw = dict(lr=1e-3, betas=(0.9, 0.95), eps=1e-8, step=7)
    (p1, fp), _, _ = RR.adamw_emu(p, m, v, grad, wd=0.05, **kw)
    (p_nowd, _), _, _ = RR.adamw_emu(p, m, v, grad, wd=0.0, **kw)
    bad = p1.clone()
    bad[-3:] = p_nowd[-3:]
    assert R.rel_l2(bad.float(), p1) < 1e-5
    ok = R.Checker("clean")
    ok.within_floor("p32", p1.float(), p1, fp, max_ratio=1.0)
    ok.finish()
    c = R.Checker("tail-no-decay")
    c.within_floor("p32", bad.float(), p1, fp, max_ratio=1.0, dims=("i",))
    msg = _fails(c.finish)
    assert "i=10000" in msg


def test_ln_modulate_row_with_other_stream_passes_composed_gate():
    """The first image row of a double block modulated with the text stream's (scale, shift): an off-by-one split.
    At (1, 64 + 4032, 1024) the composed model gate (2 x torch-bf16's rel-L2 + 1e-2) passes; the ulp check names the row."""
    g = _g(9)
    B, S_txt, S, D = 1, 64, 4096, 1024
    x = _bf(B, S, D, g=g, scale=2.0, shift=0.3)
    mod = _bf(B, 4 * D, g=g, scale=0.3)
    sc, sh, scb, shb = (mod[:, i * D:(i + 1) * D] for i in range(4))
    emu, floor, mth = RR.ln_modulate_emu(x, sc, sh, split_row=S_txt, scale_b=scb, shift_b=shb)
    bad, _, _ = RR.ln_modulate_emu(x, sc, sh, split_row=S_txt + 1, scale_b=scb, shift_b=shb)
    torch_bf16 = R.bf16r(R.bf16r(R.bf16r(F.layer_norm(x.to(F64), (D,), eps=1e-6))
                                 * R.bf16r(1 + RR.per_row(sc, scb, S, S_txt))) + RR.per_row(sh, shb, S, S_txt))
    assert R.rel_l2(bad, mth) < 2 * R.rel_l2(torch_bf16, mth) + 1e-2
    c = R.Checker("split+1")
    c.bf16("out", bad, emu, floor, dims=("b", "row", "col"), **TH)
    msg = _fails(c.finish)
    assert "row=64" in msg


def test_dscale_missing_one_chunk_in_one_column_group_passes_old_gate():
    """dscale of ln_modulate_bwd at (1, 2336, 3072): one row's term lost for one 8-column group (a column-pass bug).  The old gate (rel-L2 < 5e-3) passes; the fp32 floor of the column sums does not."""
    g = _g(10)
    B, rows, D = 1, 2336, 3072
    x = _bf(B, rows, D, g=g, scale=2.0, shift=0.5)
    dy = _bf(B, rows, D, g=g)
    sc = _bf(B, D, g=g, scale=0.3)
    _, (ds, fds), _ = RR.ln_modulate_bwd_emu(x, dy, sc)
    xh = F.layer_norm(x.to(F64), (D,), eps=1e-6)
    bad = ds.clone()
    bad[:, 2400:2408] -= (dy.to(F64) * R.bf16r(xh))[:, 170, 2400:2408]
    assert R.rel_l2(bad, ds) < 5e-3
    c = R.Checker("dscale-chunk")
    c.within_floor("dscale", bad, ds, fds, max_ratio=1.0, dims=("b", "col"))
    msg = _fails(c.finish)
    assert "col=240" in msg


def test_groupnorm_neighbour_statistics_pass_old_gate():
    """GroupNorm at (2, 1000, 128) where one (item, group) normalises with its neighbour's statistics.  The old gate
    (<= 1.5 x torch-bf16's rel-L2 + 1e-4 over the tensor) passes; the ulp check names the group's channels."""
    g = _g(11)
    N, P, C = 2, 1000, 128
    x = _bf(N, P, C, g=g, scale=2.0, shift=0.3)
    ga, be = _bf(C, g=g, scale=0.1, shift=1.0), _bf(C, g=g, scale=0.1)
    emu, floor, mth = RR.groupnorm_silu_emu(x, ga, be)
    # the neighbour's statistics applied to group 5 of item 1: normalise its 4 channels with group 6's mean / rstd
    xd = x.to(F64)
    nb = xd[1, :, 24:28]
    mu, var = nb.mean(), nb.pow(2).mean() - nb.mean() ** 2
    bad = emu.clone()
    pre = (xd[1, :, 20:24] - mu) * torch.rsqrt(var + 1e-6) * ga.to(F64)[20:24] + be.to(F64)[20:24]
    bad[1, :, 20:24] = R.bf16r(F.silu(R.bf16r(pre)))
    r16 = F.silu(F.group_norm(x.permute(0, 2, 1), 32, ga, be, eps=1e-6)).permute(0, 2, 1)
    assert R.rel_l2(bad, mth) <= 1.5 * R.rel_l2(r16, mth) + 1e-4
    c = R.Checker("gn-neighbour")
    c.bf16("y", bad, emu, floor, dims=("n", "p", "c"), **TH)
    msg = _fails(c.finish)
    assert "n=1" in msg
