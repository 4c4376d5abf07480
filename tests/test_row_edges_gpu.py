"""Edge sweeps of the HBM-bound row kernels, element by element, against the fp64 references of row_ref.py.

The shapes aim at the launch edges of each kernel:
  ln_modulate            register template switches at D = 1024 / 3072, 4-row blocks, grid-stride after
                         12 blocks per SM; the text / image split inside a 4-row block;
  rmsnorm_rope(_out/_bwd) 8-token blocks straddling batch items and the weight-set boundary n_added;
  gate_resid / gate_bwd  1024-column blocks in y, 32-row chunks of column partials, part_row0 inside a chunk;
  ln_modulate_bwd        16-row chunks, a second column pass past 2048 columns;
  grad_sumsq / adamw     the 4-deep unrolled loop, the second in-flight float4, the scalar tail and the unaligned path;
  mse_loss               the grid-stride loop past 1024 * 256 elements and ragged n;
  groupnorm              octets that span two groups (C = 128), per-thread fp32 partials, DC offsets.

Every pitched or in-place output lives inside a NaN-filled buffer, and each check asserts that nothing outside its
region changed.  Each case that targets a launch path asserts, from the launch formula, that its shape reaches it.
Every check prints a KREF line (max ulp, share > 1 ulp, mean ulp; or error / fp32 floor).  Thresholds were set from
runs of the unmodified kernels on an H100 80GB HBM3 (400 W power limit): at most 2 ulp (ln_modulate_bwd; GroupNorm
1.85, ln_modulate 1.27, every other family <= 1), a share above 1 ulp of at most 2.9e-5, a mean of at most 0.0021 ulp,
and fp32 outputs at most 0.99 of their floor (ln_modulate_bwd column sums; the floor allows the one bf16 flip of a term).
"""
import math

import pytest
import torch

import kernel_ref as R
import row_ref as RR

pytestmark = pytest.mark.gpu

# bf16 outputs against their emulation.  The floors allow an intermediate bf16 flip only where the fp32 value lies
# within its error bound of a tie; an H100 still shows a few such flips outside the bound (at most 2 ulp, in at most
# 3e-5 of the elements of a GroupNorm, ln_modulate or ln_modulate_bwd output), hence 2 ulp in at most 1e-4
TH = dict(max_ulp=2, share_gt1=1e-4, mean_ulp=0.02)
BF, F32 = torch.bfloat16, torch.float32


def _g(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _bf(*shape, g, scale=1.0, shift=0.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale + shift).to(BF)


def _nan(*shape, dtype=BF):
    return torch.full(shape, math.nan, device="cuda", dtype=dtype)


def _outside(c, name, buf, before, region):
    """Everything of `buf` outside `region` (an index into buf) equals `before` (NaN sentinels compared bitwise)."""
    mask = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    mask[region] = False
    a, b = buf[mask], before[mask]
    c.equal(f"{name}: outside the output region", a.view(torch.int16) if a.dtype == BF else a.view(torch.int32),
            b.view(torch.int16) if b.dtype == BF else b.view(torch.int32))


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------------------------------------------- ln_modulate
LN_CASES = [(D, rows, split) for D in (256, 1024, 1280, 3072, 3328, 5120) for rows, split in ((1, 0), (3, 1), (5, 4))]
LN_CASES += [(1024, 4000, 6), (3072, 4000, 6), (5120, 4000, 3999)]


@pytest.mark.parametrize("D,rows,split", LN_CASES)
def test_ln_modulate_edges(D, rows, split):
    from gpt_image_edit_b200 import ops

    B = 2
    if rows == 4000:   # the grid-stride sweep: at most 12 four-row blocks per SM (elementwise.cu ln_modulate)
        assert B * rows > 4 * 12 * _sms()
    g = _g(D + rows)
    xa = _bf(B, rows + 3, D + 64, g=g, scale=1.5, shift=0.2)
    x = xa[:, 2:2 + rows, 32:32 + D]                     # row pitch D + 64, batch stride (rows + 3)(D + 64)
    x[1, 0] = 0.5                                        # an all-constant row
    if rows > 2:
        x[0, 2] = (torch.randn(D, device="cuda", generator=g) + 30.0).to(BF)   # mean 30 x std
    mod = _bf(B, 6 * D, g=g, scale=0.4)
    sc, sh, scb, shb = mod[:, D:2 * D], mod[:, 2 * D:3 * D], mod[:, 4 * D:5 * D], mod[:, 5 * D:]
    buf = _nan(B, rows + 2, D + 24)
    before = buf.clone()
    region = (slice(None), slice(1, 1 + rows), slice(8, 8 + D))
    out = buf[region]
    kw = dict(split_row=split, scale_b=scb, shift_b=shb) if split else {}
    ops.ln_modulate(x, sc, sh, out=out, **kw)
    emu, floor, mth = RR.ln_modulate_emu(x, sc, sh, **kw)
    c = R.Checker(f"ln_modulate D{D} rows{rows} split{split}")
    c.bf16("out", out, emu, floor, math_ref=mth, rel_l2_max=2e-2, dims=("b", "row", "col"), **TH)
    big = sh[1].abs() >= 2 ** -4          # below that, bf16(LN) of the constant row's fp32 residue may still show
    c.equal("constant row == shift", out[1, 0][big], sh[1][big])
    _outside(c, "out", buf, before, region)
    c.finish()


# ---------------------------------------------------------------------------------------------------- rmsnorm + RoPE
def _flux_ids(S, n_txt):
    """FLUX position ids: text rows (0, 0, 0); image rows (0, h, w) on a grid, reaching 4096."""
    i = torch.arange(S, device="cuda", dtype=torch.float64)
    ids = torch.stack([torch.zeros_like(i), (i * 37) % 4097, (i * 611) % 4097], 1)
    ids[:n_txt] = 0
    ids[-1, 1:] = 4096
    return ids.float()


NR_CASES = [   # (H, B, S, n_added, layout)
    (1, 3, 13, 7, "double"),     # 39 tokens: blocks straddle both batch boundaries; set A / B boundary inside a block
    (3, 2, 21, 1, "single"),
    (5, 1, 9, 0, "double"),
    (24, 2, 45, 45, "single"),   # every token in set A
    (24, 2, 37, 7, "double"),
]


def _nr_inputs(H, B, S, layout, g):
    d = H * 128
    wide = 3 * d if layout == "double" else 7 * d        # [Q|K|V] or [Q|K|V|mlp]
    buf = _bf(B, S, wide, g=g, scale=1.5)
    ws = [(torch.rand(128, device="cuda", generator=g) + 0.5).to(BF) for _ in range(4)]   # q A, k A, q B, k B
    return d, buf, ws


@pytest.mark.parametrize("H,B,S,n_a,layout", NR_CASES)
def test_rmsnorm_rope_edges(H, B, S, n_a, layout):
    from gpt_image_edit_b200 import ops, train_ops as T

    g = _g(H * 100 + S)
    d, buf, ws = _nr_inputs(H, B, S, layout, g)
    if B > 1 and (B * S) % 8:
        assert any((b0 // S) != ((b0 + 7) // S) for b0 in range(0, B * S - 7, 8))   # a block spans a batch boundary
    ids = _flux_ids(S, n_a)
    cos, sin = ops.rope_tables(ids)
    c = R.Checker(f"rmsnorm_rope H{H} B{B} S{S} n_added{n_a} {layout}")
    cr, sr, (fc, fs) = RR.rope_tables_emu(ids)
    c.within_floor("rope cos", cos, cr, fc, max_ratio=1.0, dims=("token", "col"))
    c.within_floor("rope sin", sin, sr, fs, max_ratio=1.0, dims=("token", "col"))
    qkv = buf[:, :, :3 * d]
    xq, xk = (qkv[:, :, i * d:(i + 1) * d].unflatten(-1, (H, 128)) for i in range(2))
    kw = dict(wq_a=ws[0], wk_a=ws[1], n_a=n_a)
    (eq, fq, mq), (ek, fk, mk) = RR.rmsnorm_rope_emu((xq, xk), ws[2], ws[3], cos, sin, **kw)
    # out of place: single block writes [Q|K] of a 3d-pitched buffer, V columns untouched
    ob = _nan(B, S, 3 * d)
    before = ob.clone()
    T.rmsnorm_rope(qkv, H, ws[2], ws[3], cos, sin, wq_added=ws[0], wk_added=ws[1], n_added=n_a, out=ob)
    dims = ("b", "token", "head", "col")
    c.bf16("out q", ob[:, :, :d].unflatten(-1, (H, 128)), eq, fq, math_ref=mq, rel_l2_max=1e-2, dims=dims, **TH)
    c.bf16("out k", ob[:, :, d:2 * d].unflatten(-1, (H, 128)), ek, fk, math_ref=mk, rel_l2_max=1e-2, dims=dims, **TH)
    _outside(c, "out", ob, before, (slice(None), slice(None), slice(0, 2 * d)))
    # in place on the pitched buffer: V (and the mlp columns) untouched
    ip = buf.clone()
    before = ip.clone()
    ops.rmsnorm_rope_(ip[:, :, :3 * d], H, ws[2], ws[3], cos, sin, wq_added=ws[0], wk_added=ws[1], n_added=n_a)
    c.equal("in place == out of place", ip[:, :, :2 * d].view(torch.int16), ob[:, :, :2 * d].view(torch.int16))
    _outside(c, "in place", ip, before, (slice(None), slice(None), slice(0, 2 * d)))
    c.finish()


@pytest.mark.parametrize("B,S,n_a,layout", [(3, 13, 7, "double"), (2, 21, 1, "single"), (1, 9, 0, "double"),
                                            (2, 45, 45, "single"), (2, 37, 7, "double")])
def test_rmsnorm_rope_bwd_edges(B, S, n_a, layout):
    from gpt_image_edit_b200 import ops, train_ops as T

    H = 24
    g = _g(S * 7 + B)
    d, xbuf, ws = _nr_inputs(H, B, S, layout, g)
    dbuf = _bf(B, S, xbuf.shape[-1], g=g)
    cos, sin = ops.rope_tables(_flux_ids(S, n_a))
    qkv_pre, dqkv = xbuf[:, :, :3 * d], dbuf[:, :, :3 * d]
    xq, xk = (qkv_pre[:, :, i * d:(i + 1) * d].unflatten(-1, (H, 128)) for i in range(2))
    dq, dk = (dqkv[:, :, i * d:(i + 1) * d].unflatten(-1, (H, 128)) for i in range(2))
    grads, (wg_ref, wg_fl) = RR.rmsnorm_rope_bwd_emu((xq, xk), (dq.clone(), dk.clone()), ws[2], ws[3], cos, sin,
                                                     wq_a=ws[0], wk_a=ws[1], n_a=n_a)
    before = dbuf.clone()
    wg = T.rmsnorm_rope_bwd_(dqkv, qkv_pre, H, ws[2], ws[3], cos, sin, wq_added=ws[0], wk_added=ws[1], n_added=n_a)
    c = R.Checker(f"rmsnorm_rope_bwd H{H} B{B} S{S} n_added{n_a} {layout}")
    dims = ("b", "token", "head", "col")
    for i, nm in enumerate(("dq", "dk")):
        emu, fl, mth = grads[i]
        out = dbuf[:, :, i * d:(i + 1) * d].unflatten(-1, (H, 128))
        c.bf16(nm, out, emu, fl, math_ref=mth, rel_l2_max=1e-2, dims=dims, **TH)
    _outside(c, "dq/dk", dbuf, before, (slice(None), slice(None), slice(0, 2 * d)))
    # weight sets that no token uses have an exactly zero gradient
    c.within_floor("norm weight grads", wg, wg_ref, wg_fl.clamp_min(1e-30), max_ratio=1.0, dims=("set", "col"))
    c.finish()


# ---------------------------------------------------------------------------------------------------- gates
GATE_CASES = [(D, rows) for D in (8, 1016, 1024, 1032, 3072) for rows in (1, 33)]
GATE_CASES += [(1024, 31), (1024, 32), (1032, 2336), (3072, 2336)]


@pytest.mark.parametrize("D,rows", GATE_CASES)
def test_gate_resid_and_gate_bwd_edges(D, rows):
    from gpt_image_edit_b200 import train_ops as T

    B = 2
    split = rows // 2 + 3 if rows > 4 else 0           # inside a 32-row chunk
    if split:
        assert split % 32 not in (0, 31)
    if D > 1024:
        assert (D + 1023) // 1024 >= 2                 # a second column block in y
    g = _g(D * 3 + rows)
    x = _bf(B, rows, D + 16, g=g)[:, :, 8:8 + D]
    y = _bf(B, rows, D + 16, g=g)[:, :, :D]
    dout = _bf(B, rows + 1, D + 8, g=g)[:, 1:, :D]
    mod = _bf(B, 6 * D, g=g, scale=0.5)
    ga, gb = mod[:, 2 * D:3 * D], mod[:, 5 * D:]
    kw = dict(gate_b=gb, split_row=split) if split else {}
    c = R.Checker(f"gate D{D} rows{rows} split{split}")
    buf = _nan(B, rows + 1, D + 16)
    before = buf.clone()
    region = (slice(None), slice(1, None), slice(8, 8 + D))
    T.gate_resid(x, y, ga, out=buf[region], **kw)
    c.equal("gate_resid", buf[region].double(), RR.gate_resid_emu(x, y, ga, **kw))
    _outside(c, "gate_resid", buf, before, region)
    buf = _nan(B, rows + 1, D + 16)
    before = buf.clone()
    dy, col = T.gate_bwd(dout, y=y, gate=ga, part_row0=split, dy=buf[region], **kw)
    dy_e, (col_ref, col_fl) = RR.gate_bwd_emu(dout, y=y, gate=ga, part_row0=split, **kw)
    c.equal("gate_bwd dy", dy.double(), dy_e)
    _outside(c, "gate_bwd dy", buf, before, region)
    c.within_floor("dgate", col, col_ref, col_fl, max_ratio=1.0, dims=("b", "col"))
    # y = None: plain column sum (bias gradient), no dy
    none_dy, cs = T.gate_bwd(dout, want_dy=False, part_row0=split)
    _, (cs_ref, cs_fl) = RR.gate_bwd_emu(dout, part_row0=split)
    assert none_dy is None
    c.within_floor("colsum", cs, cs_ref, cs_fl, max_ratio=1.0, dims=("b", "col"))
    c.finish()


def test_bias_gradient_over_batch_and_accumulating_col_reduce():
    """The bias-gradient form: partials of B items reduced as one batch of B * chunks (flux_train.cu bias_grad), and
    col_reduce accumulating into one block of a 6d-pitched fp32 dmod row."""
    from gpt_image_edit_b200 import _lib as L, train_ops as T

    g = _g(77)
    B, rows, D = 3, 77, 1032
    dout = _bf(B, rows, D, g=g)
    nch = int(L.lib.b2f_train_chunks(rows))
    part = torch.full((B, nch, D), math.nan, device="cuda", dtype=F32)
    L.check(L.lib.b2f_gate_bwd(L.ptr(dout), dout.stride(1), dout.stride(0), None, 0, 0, None, None, 0, None, 0, 0,
                               L.ptr(part), B, rows, D, 0, 0, L.stream_ptr()), "gate_bwd")
    bias = torch.randn(1, D, device="cuda", generator=g)
    old = bias.clone()
    L.check(L.lib.b2f_col_reduce(L.ptr(part), B * nch, D, L.ptr(bias), D, 1, 1, L.stream_ptr()), "col_reduce")
    ref, fl = RR.col_reduce_emu(part.reshape(1, B * nch, D), old)
    c = R.Checker(f"bias grad B{B} rows{rows} D{D}")
    c.within_floor("bias grad", bias, ref, fl, max_ratio=1.0, dims=("b", "col"))
    tot = R.d64(dout).sum((0, 1))
    c.within_floor("bias grad vs sum", bias[0] - old[0], tot, (B * rows + nch + 2) * R.U32 * R.d64(dout).abs().sum((0, 1))
                   + R.U32 * R.d64(bias[0]).abs() * 2, max_ratio=1.0)
    # accumulate into the gate block of a [B, 6D] dmod row
    dmod = torch.randn(B, 6 * D, device="cuda", generator=g)
    before = dmod.clone()
    _, col = T.gate_bwd(dout, want_dy=False, col_out=dmod[:, 2 * D:3 * D], accumulate=True)
    _, (cs, cs_fl) = RR.gate_bwd_emu(dout)
    c.within_floor("accumulated", col, R.d64(before[:, 2 * D:3 * D]) + cs,
                   cs_fl + 2 * R.U32 * (R.d64(before[:, 2 * D:3 * D]).abs() + cs.abs()), max_ratio=1.0, dims=("b", "col"))
    _outside(c, "dmod", dmod, before, (slice(None), slice(2 * D, 3 * D)))
    c.finish()


# ---------------------------------------------------------------------------------------------------- ln_modulate_bwd
LNB_CASES = [(D, rows, sp, mode) for D in (256, 2048, 3072) for rows, sp, mode in
             ((1, 0, "none"), (15, 0, "separate"), (17, 0, "aliased"))]
LNB_CASES += [(3072, 16, 0, "separate"), (256, 2336, 24, "aliased"), (3072, 2336, 24, "aliased"),
              (2048, 2336, 24, "none")]


@pytest.mark.parametrize("D,rows,split,mode", LNB_CASES)
def test_ln_modulate_bwd_edges(D, rows, split, mode):
    from gpt_image_edit_b200 import train_ops as T

    if D == 3072:
        assert D > 256 * 8                      # phase 2 covers 2048 columns per pass: a second pass runs
    B = 2
    g = _g(D + rows * 3)
    x = _bf(B, rows, D + 8, g=g, scale=2.0, shift=0.5)[:, :, :D]
    dy = _bf(B, rows, D, g=g)
    mod = _bf(B, 6 * D, g=g, scale=0.3)
    sc, scb = mod[:, D:2 * D], mod[:, 4 * D:5 * D]
    kw = dict(scale_b=scb, split_row=split) if split else {}
    buf = _nan(B, rows + 1, D + 16)
    region = (slice(None), slice(1, None), slice(8, 8 + D))
    dres = None
    if mode == "separate":
        dres = _bf(B, rows, D, g=g)
    elif mode == "aliased":                     # flux_train.cu: the residual gradient is updated in place
        buf[region] = _bf(B, rows, D, g=g)
        dres = buf[region]
    (emu, fl, mth), (ds, ds_fl), (dh, dh_fl) = RR.ln_modulate_bwd_emu(
        x, dy, sc, part_row0=split, dres=None if dres is None else dres.clone(), **kw)
    before = buf.clone()
    out, dscale, dshift = T.ln_modulate_bwd(x, dy, sc, part_row0=split, dres=dres, out=buf[region], **kw)
    c = R.Checker(f"ln_modulate_bwd D{D} rows{rows} split{split} dres={mode}")
    c.bf16("dres_out", out, emu, fl, math_ref=mth, rel_l2_max=1e-2, dims=("b", "row", "col"), **TH)
    c.within_floor("dscale", dscale, ds, ds_fl, max_ratio=1.0, dims=("b", "col"))
    c.within_floor("dshift", dshift, dh, dh_fl, max_ratio=1.0, dims=("b", "col"))
    _outside(c, "dres_out", buf, before, region)
    c.finish()


def test_ln_modulate_bwd_final_norm_image_rows():
    """The final norm: only the image rows [S_txt, S) of a [B, S, D] buffer, scale_b None, no residual gradient."""
    from gpt_image_edit_b200 import train_ops as T

    g = _g(91)
    B, S_txt, S, D = 2, 40, 340, 3072
    xb = _bf(B, S, D, g=g, scale=2.0)
    dyb = _bf(B, S, D, g=g)
    x, dy = xb[:, S_txt:], dyb[:, S_txt:]
    sc = _bf(B, 2 * D, g=g, scale=0.3)[:, :D]
    buf = _nan(B, S, D)
    before = buf.clone()
    region = (slice(None), slice(S_txt, None), slice(None))
    out, dscale, dshift = T.ln_modulate_bwd(x, dy, sc, out=buf[region])
    (emu, fl, mth), (ds, ds_fl), (dh, dh_fl) = RR.ln_modulate_bwd_emu(x, dy, sc)
    c = R.Checker(f"ln_modulate_bwd final norm B{B} rows{S - S_txt} of {S}")
    c.bf16("dx", out, emu, fl, math_ref=mth, rel_l2_max=1e-2, dims=("b", "row", "col"), **TH)
    c.within_floor("dscale", dscale, ds, ds_fl, max_ratio=1.0, dims=("b", "col"))
    c.within_floor("dshift", dshift, dh, dh_fl, max_ratio=1.0, dims=("b", "col"))
    _outside(c, "dx", buf, before, region)
    c.finish()


# ---------------------------------------------------------------------------------------------------- small training kernels
def test_gelu_rows_on_single_block_views():
    """The single block's MLP: pre-activations in columns [3d, 7d) of the fused projection, outputs into [d, 5d)."""
    from gpt_image_edit_b200 import train_ops as T

    g = _g(5)
    rows, d = 37, 256
    src = _bf(rows, 7 * d, g=g)
    src[:, 3 * d:] = (torch.rand(rows, 4 * d, device="cuda", generator=g) * 20 - 10).to(BF)
    src[0, 3 * d:3 * d + 2] = torch.tensor([-10.0, 10.0], device="cuda").to(BF)
    buf = _nan(rows, 5 * d)
    before = buf.clone()
    T.gelu(src[:, 3 * d:], out=buf[:, d:])
    emu, fl, mth = RR.gelu_rows_emu(src[:, 3 * d:])
    c = R.Checker("gelu_rows 7d -> 5d")
    c.bf16("y", buf[:, d:], emu, fl, math_ref=mth, rel_l2_max=1e-2, dims=("row", "col"), **TH)
    _outside(c, "y", buf, before, (slice(None), slice(d, None)))
    c.finish()


@pytest.mark.parametrize("B,N,K", [
    (1, 18432, 3072),     # the AdaLN linear of a double block: 6d rows of the weight, d = 3072 inputs
    (3, 18432, 3072),
    (3, 24, 18432),       # K / 4 = 4608 = 18 whole 256-thread blocks
    (2, 40, 1028),        # K / 4 = 257: one thread in the last block
])
def test_outer_acc_edges(B, N, K):
    from gpt_image_edit_b200 import train_ops as T

    g = _g(B * N + K)
    dmod = torch.randn(B, 6 * N, device="cuda", generator=g)[:, N:2 * N]
    act = _bf(B, K + 64, g=g)[:, :K]
    c = R.Checker(f"outer_acc B{B} N{N} K{K}")
    dw = T.outer_acc(dmod, act)
    ref, fl = RR.outer_acc_emu(dmod, act)
    c.within_floor("dW", dw, ref, fl, max_ratio=1.0, dims=("n", "k"))
    old = dw.clone()
    T.outer_acc(dmod, act, out=dw, accumulate=True)
    ref, fl = RR.outer_acc_emu(dmod, act, old)
    c.within_floor("dW accumulated", dw, ref, fl, max_ratio=1.0, dims=("n", "k"))
    c.finish()


@pytest.mark.parametrize("S", [1, 127, 128, 129])
def test_attn_delta_edges(S):
    from gpt_image_edit_b200 import _lib as L, train_ops as T

    g = _g(S)
    B, H = 2, 3
    d = H * 128
    ob = _bf(B * S, 5 * d, g=g)                 # attention output inside the single block's [attn | mlp] rows
    o = ob[:, :d]
    do = _bf(B * S, d, g=g)
    sp = T.s_pad(S)
    delta = torch.full((B, H, sp), math.nan, device="cuda", dtype=F32)
    lse = torch.randn(B, H, sp, device="cuda", generator=g)
    before = lse.clone()
    L.check(L.lib.b2f_attn_delta(L.ptr(o), o.stride(0), L.ptr(do), do.stride(0), L.ptr(delta), L.ptr(lse), B, H, S, sp,
                                 L.stream_ptr()), "attn_delta")
    ref, fl = RR.attn_delta_emu(o, do, B, H, S)
    c = R.Checker(f"attn_delta S{S}")
    c.within_floor("delta", delta[..., :S], ref, fl, max_ratio=1.0, dims=("b", "h", "s"))
    c.equal("padding delta == 0", delta[..., S:], torch.zeros_like(delta[..., S:]))
    c.equal("padding lse == +inf", lse[..., S:], torch.full_like(lse[..., S:], math.inf))
    c.equal("lse rows untouched", lse[..., :S], before[..., :S])
    c.finish()


# ---------------------------------------------------------------------------------------------------- timestep embedding, cast
def test_temb_sinusoid_edges():
    """Timesteps of the denoising loop (sigma * 1000) and of the guidance embedding, up to t = 1000, where the fp32
    angle t f carries the largest absolute error."""
    from gpt_image_edit_b200 import _lib as L

    t = torch.tensor([0.0, 1e-3, 0.5, 1.0, 3.5, 37.25, 500.0, 731.5, 999.0, 999.75, 1000.0], device="cuda")
    rows = t.numel()
    out = _nan(rows + 1, 256)
    L.check(L.lib.b2f_temb_sinusoid(L.ptr(t), L.ptr(out), rows, L.stream_ptr()), "temb_sinusoid")
    emu, fl, mth = RR.temb_sinusoid_emu(t)
    c = R.Checker(f"temb_sinusoid rows{rows}")
    c.bf16("[cos | sin]", out[:rows], emu, fl, math_ref=mth, rel_l2_max=1e-2, dims=("row", "col"), **TH)
    c.equal("past the last row", out[rows].view(torch.int16), _nan(256).view(torch.int16))
    c.finish()


@pytest.mark.parametrize("n", [8, 3072 * 3, 2056 * 128 + 8])
def test_silu_and_temb_combine_edges(n):
    from gpt_image_edit_b200 import _lib as L

    g = _g(n)
    x = _bf(n, g=g, scale=6.0)
    x[:2] = torch.tensor([-20.0, 20.0], device="cuda").to(BF)
    c = R.Checker(f"silu / temb_combine n{n}")
    y = _nan(n + 8)
    L.check(L.lib.b2f_silu(L.ptr(x), L.ptr(y), n, L.stream_ptr()), "silu")
    emu, fl, mth = RR.silu_emu(x)
    c.bf16("silu", y[:n], emu, fl, math_ref=mth, rel_l2_max=1e-2, dims=("i",), **TH)
    c.equal("silu past n", y[n:].view(torch.int16), _nan(8).view(torch.int16))
    tt, gg, txt = _bf(n, g=g, scale=2.0), _bf(n, g=g, scale=2.0), _bf(n, g=g, scale=2.0)
    for with_g in (True, False):
        temb, st = _nan(n + 8), _nan(n + 8)
        L.check(L.lib.b2f_temb_combine(L.ptr(tt), L.ptr(gg) if with_g else None, L.ptr(txt), L.ptr(temb), L.ptr(st), n,
                                       L.stream_ptr()), "temb_combine")
        te, (se, sf, sm) = RR.temb_combine_emu(tt, gg if with_g else None, txt)
        c.equal(f"temb g={with_g}", temb[:n].double(), te)
        c.bf16(f"silu_temb g={with_g}", st[:n], se, sf, math_ref=sm, rel_l2_max=1e-2, dims=("i",), **TH)
        c.equal(f"g={with_g} past n", torch.cat([temb[n:], st[n:]]).view(torch.int16), _nan(16).view(torch.int16))
    c.finish()


@pytest.mark.parametrize("n", [1, 7, 4099, 5_000_003])
@pytest.mark.parametrize("offset", [0, 1])
def test_cast_edges(n, offset):
    from gpt_image_edit_b200 import train_ops as T

    if n > 5_000_000 and not offset:
        assert n // 8 > min((n + 255) // 256, ADAMW_MAX_BLOCKS) * 256     # the vector loop strides more than once
    g = _g(n + offset)
    src = (torch.randn(n + 2, device="cuda", generator=g) * torch.exp(torch.randn(n + 2, device="cuda", generator=g) * 4))
    src = src[offset:offset + n]                     # offset by one element: the scalar path
    c = R.Checker(f"cast n{n} offset{offset}")
    b = T.cast(src, BF)
    c.equal("fp32 -> bf16", b.double(), RR.cast_emu(src, False))
    b16 = _bf(n + 2, g=g, scale=100.0)[offset:offset + n]
    f = T.cast(b16, F32)
    c.equal("bf16 -> fp32", f.double(), RR.cast_emu(b16, True))
    c.finish()


# ---------------------------------------------------------------------------------------------------- loss, norm, optimizer
@pytest.mark.parametrize("n", [1, 255, 257, 300_000])
@pytest.mark.parametrize("weighted", [False, True])
def test_mse_loss_edges(n, weighted):
    from gpt_image_edit_b200 import train_ops as T

    blocks = max(1, min(n // 256, 1024))
    if n == 300_000:
        assert n > blocks * 256                 # a second pass of the grid-stride loop
    g = _g(n + weighted)
    pred = _bf(n, g=g)
    target = torch.randn(n, device="cuda", generator=g)
    w = torch.rand(n, device="cuda", generator=g) * 2 if weighted else None
    loss, dpred = T.mse_loss(pred, target, weight=w, grad_scale=0.7)
    (lr, lf), (emu, fl, mth) = RR.mse_loss_emu(pred, target, w, grad_scale=0.7)
    c = R.Checker(f"mse_loss n{n} weighted={weighted}")
    c.within_floor("loss", loss, lr.reshape(1), lf.reshape(1), max_ratio=1.0)
    c.bf16("dpred", dpred, emu, fl, math_ref=mth, rel_l2_max=1e-2, dims=("i",), **TH)
    c.finish()


ADAMW_MAX_BLOCKS = 148 * 16          # grid cap of adamw_step and cast_bf16_f32 (train_kernels.cu)
OPT_N = [1, 5, 100_003, 4 * 2 ** 20 + 3]


@pytest.mark.parametrize("n", OPT_N)
@pytest.mark.parametrize("offset", [0, 1])
def test_grad_sumsq_edges(n, offset):
    from gpt_image_edit_b200 import train_ops as T

    blocks = RR.sumsq_blocks(n)
    if n > 4_000_000 and not offset:
        assert n // 4 > 3 * blocks * 256        # the 4-deep unrolled loop runs
    g = _g(n + offset)
    buf = torch.randn(n + 4, device="cuda", generator=g) * 3
    x = buf[offset:offset + n]                   # offset by one float: the scalar path
    ss = T.grad_sumsq(x)
    ref, fl = RR.grad_sumsq_emu(x)
    c = R.Checker(f"grad_sumsq n{n} offset{offset}")
    c.within_floor("sumsq", ss, ref.reshape(1), fl.reshape(1), max_ratio=1.0)
    old = ss.clone()
    T.grad_sumsq(x, out=ss, accumulate=True)
    ref, fl = RR.grad_sumsq_emu(x, old)
    c.within_floor("sumsq accumulated", ss, ref.reshape(1), fl.reshape(1) * 2, max_ratio=1.0)
    c.finish()


@pytest.mark.parametrize("max_norm,rel", [(1.0, 0.5), (1.0, 1.0), (1.0, 3.0), (0.0, 3.0)])
def test_clip_coef_edges(max_norm, rel):
    from gpt_image_edit_b200 import train_ops as T

    norm = max_norm * rel if max_norm else 2.5
    ss = torch.tensor([norm * norm], device="cuda", dtype=F32)
    for pre in (1.0, 0.5):
        coef, nrm = T.clip_coef(ss, max_norm, pre)
        ce, cf, ne, nf = RR.clip_coef_emu(ss, max_norm, pre)
        c = R.Checker(f"clip_coef max_norm{max_norm} norm/max{rel} pre{pre}")
        c.within_floor("coef", coef, ce.reshape(1), cf.reshape(1), max_ratio=1.0)
        c.within_floor("norm", nrm, ne.reshape(1), nf.reshape(1), max_ratio=1.0)
        c.finish()


@pytest.mark.parametrize("n", OPT_N)
@pytest.mark.parametrize("variant", ["plain", "p16+gscale", "offset", "step1000"])
def test_adamw_edges(n, variant):
    from gpt_image_edit_b200 import train_ops as T

    if n > 4_000_000 and variant != "offset":
        blocks = min((n + 255) // 256, ADAMW_MAX_BLOCKS)
        assert n // 4 > blocks * 256            # the second in-flight float4 (on[1]) is enabled
    g = _g(n * 3 + len(variant))
    off = 1 if variant == "offset" else 0
    mk = lambda s: (torch.randn(n + 4, device="cuda", generator=g) * s)[off:off + n]
    p, m, grad = mk(1.0), mk(0.01), mk(1.0)
    v = (torch.rand(n + 4, device="cuda", generator=g) * 1e-4)[off:off + n]
    step = 1000 if variant == "step1000" else 1
    if step == 1:
        m.zero_(), v.zero_()
    gscale = torch.tensor([0.37], device="cuda") if variant == "p16+gscale" else None
    p16 = torch.full((n,), math.nan, device="cuda", dtype=BF) if variant == "p16+gscale" else None
    kw = dict(lr=1e-3, betas=(0.9, 0.95), eps=1e-8, step=step)
    (pr, pf), (mr, mf), (vr, vf) = RR.adamw_emu(p, m, v, grad, wd=0.05, gscale=gscale, **kw)
    T.adamw_step_(p, m, v, grad, p16=p16, weight_decay=0.05, gscale=gscale, **kw)
    c = R.Checker(f"adamw n{n} {variant}")
    c.within_floor("p32", p, pr, pf, max_ratio=1.0, dims=("i",))
    c.within_floor("m", m, mr, mf.clamp_min(1e-30), max_ratio=1.0, dims=("i",))
    c.within_floor("v", v, vr, vf.clamp_min(1e-30), max_ratio=1.0, dims=("i",))
    if p16 is not None:
        c.equal("p16 == bf16(p32)", p16.view(torch.int16), p.to(BF).view(torch.int16))
    c.finish()


# ---------------------------------------------------------------------------------------------------- LLM / text encoders
@pytest.mark.parametrize("D", [1280, 1536, 3584, 3840])
def test_rmsnorm_edges(D):
    from gpt_image_edit_b200 import ops

    g = _g(D)
    rows = 7
    x = _bf(rows, D + 64, g=g, scale=2.0, shift=0.5)[:, :D]
    w = _bf(D, g=g, scale=0.3, shift=1.0)
    buf = _nan(rows, D + 16)
    before = buf.clone()
    ops.rmsnorm(x, w, out=buf[:, :D])
    emu, fl, mth = RR.rmsnorm_emu(x, w)
    c = R.Checker(f"rmsnorm D{D}")
    c.bf16("y", buf[:, :D], emu, fl, math_ref=mth, rel_l2_max=1e-2, dims=("row", "col"), **TH)
    _outside(c, "y", buf, before, (slice(None), slice(0, D)))
    c.finish()


@pytest.mark.parametrize("D", [768, 1280, 1536])
def test_layernorm_edges(D):
    from gpt_image_edit_b200 import ops

    g = _g(D + 1)
    rows = 9
    x = _bf(rows, D, g=g, scale=1.0, shift=20.0)         # a DC offset: 20 x std
    w, b = _bf(D, g=g, scale=0.3, shift=1.0), _bf(D, g=g, scale=0.3)
    buf = _nan(rows, D + 16)
    before = buf.clone()
    ops.layernorm(x, w, b, out=buf[:, :D])
    emu, fl, mth = RR.layernorm_emu(x, w, b)
    c = R.Checker(f"layernorm D{D}")
    c.bf16("y", buf[:, :D], emu, fl, math_ref=mth, rel_l2_max=1e-2, dims=("row", "col"), **TH)
    _outside(c, "y", buf, before, (slice(None), slice(0, D)))
    c.finish()


@pytest.mark.parametrize("path", ["vision", "text"])
def test_rope_half_layouts(path):
    """The ViT layout (2 nh heads of 80 then V) and the text decoder's (nq + nkv heads of 128 then V)."""
    from gpt_image_edit_b200 import ops

    g = _g(len(path))
    if path == "vision":
        heads, hp, tokens, width = 2 * 16, 80, 37, 3 * 16 * 80
    else:
        heads, hp, tokens, width = 28 + 4, 128, 21, (28 + 2 * 4) * 128
    x = _bf(tokens, width, g=g, scale=2.0)
    ang = torch.rand(tokens, hp // 2, device="cuda", generator=g) * 50
    cos = torch.cat([torch.cos(ang)] * 2, -1)
    sin = torch.cat([torch.sin(ang)] * 2, -1)
    if path == "text":                                    # the text tables are bf16 values
        cos, sin = cos.to(BF).float(), sin.to(BF).float()
    emu, fl, mth = RR.rope_half_emu(x, heads, hp, cos, sin, fp32_math=path == "vision")
    y = x.clone()
    ops.rope_half_(y, heads, hp, cos, sin, fp32_math=path == "vision")
    c = R.Checker(f"rope_half {path}")
    rot = heads * hp
    if path == "vision":
        c.bf16("rotated", y[:, :rot], emu[:, :rot], fl[:, :rot], math_ref=mth[:, :rot], rel_l2_max=1e-2,
               dims=("token", "col"), **TH)
    else:
        c.equal("rotated (bf16 chain)", y[:, :rot].double(), emu[:, :rot])
    c.equal("V untouched", y[:, rot:].view(torch.int16), x[:, rot:].view(torch.int16))
    c.finish()


@pytest.mark.parametrize("inter", [344, 18944])
def test_swiglu_geglu_edges(inter):
    from gpt_image_edit_b200 import ops

    g = _g(inter)
    rows = 5 if inter > 1000 else 33
    gu = _bf(rows, 2 * inter + 8, g=g, scale=3.0)[:, :2 * inter]
    c = R.Checker(f"gated I{inter}")
    for name, fn, ref in (("swiglu", ops.swiglu, RR.swiglu_emu), ("geglu", ops.geglu, RR.geglu_emu)):
        buf = _nan(rows, inter + 8)
        before = buf.clone()
        fn(gu, inter, out=buf[:, :inter])
        emu, fl, mth = ref(gu, inter)
        c.bf16(name, buf[:, :inter], emu, fl, math_ref=mth, rel_l2_max=1e-2, dims=("row", "col"), **TH)
        _outside(c, name, buf, before, (slice(None), slice(0, inter)))
    c.finish()


# ---------------------------------------------------------------------------------------------------- VAE
@pytest.mark.parametrize("C", [32, 128, 256, 512])
@pytest.mark.parametrize("P", [1, 511, 513, 20000])
def test_groupnorm_silu_edges(C, P):
    from gpt_image_edit_b200 import _lib as L

    N = 2
    g = _g(C + P)
    x = _bf(N, P, C, g=g, scale=2.0)
    x[1] += 24.0                                          # item 1 with a DC offset of 12 x std
    x = x.to(BF)
    ga, be = _bf(C, g=g, scale=0.2, shift=1.0), _bf(C, g=g, scale=0.2)
    c = R.Checker(f"groupnorm N{N} P{P} C{C}")
    for silu in (1, 0):
        y = torch.full((N, P + 1, C), math.nan, device="cuda", dtype=BF)
        stats = torch.empty(64 * N, device="cuda", dtype=torch.float64)
        L.check(L.lib.b2f_groupnorm_silu(L.ptr(x), L.ptr(ga), L.ptr(be), L.ptr(y), L.ptr(stats), N, P, C, 1e-6, silu,
                                         L.stream_ptr()), "gn")
        yv = y.view(-1)[:N * P * C].view(N, P, C)
        emu, fl, mth = RR.groupnorm_silu_emu(x, ga, be, silu_on=bool(silu))
        c.bf16(f"y silu={silu}", yv, emu, fl, math_ref=mth, rel_l2_max=1e-2, dims=("n", "p", "c"), **TH)
        c.equal(f"silu={silu} past the end", y.view(-1)[N * P * C:].view(torch.int16),
                torch.full((C * N,), math.nan, device="cuda", dtype=BF).view(torch.int16))
    c.finish()


# ragged L (the VAE's mid-block attention over P = 13 x 21 and 90 x 182 latent pixels) and its 1024^2 row, L = 16384
@pytest.mark.parametrize("L_", [8, 2056, 273, 16380, 16384])
def test_softmax_rows_edges(L_):
    from gpt_image_edit_b200 import _lib as L

    g = _g(L_)
    rows = 5
    L8 = -(-L_ // 8) * 8
    s = _bf(rows, L8 + 8, g=g, scale=4.0)                 # pitch ld = L8 + 8: one vector past the padded row
    x = s[:, :L_].clone()
    before = s.clone()
    L.check(L.lib.b2f_softmax_rows(L.ptr(s), s.stride(0), rows, L_, 512 ** -0.5, L.stream_ptr()), "softmax")
    emu, fl, mth = RR.softmax_rows_emu(x, 512 ** -0.5)
    c = R.Checker(f"softmax_rows L{L_}")
    c.bf16("p", s[:, :L_], emu, fl, math_ref=mth, rel_l2_max=1e-2, dims=("row", "col"), **TH)
    c.equal("p: zeroed tail [L, round_up(L, 8))", s[:, L_:L8].view(torch.int16), torch.zeros_like(s[:, L_:L8]).view(torch.int16))
    _outside(c, "p", s, before, (slice(None), slice(0, L8)))
    c.finish()
    # the pitch must be a multiple of 8 and hold the padded row
    for ld in (L8 - 8, L8 + 4):
        if ld > 0 and ld != L8:
            assert L.lib.b2f_softmax_rows(L.ptr(s), ld, 1, L_, 1.0, L.stream_ptr()) != 0, f"ld {ld} accepted"


# fp32 scores in, bf16 probabilities out (the VAE's mid-block attention, whose logits are never rounded to bf16)
@pytest.mark.parametrize("L_", [8, 273, 16380, 16384])
def test_softmax_rows_f32_edges(L_):
    from gpt_image_edit_b200 import _lib as L

    g = _g(L_ + 1)
    rows = 5
    L8 = -(-L_ // 8) * 8
    s = torch.randn(rows, L8 + 8, device="cuda", generator=g) * 90.0      # unscaled logits of std 4 after 512^-0.5
    s_before = s.clone()
    p = torch.full((rows, L8 + 16), math.nan, device="cuda", dtype=BF)
    before = p.clone()
    L.check(L.lib.b2f_softmax_rows_f32(L.ptr(s), s.stride(0), L.ptr(p), p.stride(0), rows, L_, 512 ** -0.5,
                                       L.stream_ptr()), "softmax f32")
    emu, fl, mth = RR.softmax_rows_emu(s[:, :L_], 512 ** -0.5)
    c = R.Checker(f"softmax_rows_f32 L{L_}")
    c.bf16("p", p[:, :L_], emu, fl, math_ref=mth, rel_l2_max=1e-2, dims=("row", "col"), **TH)
    c.equal("p: zeroed tail [L, round_up(L, 8))", p[:, L_:L8].view(torch.int16), torch.zeros_like(p[:, L_:L8]).view(torch.int16))
    _outside(c, "p", p, before, (slice(None), slice(0, L8)))
    c.equal("s untouched", s.view(torch.int32), s_before.view(torch.int32))
    c.finish()
