"""The persistent ping-pong GEMM (gemm.cu) on shapes where CTAs run several tiles, element by element against the fp64
references of kernel_ref.py.

The kernel launches min(tiles, SMs) CTAs; CTA b runs tiles b, b + grid, ... and its two consumer warpgroups alternate
between them, while the producer streams k-blocks through a 4-stage ring across tile boundaries.  The shapes are chosen
from the SM count of the device under test so that:
  - every CTA runs at least 3 tiles and its two consumers run different numbers of tiles (3 = 2 + 1), or the grid is
    smaller than the SM count (1 tile; SMs + 1 tiles, where only CTA 0 runs a second tile);
  - the number of k-blocks per tile is not a multiple of the 4 ring stages, so a tile starts at a different ring slot
    and phase than the one before it; and K = 64 (one k-block per tile: the turn-taking and the staging tile reuse are
    all there is);
  - one CTA's tile list crosses batch items, n-panels (16 n-blocks) and the [Q|K|V | MLP] split of the single-block
    launch.
Outputs are views into NaN-filled buffers: every element of the view must be written, nothing outside it.
"""
import pytest
import torch

import kernel_ref as R

pytestmark = pytest.mark.gpu

TH_GEMM = dict(max_ulp=2, share_gt1=1e-3, mean_ulp=0.1)   # as in test_sm90_edges_gpu.py


def _g(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _bf(*shape, g, scale=1.0, shift=0.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale + shift).bfloat16()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cdiv(a, b):
    return -(-a // b)


def _n_blocks_for(m_blocks, min_tiles):
    """n-blocks such that m_blocks x n_blocks >= min_tiles."""
    return _cdiv(min_tiles, m_blocks)


def _nan_view(shape, dtype=torch.bfloat16, pad_rows=3, pad_cols=16):
    """(buffer, view): a NaN-filled buffer one row and pad_cols / 2 columns larger on each side than `shape`."""
    *lead, rows, cols = shape
    buf = torch.full((*lead, rows + pad_rows, cols + pad_cols), float("nan"), device="cuda", dtype=dtype)
    c0 = pad_cols // 2
    return buf, buf[..., 1:1 + rows, c0:c0 + cols]


def _outside_untouched(c, buf, view_slices, what="outside the view"):
    mask = torch.ones_like(buf, dtype=torch.bool)
    mask[view_slices] = False
    c.equal(what + " (still NaN)", torch.isnan(buf[mask]), torch.ones_like(buf[mask], dtype=torch.bool))


def _slices(buf, rows, cols, pad_cols=16):
    c0 = pad_cols // 2
    return (Ellipsis, slice(1, 1 + rows), slice(c0, c0 + cols))


def _tile_counts(tiles):
    """(grid, tiles of the busiest CTA, tiles of the least busy CTA) of the persistent launch."""
    grid = min(tiles, _sms())
    return grid, _cdiv(tiles, grid), tiles // grid


# ---------------------------------------------------------------------------------------------------- forward
def _many_tile_shapes():
    S = _sms()
    n_blk = 17                                  # a panel of 16 n-blocks, then a 1-wide panel
    m_blk = _cdiv(3 * S, n_blk) + 1             # >= 3 tiles per CTA, fewer than 4 * S tiles
    return [
        (m_blk * 128 - 51, n_blk * 128, 328),   # 6 k-blocks (8-wide tail): tiles start at ring slots 0, 2, 0, ...
        (m_blk * 128 - 51, n_blk * 128, 64),    # one k-block per tile
        (100, 8, 72),                           # 1 tile
        (128, (S + 1) * 128 - 64, 200),         # S + 1 tiles: only CTA 0 runs a second one (last n-block 64 wide)
    ]


@pytest.mark.parametrize("case", range(4))
def test_gemm_many_tiles_per_cta(case):
    from gpt_image_edit_b200 import ops

    M, N, K = _many_tile_shapes()[case]
    tiles = _cdiv(M, 128) * _cdiv(N, 128)
    grid, hi, lo = _tile_counts(tiles)
    if case < 2:   # >= 3 tiles per CTA, and some CTA runs an odd number: its consumers run different counts
        assert lo >= 3 and (lo % 2 == 1 or hi % 2 == 1), (tiles, grid)
    g = _g(100 + case)
    x, w, b = _bf(M, K, g=g), _bf(N, K, g=g, scale=K ** -0.5), _bf(N, g=g, scale=0.5)
    buf, out = _nan_view((M, N))
    ops.linear(x, w, b, out=out)
    emu, floor, acc = R.linear_emu(x, w, b)
    c = R.Checker(f"gemm M{M} N{N} K{K} tiles={tiles} grid={grid} per-CTA {lo}..{hi}")
    c.bf16("out", out, emu, floor, math_ref=acc, rel_l2_max=4e-3, dims=("row", "col"), **TH_GEMM)
    _outside_untouched(c, buf, _slices(buf, M, N))
    c.finish()


def test_gemm_batch_boundaries_inside_cta():
    """B = 5 batch items of 2 ragged m-blocks each: consecutive tiles of a CTA change batch item mid-list."""
    from gpt_image_edit_b200 import ops

    S = _sms()
    B, M, K = 5, 130, 392                     # 7 k-blocks
    m_blocks = B * 2
    N = _n_blocks_for(m_blocks, 3 * S + 1) * 128
    g = _g(7)
    x, w, b = _bf(B, M, K, g=g), _bf(N, K, g=g, scale=K ** -0.5), _bf(N, g=g, scale=0.5)
    buf, out = _nan_view((B, M, N))
    ops.linear(x, w, b, out=out)
    emu, floor, acc = R.linear_emu(x, w, b)
    c = R.Checker(f"gemm B{B} M{M} N{N} K{K}")
    c.bf16("out", out, emu, floor, math_ref=acc, rel_l2_max=4e-3, dims=("b", "row", "col"), **TH_GEMM)
    _outside_untouched(c, buf, _slices(buf, M, N))
    c.finish()


@pytest.mark.parametrize("epi", [R.EPI_BIAS, R.EPI_GELU_TANH, R.EPI_GELU_ERF, R.EPI_SILU, R.EPI_QUICK_GELU,
                                 R.EPI_GATE_RESID, R.EPI_RESID])
@pytest.mark.parametrize("K", [64, 136])
def test_gemm_epilogues_many_tiles(epi, K):
    """Every forward epilogue with >= 3 tiles per CTA, batched; the residual epilogues in place (resid aliases out)."""
    from gpt_image_edit_b200 import ops

    S = _sms()
    B, M = 2, 300                               # 3 m-blocks per batch item, the last 44 rows
    N = _n_blocks_for(B * 3, 3 * S + 1) * 128
    g = _g(200 + epi + K)
    x, w, b = _bf(B, M, K, g=g), _bf(N, K, g=g, scale=K ** -0.5 * 2), _bf(N, g=g, scale=0.5)
    resid, gate = _bf(B, M, N, g=g), _bf(B, N, g=g)
    buf, out = _nan_view((B, M, N))
    if epi in (R.EPI_GATE_RESID, R.EPI_RESID):
        out.copy_(resid)
        ops.linear(x, w, b, epilogue=epi, resid=out, gate=gate if epi == R.EPI_GATE_RESID else None, out=out)
    else:
        ops.linear(x, w, b, epilogue=epi, out=out)
    emu, floor, _ = R.linear_emu(x, w, b, epi, resid=resid, gate=gate)
    c = R.Checker(f"gemm epi{epi} B{B} M{M} N{N} K{K}")
    c.bf16("out", out, emu, floor, dims=("b", "row", "col"), **TH_GEMM)
    _outside_untouched(c, buf, _slices(buf, M, N))
    c.finish()


def _rope(S, g):
    ang = torch.rand(S, 64, device="cuda", generator=g) * 6.28
    return torch.cos(ang).repeat_interleave(2, 1).contiguous(), torch.sin(ang).repeat_interleave(2, 1).contiguous()


@pytest.mark.parametrize("extra", [True, False])
def test_gemm_qkv_norm_rope_many_tiles(extra):
    """[Q|K|V] (+ the GELU'd MLP block) with >= 3 tiles per CTA: 3 heads, so a CTA's tiles cross Q / K / V, the
    split at 3d (n-block 9), and the n-panel edge at n-block 16 (21 n-blocks with the MLP block)."""
    from gpt_image_edit_b200 import ops

    S = _sms()
    B, H, K, row0 = 2, 3, 320, 24
    d = H * 128
    n_extra = 4 * d if extra else 0
    n_blocks = (3 * d + n_extra) // 128
    m_per_b = _cdiv(3 * S + 1, B * n_blocks)
    M = m_per_b * 128 - 77
    g = _g(300 + extra)
    x = _bf(B, M, K, g=g)
    w, b = _bf(3 * d + n_extra, K, g=g, scale=K ** -0.5), _bf(3 * d + n_extra, g=g, scale=0.5)
    nq, nk = _bf(128, g=g, scale=0.1, shift=1.0), _bf(128, g=g, scale=0.1, shift=1.0)
    cos, sin = _rope(row0 + M + 3, g)
    buf, out = _nan_view((B, M, 3 * d))
    cat = out_extra = None
    if extra:
        cat_buf, cat = _nan_view((B, M, d + n_extra))
        out_extra = cat[:, :, d:]
    ops.linear_qkv_norm_rope(x, w, b, nq, nk, cos, sin, rope_row0=row0, out=out, out_extra=out_extra,
                             epi_extra=ops.EPI_GELU_TANH)
    emu, floor, mth = R.qkv_norm_rope_emu(x, w, b, nq, nk, cos, sin, rope_row0=row0, n_extra=n_extra,
                                          epi_extra=R.EPI_GELU_TANH)
    c = R.Checker(f"qkv_norm_rope B{B} M{M} H{H} extra={n_extra} tiles={B * m_per_b * n_blocks}")
    dims = ("b", "row", "col")
    c.bf16("Q", out[..., :d], emu[..., :d], floor[..., :d], math_ref=mth[..., :d], rel_l2_max=8e-3, dims=dims,
           **TH_GEMM)
    c.bf16("K", out[..., d:2 * d], emu[..., d:2 * d], floor[..., d:2 * d], math_ref=mth[..., d:2 * d],
           rel_l2_max=8e-3, dims=dims, **TH_GEMM)
    c.bf16("V", out[..., 2 * d:], emu[..., 2 * d:3 * d], floor[..., 2 * d:3 * d], dims=dims, **TH_GEMM)
    _outside_untouched(c, buf, _slices(buf, M, 3 * d))
    if extra:
        c.bf16("mlp", out_extra, emu[..., 3 * d:], floor[..., 3 * d:], math_ref=mth[..., 3 * d:], rel_l2_max=6e-3,
               dims=dims, **TH_GEMM)
        c.equal("attn columns of [attn|mlp] (still NaN)", torch.isnan(cat[:, :, :d]),
                torch.ones_like(cat[:, :, :d], dtype=torch.bool))
        _outside_untouched(c, cat_buf, _slices(cat_buf, M, d + n_extra), "outside [attn|mlp]")
    c.finish()


# ---------------------------------------------------------------------------------------------------- dgrad / wgrad
@pytest.mark.parametrize("epi", [R.EPI_BIAS, R.EPI_DGELU, R.EPI_DSILU, R.EPI_RESID])
def test_dgrad_many_tiles(epi):
    from gpt_image_edit_b200 import train_ops as T

    S = _sms()
    B, M, K = 2, 200, 392                       # 2 m-blocks per batch item, 7 k-blocks
    N = _n_blocks_for(B * 2, 3 * S + 1) * 128
    g = _g(400 + epi)
    dy, w = _bf(B, M, K, g=g), _bf(K, N, g=g, scale=K ** -0.5)
    aux = _bf(B, M, N, g=g, scale=2.0)
    buf, out = _nan_view((B, M, N))
    if epi == R.EPI_RESID:
        out.copy_(aux)
        T.linear_dgrad(dy, w, epilogue=epi, aux=out, out=out)
    else:
        T.linear_dgrad(dy, w, epilogue=epi, aux=None if epi == R.EPI_BIAS else aux, out=out)
    emu, floor, mth = R.dgrad_emu(dy, w, epi, aux=aux)
    c = R.Checker(f"dgrad epi{epi} B{B} M{M} N{N} K{K}")
    c.bf16("dx", out, emu, floor, math_ref=mth, rel_l2_max=6e-3, dims=("b", "row", "col"), **TH_GEMM)
    _outside_untouched(c, buf, _slices(buf, M, N))
    c.finish()


@pytest.mark.parametrize("B,rows", [(3, 150), (1, 64)])
def test_wgrad_many_tiles(B, rows):
    """fp32 weight gradient with >= 3 tiles per CTA: 3 batch items x 3 k-blocks (the last a 22-row tail) = 9 k-blocks
    per tile, or a single k-block; plain store and accumulate."""
    from gpt_image_edit_b200 import train_ops as T

    S = _sms()
    M = 17 * 128 - 24                           # 17 m-blocks, the last 104 rows
    N = _n_blocks_for(17, 3 * S + 1) * 128 - 8
    g = _g(500 + rows)
    dy, x = _bf(B, rows, M, g=g), _bf(B, rows, N, g=g)
    ref, floor = R.wgrad_math(dy, x)
    buf, dw = _nan_view((M, N), dtype=torch.float32, pad_rows=2, pad_cols=8)
    T.linear_wgrad(dy, x, out=dw)
    prior = torch.randn(M, N, device="cuda", generator=g)
    buf2, dw2 = _nan_view((M, N), dtype=torch.float32, pad_rows=2, pad_cols=8)
    dw2.copy_(prior)
    T.linear_wgrad(dy, x, out=dw2, accumulate=True)
    c = R.Checker(f"wgrad B{B} rows{rows} M{M} N{N}")
    c.within_floor("dw", dw, ref, floor, max_ratio=1.0, rel_l2_max=1e-5, dims=("m", "n"))
    c.within_floor("dw accumulate", dw2, ref + prior.double(), floor + R.U32 * (prior.double().abs() + ref.abs()),
                   max_ratio=1.0, dims=("m", "n"))
    _outside_untouched(c, buf, _slices(buf, M, N, pad_cols=8))
    _outside_untouched(c, buf2, _slices(buf2, M, N, pad_cols=8), "outside the accumulated view")
    c.finish()


# ---------------------------------------------------------------------------------------------------- toy cases
@pytest.mark.parametrize("tiles", ["1", "3", "sms+1"])
def test_gemm_toy_tile_counts(tiles):
    """Gate-residual GEMM on 1, 3 and SMs + 1 tiles of one m-block, 6 k-blocks each: small enough for the sanitizers
    (scripts/sanitize_select.py), and the last one makes CTA 0 reuse its ring and staging tile for a second tile."""
    from gpt_image_edit_b200 import ops

    n_tiles = _sms() + 1 if tiles == "sms+1" else int(tiles)
    M, N, K = 100, n_tiles * 128, 328
    g = _g(600 + n_tiles)
    x, w, b = _bf(1, M, K, g=g), _bf(N, K, g=g, scale=K ** -0.5), _bf(N, g=g, scale=0.5)
    resid, gate = _bf(1, M, N, g=g), _bf(1, N, g=g)
    buf, out = _nan_view((1, M, N))
    out.copy_(resid)
    ops.linear(x, w, b, epilogue=R.EPI_GATE_RESID, resid=out, gate=gate, out=out)
    emu, floor, _ = R.linear_emu(x, w, b, R.EPI_GATE_RESID, resid=resid, gate=gate)
    c = R.Checker(f"gemm toy M{M} N{N} K{K}")
    c.bf16("out", out, emu, floor, dims=("b", "row", "col"), **TH_GEMM)
    _outside_untouched(c, buf, _slices(buf, M, N))
    c.finish()
