"""The forward GEMM's two tiles (gemm.cu): 128 x 128 with ping-pong consumers and 128 x 256 with both consumers on one
tile.  b2f_gemm_set_tile_override forces each path, and both must give bit-identical outputs for every forward
epilogue:
  - M in {1, 127, 129, 255, 257, 544, 8736}: fewer tiles than SMs, m-block tails of 127 / 1 rows, the text rows of the
    edit and the single-block rows (69 m-blocks, an odd count);
  - N at and around the 256-column edge, so that the last wide tile is full, 8 columns wide or 248 columns wide;
  - batch 3 with M 257, so that consecutive tiles of a CTA cross batch items;
  - the fused QKV epilogue at d 3072 with the single block's [Q|K|V | MLP] split and rope_row0 > 0.
Outputs are views into NaN-filled buffers: both paths must write every element of the view and nothing outside it.
The wide path is also checked against kernel_ref's emulation, and the automatic rule against the loop's shapes.
"""
import pytest
import torch

import kernel_ref as R

pytestmark = pytest.mark.gpu

TH_GEMM = dict(max_ulp=2, share_gt1=1e-3, mean_ulp=0.1)   # as in test_sm90_edges_gpu.py
EPIS = [R.EPI_BIAS, R.EPI_GELU_TANH, R.EPI_GELU_ERF, R.EPI_SILU, R.EPI_QUICK_GELU, R.EPI_GATE_RESID, R.EPI_RESID]


@pytest.fixture(autouse=True)
def _automatic_after():
    yield
    from gpt_image_edit_b200 import _lib

    _lib.check(_lib.lib.b2f_gemm_set_tile_override(0), "b2f_gemm_set_tile_override")


def _force(tile):
    from gpt_image_edit_b200 import _lib

    _lib.check(_lib.lib.b2f_gemm_set_tile_override(tile), "b2f_gemm_set_tile_override")


def _g(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _bf(*shape, g, scale=1.0, shift=0.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale + shift).bfloat16()


def _nan_view(shape, pad_cols=16):
    """(buffer, view): a NaN-filled buffer with a row above and below and pad_cols / 2 columns on each side of `shape`."""
    *lead, rows, cols = shape
    buf = torch.full((*lead, rows + 2, cols + pad_cols), float("nan"), device="cuda", dtype=torch.bfloat16)
    c0 = pad_cols // 2
    return buf, buf[..., 1:1 + rows, c0:c0 + cols]


def _outside_nan(buf, rows, cols, pad_cols=16):
    mask = torch.ones_like(buf, dtype=torch.bool)
    mask[..., 1:1 + rows, pad_cols // 2:pad_cols // 2 + cols] = False
    return bool(torch.isnan(buf[mask]).all())


def _tags(fn):
    """Profiling tags of the GEMM launches `fn` makes (each ends in " t128" or " t256", the tile that ran)."""
    from gpt_image_edit_b200 import _lib

    _lib.prof_enable(True)
    try:
        _lib.prof_shapes()
        fn()
        tags = [t for t, *_ in _lib.prof_shapes()]
        _lib.prof_collect()
    finally:
        _lib.prof_enable(False)
    return tags


def _ran_on(tags, tile):
    assert len(tags) == 1 and tags[0].endswith(f" t{tile}"), (tile, tags)


def _linear(tile, x, w, b, epi, resid, gate):
    from gpt_image_edit_b200 import ops

    _force(tile)
    B, M, _ = x.shape
    buf, out = _nan_view((B, M, w.shape[0]))
    if epi in (R.EPI_GATE_RESID, R.EPI_RESID):
        out.copy_(resid)   # in place: resid aliases out
        fn = lambda: ops.linear(x, w, b, epilogue=epi, resid=out, gate=gate if epi == R.EPI_GATE_RESID else None,
                                out=out)
    else:
        fn = lambda: ops.linear(x, w, b, epilogue=epi, out=out)
    _ran_on(_tags(fn), tile)
    return buf, out


@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("N", [248, 256, 264, 520])
@pytest.mark.parametrize("B,M", [(1, 1), (1, 127), (1, 129), (1, 255), (1, 257), (1, 544), (1, 8736), (3, 257)])
def test_wide_equals_narrow(B, M, N, epi):
    K = 200   # 4 k-blocks, the last 8 wide
    g = _g(1000 * B + M + 7 * N + epi)
    x, w, b = _bf(B, M, K, g=g), _bf(N, K, g=g, scale=K ** -0.5 * 2), _bf(N, g=g, scale=0.5)
    resid, gate = _bf(B, M, N, g=g), _bf(B, N, g=g)
    buf128, out128 = _linear(128, x, w, b, epi, resid, gate)
    buf256, out256 = _linear(256, x, w, b, epi, resid, gate)
    assert _outside_nan(buf128, M, N) and _outside_nan(buf256, M, N), "a path wrote outside its output"
    assert not torch.isnan(out256).any(), "the wide path left output elements unwritten"
    assert torch.equal(out128, out256), f"wide tile differs from 128 x 128: {(out128 != out256).sum().item()} elements"
    if M <= 544 or epi in (R.EPI_BIAS, R.EPI_GATE_RESID):
        emu, floor, _ = R.linear_emu(x, w, b, epi, resid=resid, gate=gate)
        c = R.Checker(f"wide gemm epi{epi} B{B} M{M} N{N} K{K}")
        c.bf16("out", out256, emu, floor, dims=("b", "row", "col"), **TH_GEMM)
        c.finish()


def _rope(S, g):
    ang = torch.rand(S, 64, device="cuda", generator=g) * 6.28
    return torch.cos(ang).repeat_interleave(2, 1).contiguous(), torch.sin(ang).repeat_interleave(2, 1).contiguous()


def _qkv(tile, x, w, b, nq, nk, cos, sin, row0, d, n_extra, ran_on=None):
    """The fused QKV launch forced onto `tile`; it must run on `ran_on` (default: `tile`)."""
    from gpt_image_edit_b200 import ops

    _force(tile)
    B, M, _ = x.shape
    buf, out = _nan_view((B, M, 3 * d))
    cat_buf = cat = out_extra = None
    if n_extra:
        cat_buf, cat = _nan_view((B, M, d + n_extra))
        out_extra = cat[:, :, d:]
    _ran_on(_tags(lambda: ops.linear_qkv_norm_rope(x, w, b, nq, nk, cos, sin, rope_row0=row0, out=out,
                                                   out_extra=out_extra, epi_extra=ops.EPI_GELU_TANH)),
            ran_on or tile)
    return buf, out, cat_buf, cat


@pytest.mark.parametrize("B,M,d,extra,K", [(1, 8736, 3072, True, 136), (1, 544, 3072, False, 136),
                                           (3, 257, 512, True, 200), (1, 129, 256, False, 200),
                                           (1, 1, 256, True, 64)])
def test_wide_qkv_norm_rope_equals_narrow(B, M, d, extra, K):
    """[Q|K|V] (+ the GELU'd MLP block into the pitched [attn|mlp] buffer) on both tiles; rope_row0 > 0."""
    n_extra = 4 * d if extra else 0
    row0 = 17
    g = _g(M + d + extra)
    x = _bf(B, M, K, g=g)
    w, b = _bf(3 * d + n_extra, K, g=g, scale=K ** -0.5), _bf(3 * d + n_extra, g=g, scale=0.5)
    nq, nk = _bf(128, g=g, scale=0.1, shift=1.0), _bf(128, g=g, scale=0.1, shift=1.0)
    cos, sin = _rope(row0 + M + 3, g)
    r128 = _qkv(128, x, w, b, nq, nk, cos, sin, row0, d, n_extra)
    r256 = _qkv(256, x, w, b, nq, nk, cos, sin, row0, d, n_extra)
    for buf, out, cat_buf, cat in (r128, r256):
        assert _outside_nan(buf, M, 3 * d)
        if extra:
            assert _outside_nan(cat_buf, M, d + n_extra)
            assert torch.isnan(cat[:, :, :d]).all(), "the attention columns of [attn|mlp] were written"
    assert not torch.isnan(r256[1]).any()
    assert torch.equal(r128[1], r256[1]), "QKV differs between the tiles"
    if extra:
        assert not torch.isnan(r256[3][:, :, d:]).any()
        assert torch.equal(r128[3][:, :, d:], r256[3][:, :, d:]), "MLP block differs between the tiles"
    if M * (3 * d + n_extra) <= 2 ** 24:
        emu, floor, mth = R.qkv_norm_rope_emu(x, w, b, nq, nk, cos, sin, rope_row0=row0, n_extra=n_extra,
                                              epi_extra=R.EPI_GELU_TANH)
        c = R.Checker(f"wide qkv_norm_rope B{B} M{M} d{d} extra={n_extra}")
        dims = ("b", "row", "col")
        out = r256[1]
        c.bf16("Q", out[..., :d], emu[..., :d], floor[..., :d], math_ref=mth[..., :d], rel_l2_max=8e-3, dims=dims,
               **TH_GEMM)
        c.bf16("K", out[..., d:2 * d], emu[..., d:2 * d], floor[..., d:2 * d], math_ref=mth[..., d:2 * d],
               rel_l2_max=8e-3, dims=dims, **TH_GEMM)
        c.bf16("V", out[..., 2 * d:], emu[..., 2 * d:3 * d], floor[..., 2 * d:3 * d], dims=dims, **TH_GEMM)
        if extra:
            c.bf16("mlp", r256[3][:, :, d:], emu[..., 3 * d:], floor[..., 3 * d:], math_ref=mth[..., 3 * d:],
                   rel_l2_max=6e-3, dims=dims, **TH_GEMM)
        c.finish()


def test_qkv_head_straddle_stays_narrow():
    """d_model = 384 (3 heads): a wide tile would straddle Q / K, so even a forced 256 runs the 128 x 128 tile."""
    g = _g(5)
    d, K, M = 384, 64, 300
    x, w, b = _bf(1, M, K, g=g), _bf(3 * d, K, g=g, scale=K ** -0.5), _bf(3 * d, g=g)
    nq = _bf(128, g=g, scale=0.1, shift=1.0)
    cos, sin = _rope(M, g)
    r256 = _qkv(256, x, w, b, nq, nq, cos, sin, 0, d, 0, ran_on=128)
    r128 = _qkv(128, x, w, b, nq, nq, cos, sin, 0, d, 0)
    assert torch.equal(r128[1], r256[1])


def test_override_rejects_other_widths():
    from gpt_image_edit_b200 import _lib

    assert _lib.lib.b2f_gemm_set_tile_override(192) == -1
    assert _lib.lib.b2f_gemm_set_tile_override(-128) == -1


# The loop's linears at 1024^2 (d 3072) with the tile the automatic rule gives them on 132 SMs.
LOOP = [
    ("qkv img", 8192, 3 * 3072, 3072, "qkv", 128),
    ("qkv txt", 544, 3 * 3072, 3072, "qkv", 128),
    ("single qkv+mlp", 8736, 7 * 3072, 3072, "qkv_split", 256),
    ("to_out img", 8192, 3072, 3072, R.EPI_GATE_RESID, 256),
    ("to_out txt", 544, 3072, 3072, R.EPI_GATE_RESID, 128),
    ("ff1 img", 8192, 4 * 3072, 3072, R.EPI_GELU_TANH, 256),
    ("ff1 txt", 544, 4 * 3072, 3072, R.EPI_GELU_TANH, 256),
    ("ff2 img", 8192, 3072, 4 * 3072, R.EPI_GATE_RESID, 256),
    ("ff2 txt", 544, 3072, 4 * 3072, R.EPI_GATE_RESID, 128),
    ("single proj_out", 8736, 3072, 5 * 3072, R.EPI_GATE_RESID, 256),
]


@pytest.mark.parametrize("name,M,N,K,epi,tile", LOOP, ids=[c[0] for c in LOOP])
def test_automatic_tile_of_loop_shapes(name, M, N, K, epi, tile):
    from gpt_image_edit_b200 import ops

    if torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip("the expected tiles are those of a 132-SM H100")
    g = _g(9)
    x, w, b = _bf(1, M, K, g=g, scale=0.1), _bf(N, K, g=g, scale=0.01), _bf(N, g=g)
    if epi in ("qkv", "qkv_split"):
        d = 3072
        nq = torch.ones(128, device="cuda").bfloat16()
        cos, sin = _rope(M, g)
        out = torch.empty(1, M, 3 * d, device="cuda", dtype=torch.bfloat16)
        extra = torch.empty(1, M, N - 3 * d, device="cuda", dtype=torch.bfloat16) if epi == "qkv_split" else None
        fn = lambda: ops.linear_qkv_norm_rope(x, w, b, nq, nq, cos, sin, out=out, out_extra=extra,
                                              epi_extra=ops.EPI_GELU_TANH)
    else:
        out = torch.zeros(1, M, N, device="cuda", dtype=torch.bfloat16)
        gate = torch.ones(1, N, device="cuda").bfloat16() if epi == R.EPI_GATE_RESID else None
        fn = lambda: ops.linear(x, w, b, epilogue=epi, out=out, resid=out if gate is not None else None, gate=gate)
    _ran_on(_tags(fn), tile)
