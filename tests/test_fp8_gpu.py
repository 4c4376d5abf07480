"""The FP8 path on the GPU: the row quantizer and the fused LayerNorm bit for bit against the row rule, the FP8 GEMM
element by element against its emulation (tests/fp8_ref.py), and the FP8 FLUX forward stage by stage and end to end
against the fp64 FP8 emulation and the fp64 unquantized forward.

Accumulation floor of the FP8 tensor cores.  wgmma ...e4m3.e4m3 accumulates in fp32 registers, but its partial sums are
reported to carry fewer mantissa bits than fp32.  test_gemm_fp8_accumulation_precision measures the error on dot
products whose exact value is 0 (the output is then the accumulation error alone) at the model's contraction lengths.
Measured on an H100 80GB HBM3 (700 W), the worst element over M = 256, N = 384, written as K * 2^-p * absref, had
p = 23.67 at K = 3072, 25.63 at K = 12288 and 25.92 at K = 15360: 2^-12.08, 2^-12.05 and 2^-12.01 times absref.  The
error does not grow with K; it is that of partial sums kept to about 12 bits below the sum of |products|.  A floor
K * 2^-23.67 * absref fails the K = 208 / 336 cases below, so the emulations use max(K * 2^-24, 2^-P_ACC) * absref with
P_ACC = 11, a factor 2 above the measured worst case.  The model-level quality gate passes with the fp32 accumulators
as they are, so the GEMM promotes no partial sums on the CUDA cores.
"""
import pytest
import torch

import fp8_ref as Q
import infer_block_ref as IB
import kernel_ref as R
from oracle import flux_oracle as fo
from test_flux_blocks_gpu import CASES, _fwd, _report, _setup, _temb_mod
from test_gemm_persistent_gpu import _cdiv, _nan_view, _outside_untouched, _sms, _slices

pytestmark = pytest.mark.gpu

# accumulation floor max(K * 2^-24, 2^-P_ACC) * absref of the FP8 GEMM (module docstring: measured worst 2^-12.01)
P_ACC = 11.0
TH_GEMM = dict(max_ulp=2, share_gt1=1e-3, mean_ulp=0.1)
f64, bf16 = torch.float64, torch.bfloat16


def _g(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _bf(*shape, g, scale=1.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).bfloat16()


def _u8(t):
    return t.view(torch.uint8)


# ---------------------------------------------------------------------------------------------------- quantizer
@pytest.mark.parametrize("K", [16, 48, 272, 3072, 15360])
def test_quant_rows_bit_exact(K):
    """Batched rows with a batch stride, a row pitch wider than K on both sides, zero rows, rows spanning 6 decades."""
    from gpt_image_edit_b200 import ops

    g = _g(K)
    B, rows = 3, 37
    src = torch.randn(B, rows + 2, K + 24, device="cuda", generator=g)
    src *= torch.logspace(-4, 2, rows + 2, device="cuda")[None, :, None]
    x = src.bfloat16()[:, 1:rows + 1, 8:8 + K]
    x[1, 3] = 0
    x[2, 5] = -0.0
    qbuf = torch.full((B, rows, K + 32), 0x7F, device="cuda", dtype=torch.uint8)   # 0x7f: an e4m3 NaN
    q = qbuf[:, :, 16:16 + K].view(Q.E4M3)
    sbuf = torch.full((B, rows + 5), float("nan"), device="cuda")
    ops.quant_fp8_rows(x, out=q, scale=sbuf[:, :rows])
    qr, sr = Q.quant_rows(x)
    c = R.Checker(f"quant K{K}")
    c.equal("e4m3 bytes", _u8(q), _u8(qr))
    c.equal("scales", sbuf[:, :rows], sr)
    c.equal("bytes outside the view", qbuf[:, :, :16].ne(0x7F).sum() + qbuf[:, :, 16 + K:].ne(0x7F).sum(),
            torch.zeros((), device="cuda", dtype=torch.long))
    c.equal("scales outside the view", torch.isnan(sbuf[:, rows:]).all(), torch.tensor(True, device="cuda"))
    c.finish()


def test_quant_rows_pitched_cat_slice():
    """The model's launch: columns [d, 5d) of cat [B, S, 5d] -> q8 [B, S, 5d] (pitch 5d bytes), scales [B, S]."""
    from gpt_image_edit_b200 import ops

    g = _g(5)
    B, S, d = 2, 257, 512
    cat = _bf(B, S, 5 * d, g=g)
    q8 = torch.zeros(B, S, 5 * d, device="cuda", dtype=Q.E4M3)
    s = torch.zeros(B, S, device="cuda")
    ops.quant_fp8_rows(cat[:, :, d:], out=q8[:, :, :4 * d], scale=s)
    qr, sr = Q.quant_rows(cat[:, :, d:])
    assert torch.equal(_u8(q8[:, :, :4 * d]), _u8(qr)) and torch.equal(s, sr)
    assert not _u8(q8[:, :, 4 * d:]).any()


# ---------------------------------------------------------------------------------------------------- fused LN
@pytest.mark.parametrize("D,split", [(3072, 77), (3072, 0), (1024, 5)])
def test_ln_modulate_fp8_equals_ln_then_quant(D, split):
    from gpt_image_edit_b200 import ops

    g = _g(D + split)
    B, rows = 2, 300
    x = _bf(B, rows, D, g=g, scale=3.0)
    x[1, 7] = 0.5                                 # a constant row: LN gives 0 -> an all-shift row
    mod = _bf(B, 4 * D, g=g, scale=0.5)
    sc, sh, sc_b, sh_b = mod[:, :D], mod[:, D:2 * D], mod[:, 2 * D:3 * D], mod[:, 3 * D:]
    kw = dict(split_row=split, scale_b=sc_b if split else None, shift_b=sh_b if split else None)
    y = ops.ln_modulate(x, sc, sh, **kw)
    qr, sr = ops.quant_fp8_rows(y)
    qbuf = torch.zeros(B, rows, D + 64, device="cuda", dtype=Q.E4M3)
    sbuf = torch.zeros(B, rows + 3, device="cuda")
    q, s = ops.ln_modulate_fp8(x, sc, sh, out=qbuf[:, :, :D], row_scale=sbuf[:, :rows], **kw)
    assert torch.equal(_u8(q), _u8(qr)) and torch.equal(s, sr)
    q2, s2 = Q.quant_rows(y)
    assert torch.equal(_u8(q), _u8(q2)) and torch.equal(s, s2)


# ---------------------------------------------------------------------------------------------------- GEMM
def _operands(B, M, N, K, g, pitch_pad=32):
    """e4m3 x [B, M, K] as a pitched view (row pitch K + pitch_pad), w [N, K], their scales, a bias."""
    from gpt_image_edit_b200 import ops

    x = _bf(B, M, K, g=g) * torch.logspace(-2, 1, M, device="cuda").bfloat16()[None, :, None]
    w = _bf(N, K, g=g, scale=K ** -0.5)
    xbuf = torch.zeros(B, M, K + pitch_pad, device="cuda", dtype=Q.E4M3)
    xq, xs = ops.quant_fp8_rows(x, out=xbuf[:, :, :K])
    wq, ws = ops.quant_fp8_rows(w)
    return xq, xs, wq, ws, _bf(N, g=g, scale=0.5)


def _acc_bits(out, xq, xs, wq, ws):
    """-log2 of the largest accumulation error relative to absref that `out` shows (exact products are 0)."""
    sc = xs.double()[..., :, None] * ws.double()[None, :]
    absref = (xq.double().abs() @ wq.double().abs().T) * sc
    e = (R.d64(out).abs() / absref).max().item()
    return float("inf") if e == 0 else -torch.log2(torch.tensor(e)).item()


@pytest.mark.parametrize("K", [3072, 12288, 15360])
def test_gemm_fp8_accumulation_precision(K):
    """x = [a, a], w = [b, -b] along K: every exact dot product is 0 while its partial sums are not, so the output is
    the tensor cores' accumulation error (times the scales) rounded once to bf16."""
    from gpt_image_edit_b200 import ops

    g = _g(K)
    M, N, h = 256, 384, K // 2
    a = _bf(M, h, g=g)
    b = _bf(N, h, g=g)
    xq, xs = ops.quant_fp8_rows(torch.cat([a, a], 1))
    wq, ws = ops.quant_fp8_rows(torch.cat([b, -b], 1))
    out = ops.linear_fp8(xq, xs, wq, ws)
    p = _acc_bits(out, xq, xs, wq, ws)
    k = torch.log2(torch.tensor(float(K))).item()
    nz = (out != 0).double().mean().item()
    print(f"KREF fp8 accumulation K={K}: worst |err| = 2^-{p:.2f} * absref = K * 2^-{p + k:.2f} * absref; "
          f"nonzero outputs {nz:.3g}")
    assert p >= P_ACC, f"accumulation error 2^-{p:.2f} * absref exceeds the stated floor 2^-{P_ACC}"


def _many_tiles():
    S = _sms()
    n_blk = 17
    m_blk = _cdiv(3 * S, n_blk) + 1
    return [(1, m_blk * 128 - 51, n_blk * 128, 400),   # >= 3 tiles per CTA; 4 k-blocks, the last 16 wide
            (2, 130, 8 * 128 + 40, 208),               # batch 2, ragged M and N
            (1, 100, 8, 3072)]                         # one tile, N = 8


@pytest.mark.parametrize("epi", [R.EPI_BIAS, R.EPI_GELU_TANH, R.EPI_GELU_ERF, R.EPI_SILU, R.EPI_QUICK_GELU,
                                 R.EPI_GATE_RESID, R.EPI_RESID])
@pytest.mark.parametrize("case", range(3))
def test_gemm_fp8_epilogues(epi, case):
    from gpt_image_edit_b200 import ops

    B, M, N, K = _many_tiles()[case]
    g = _g(100 * epi + case)
    xq, xs, wq, ws, b = _operands(B, M, N, K, g)
    bias = None if case == 2 else b
    resid, gate = _bf(B, M, N, g=g), _bf(B, N, g=g)
    buf, out = _nan_view((B, M, N))
    if epi in (R.EPI_GATE_RESID, R.EPI_RESID):
        out.copy_(resid)
        ops.linear_fp8(xq, xs, wq, ws, bias, epilogue=epi, resid=out, gate=gate if epi == R.EPI_GATE_RESID else None,
                       out=out)
    else:
        ops.linear_fp8(xq, xs, wq, ws, bias, epilogue=epi, out=out)
    emu, floor, _ = Q.linear_fp8_emu(xq, xs, wq, ws, bias, epi, p=P_ACC, resid=resid, gate=gate)
    c = R.Checker(f"gemm fp8 epi{epi} B{B} M{M} N{N} K{K}")
    c.bf16("out", out, emu, floor, dims=("b", "row", "col"), **TH_GEMM)
    _outside_untouched(c, buf, _slices(buf, M, N))
    c.finish()


@pytest.mark.parametrize("extra", [True, False])
def test_gemm_fp8_qkv_norm_rope(extra):
    from gpt_image_edit_b200 import ops
    from test_gemm_persistent_gpu import _rope

    B, H, K, row0 = 2, 3, 336, 24
    d = H * 128
    n_extra = 4 * d if extra else 0
    M = 300
    g = _g(300 + extra)
    xq, xs, wq, ws, b = _operands(B, M, 3 * d + n_extra, K, g)
    nq, nk = (_bf(128, g=g, scale=0.1) + 1).bfloat16(), (_bf(128, g=g, scale=0.1) + 1).bfloat16()
    cos, sin = _rope(row0 + M + 3, g)
    buf, out = _nan_view((B, M, 3 * d))
    cat = out_extra = None
    if extra:
        cat_buf, cat = _nan_view((B, M, d + n_extra))
        out_extra = cat[:, :, d:]
    ops.linear_qkv_norm_rope_fp8(xq, xs, wq, ws, b, nq, nk, cos, sin, rope_row0=row0, out=out, out_extra=out_extra,
                                 epi_extra=ops.EPI_GELU_TANH)
    emu, floor, _ = Q.qkv_fp8_emu(xq, xs, wq, ws, b, nq, nk, cos, sin, p=P_ACC, rope_row0=row0, n_extra=n_extra,
                                  epi_extra=R.EPI_GELU_TANH)
    c = R.Checker(f"qkv fp8 B{B} M{M} H{H} extra={n_extra}")
    dims = ("b", "row", "col")
    c.bf16("QKV", out, emu[..., :3 * d], floor[..., :3 * d], dims=dims, **TH_GEMM)
    _outside_untouched(c, buf, _slices(buf, M, 3 * d))
    if extra:
        c.bf16("mlp", out_extra, emu[..., 3 * d:], floor[..., 3 * d:], dims=dims, **TH_GEMM)
        c.equal("attn columns (still NaN)", torch.isnan(cat[:, :, :d]), torch.ones_like(cat[:, :, :d], dtype=torch.bool))
        _outside_untouched(c, cat_buf, _slices(cat_buf, M, d + n_extra), "outside [attn|mlp]")
    c.finish()


def test_gemm_fp8_refuses_unmappable_operands():
    from gpt_image_edit_b200 import _lib, ops

    g = _g(9)
    xq, xs, wq, ws, _ = _operands(1, 64, 128, 64, g)
    with pytest.raises(_lib.B2FError):      # row pitch 72 bytes: not a multiple of 16
        ops.linear_fp8(torch.zeros(64, 72, device="cuda", dtype=Q.E4M3)[:, :64], xs, wq, ws)
    with pytest.raises(_lib.B2FError):      # K = 40
        ops.linear_fp8(xq[..., :40], xs, wq[:, :40], ws)


def test_fp8_wrappers_refuse_wrong_shapes():
    """Buffers that do not match the operands raise instead of being written past their end."""
    from gpt_image_edit_b200 import _lib, ops

    g = _g(10)
    x = _bf(2, 64, 256, g=g)
    for kw in (dict(out=torch.empty(2, 32, 256, device="cuda", dtype=Q.E4M3)),
               dict(scale=torch.empty(2, 32, device="cuda")), dict(scale=torch.empty(64, device="cuda"))):
        with pytest.raises(_lib.B2FError):
            ops.quant_fp8_rows(x, **kw)
    mod = _bf(2, 512, g=g)
    with pytest.raises(_lib.B2FError):
        ops.ln_modulate_fp8(x, mod[:, :256], mod[:, 256:], row_scale=torch.empty(2, 16, device="cuda"))
    xq, xs, wq, ws, b = _operands(2, 64, 128, 256, g)
    bad = [dict(wq=wq[:, :128]), dict(ws=ws[:64]), dict(b=b[:64]),
           dict(xs=xs[:1]), dict(out=torch.empty(2, 64, 64, device="cuda", dtype=bf16))]
    for kw in bad:
        a = dict(xq=xq, xs=xs, wq=wq, ws=ws, b=b, out=None) | kw
        with pytest.raises(_lib.B2FError):
            ops.linear_fp8(a["xq"], a["xs"], a["wq"], a["ws"], a["b"], out=a["out"])
    with pytest.raises(_lib.B2FError):      # residual of the wrong shape
        ops.linear_fp8(xq, xs, wq, ws, b, epilogue=ops.EPI_RESID, resid=torch.empty(2, 32, 128, device="cuda", dtype=bf16))


# ---------------------------------------------------------------------------------------------------- the model
def _model_inputs(s):
    return dict(hidden_states=s.hs, encoder_hidden_states=s.enc, pooled_projections=s.pooled, timestep=s.t,
                img_ids=s.img_ids, txt_ids=s.txt_ids, guidance=s.gd, return_dict=False)


def test_fp8_forward_stagewise_matches_fp8_emulation():
    """Each block's output against the fp64 FP8 emulation run from the engine's own input to that block (torch-bf16 of
    the same quantized stage is the yardstick), at d = 3072 with ragged S_txt / S_img and B = 2."""
    s = _setup(*CASES["ragged"])
    s.model.enable_fp8()
    _, mod, _ = _temb_mod(s, s.t, s.gd, s.pooled)
    _fwd(s, (0, 0))
    h = s.model.debug_buffers(s.B, s.S_img, s.S_txt).h.clone()
    checks = []
    d = s.ocfg.inner_dim
    for blk in range(s.nblk):
        h_in = h
        _fwd(s, (blk, blk + 1))
        bufs = s.model.debug_buffers(s.B, s.S_img, s.S_txt)
        K = {"h": bufs.h.clone(), "qkv": bufs.qkv.clone(), "attn": bufs.cat[..., :d].clone(),
             "mlp": bufs.cat[..., d:].clone()}
        h = K["h"]
        if blk < s.ocfg.num_layers:
            name, f = f"double{blk}", (lambda sd, dt: IB.double_stage(sd, s.ocfg, blk, h_in, mod, s.cos, s.sin,
                                                                       s.S_txt, dt))
        else:
            si = blk - s.ocfg.num_layers
            name, f = f"single{si}", (lambda sd, dt: IB.single_stage(sd, s.ocfg, si, h_in, mod, s.cos, s.sin, dt))
        with Q.fp8_linears():
            Rf, Yf = f(s.sd, f64), f(s.sd, bf16)
        checks += IB.token_gates(name, "h", K["h"], Rf["h"], Yf["h"], s.S_txt, base=h_in)
        for n in ("qkv", "attn"):
            checks += IB.token_gates(name, n, K[n], Rf[n], Yf[n], s.S_txt, heads=True)
        checks += IB.token_gates(name, "mlp", K["mlp"], Rf["mlp"], Yf["mlp"], s.S_txt)
        del K, Rf, Yf
    bad = _report("fp8 stagewise", s, checks)
    assert not bad, "\n".join(bad)


def test_fp8_forward_quality_gate():
    """rel-L2 of the FP8 engine to the fp64 unquantized forward <= E_emu (what FP8 itself costs: fp64 FP8 emulation vs
    fp64) + E_bf16 (what bf16 costs: the bf16 engine vs fp64).

    The engine receives timestep and guidance as bf16(x) * 1000 in bf16 (the diffusers chain), the fp64 oracle as
    x * 1000 in fp64: the values are chosen so that both are exact (3.5 would become 3504 in the engine against 3500 in
    the reference, and E_bf16 would measure that input change instead of bf16 arithmetic)."""
    s = _setup(*CASES["ragged"])
    s.gd = torch.tensor([4.0, 2.0], device="cuda")
    for v in (s.t, s.gd):
        assert torch.equal(s.model._times1000(v).double(), v.double() * 1000), "x1000 not exact in bf16"
    out_bf16 = s.model(**_model_inputs(s))[0].clone()
    s.model.enable_fp8()
    out_fp8 = s.model(**_model_inputs(s))[0].clone()
    sd64 = {k: v.double() for k, v in s.sd.items()}
    args = (s.hs.double(), s.enc.double(), s.pooled.double(), s.t, s.img_ids, s.txt_ids)
    ref = fo.flux_forward(sd64, s.ocfg, *args, guidance=s.gd)
    with Q.fp8_linears():
        emu = fo.flux_forward(sd64, s.ocfg, *args, guidance=s.gd)
    e_emu, e_bf16, e_fp8 = R.rel_l2(emu, ref), R.rel_l2(out_bf16, ref), R.rel_l2(out_fp8, ref)
    # Printed, not gated: the engine quantizes bf16 activations and the emulation fp64 ones, so elements on either side
    # of an e4m3 rounding boundary differ by a whole e4m3 step and the two runs carry different quantization noise of
    # the same size (measured on an H100: 0.063 with E_emu 0.071).  The engine is held to the emulation block by block,
    # from its own input to each block, in test_fp8_forward_stagewise_matches_fp8_emulation.
    e_vs_emu = R.rel_l2(out_fp8, emu)
    print(f"KREF fp8 quality: E_emu={e_emu:.4g} E_bf16={e_bf16:.4g} FP8 engine={e_fp8:.4g} "
          f"(FP8 engine vs emulation {e_vs_emu:.4g})")
    assert e_fp8 <= e_emu + e_bf16


def test_fp8_switching():
    """enable -> disable gives the never-enabled bits; fuse_lora / load_state_dict while enabled give the bits of
    enabling afterwards; unfused adapters and training are refused while FP8 is on."""
    import lora_ref as LR
    from gpt_image_edit_b200 import _lib
    from gpt_image_edit_b200.training import FluxTrainGraph

    s = _setup(*CASES["toy_text_of_one"])
    m, inp = s.model, _model_inputs(s)
    base = m(**inp)[0].clone()
    m.enable_fp8()
    assert m.fp8_enabled
    fp8 = m(**inp)[0].clone()
    assert not torch.equal(fp8, base)
    m.disable_fp8()
    assert not m.fp8_enabled and torch.equal(m(**inp)[0], base)

    # load_state_dict while enabled == enabling after the load
    sd2 = {k: (v.float() * 1.01).bfloat16() for k, v in m.state_dict().items()}
    m.enable_fp8()
    m.load_state_dict(sd2)
    a = m(**inp)[0].clone()
    m.disable_fp8()
    m.enable_fp8()
    assert torch.equal(m(**inp)[0], a)

    # an unfused adapter is refused by the forward; fusing it while enabled == enabling after the fuse
    la = LR.make_lora(s.ocfg, rank=8, seed=3, alpha=16.0, a_std=0.03, b_std=0.03)
    m.load_lora_adapter(LR.to_diffusers(la), adapter_name="a")
    with pytest.raises(_lib.B2FError, match="fuse_lora"):
        m(**inp)
    m.fuse_lora()
    fused = m(**inp)[0].clone()
    m.disable_fp8()
    m.enable_fp8()
    assert torch.equal(m(**inp)[0], fused)
    m.unfuse_lora()                                   # unfused again: refused; disabling FP8 runs it unfused
    with pytest.raises(_lib.B2FError, match="fuse_lora"):
        m(**inp)
    m.disable_fp8()                                   # FP8 off: the adapter is bound and acts unfused
    assert m.lora_unfused_active()
    with pytest.raises(_lib.B2FError, match="fuse_lora"):
        m.enable_fp8()                                # refused while an adapter is unfused
    assert not m.fp8_enabled
    m(**inp)
    m.unload_lora()

    # the training graph refuses a denoiser with FP8 on
    m.enable_fp8()
    den = type("Tower", (), {})()
    den.denoiser = m
    model = type("M", (), {})()
    model.denoise_tower = den
    with pytest.raises(_lib.B2FError, match="disable_fp8"):
        FluxTrainGraph(model, [])
