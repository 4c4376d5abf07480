"""Unfused LoRA on the FP8 block linears, on the GPU: b2f_gemm_fp8_lora / b2f_gemm_qkv_norm_rope_fp8_lora element by
element against their emulation (tests/lora_fp8_ref.py) at the tile edges, the fidelity of an adapter's update against
fusing it into the e4m3 weights, the FP8 forward with adapters stage by stage against the fp64 FP8 oracle with PEFT-style
unfused adapters, and the model's switching contract (enable_fp8(unfused_lora=True))."""
import pytest
import torch

import attn_fp8_ref as A
import fp8_ref as Q
import infer_block_ref as IB
import kernel_ref as R
import lora_fp8_ref as LQ
import lora_ref as LR
from test_flux_blocks_gpu import CASES, _fwd, _report, _setup, _temb_mod
from test_fp8_gpu import P_ACC, TH_GEMM
from test_gemm_persistent_gpu import _cdiv, _nan_view, _outside_untouched, _rope, _slices, _sms

pytestmark = pytest.mark.gpu

f64, bf16 = torch.float64, torch.bfloat16


def _g(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _bf(*shape, g, scale=1.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).bfloat16()


def _operands(B, M, N, K, r_pad, g):
    """e4m3 x [B, M, K] (row pitch K + 32) with its scales, e4m3 w [N, K] with its scales, bf16 T [B, M, r_pad] (row
    pitch r_pad + 8) and Bcat [N, r_pad] (pitch r_pad + 16), a bias."""
    from gpt_image_edit_b200 import ops

    x = _bf(B, M, K, g=g) * torch.logspace(-2, 1, M, device="cuda").bfloat16()[None, :, None]
    w = _bf(N, K, g=g, scale=K ** -0.5)
    xbuf = torch.zeros(B, M, K + 32, device="cuda", dtype=Q.E4M3)
    xq, xs = ops.quant_fp8_rows(x, out=xbuf[:, :, :K])
    wq, ws = ops.quant_fp8_rows(w)
    t = (_bf(B, M, r_pad + 8, g=g) * torch.logspace(-2, 1, M, device="cuda").bfloat16()[None, :, None])[..., :r_pad]
    bcat = _bf(N, r_pad + 16, g=g, scale=r_pad ** -0.5)[:, :r_pad]
    return xq, xs, wq, ws, t, bcat, _bf(N, g=g, scale=0.5)


def _many_tiles():
    S = _sms()
    n_blk = 17
    return (1, (_cdiv(3 * S, n_blk) + 1) * 128 - 51, n_blk * 128, 3072, 64)   # >= 3 tiles per CTA


GEMM_CASES = [  # (B, M, N, K, r_pad)
    (1, 1, 136, 3072, 64),
    (1, 127, 392, 12288, 128),
    (2, 129, 1032, 3072, 192),          # batch 2, pitched views, ragged N
    (1, 4641, 1032, 15360, 64),
    (2, 300, 520, 336, 128),             # K % 128 != 0: the last e4m3 k-block is partly out of bounds
]


@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("case", range(len(GEMM_CASES) + 1))
def test_gemm_fp8_lora_shapes(case, bias):
    from gpt_image_edit_b200 import ops

    B, M, N, K, r_pad = GEMM_CASES[case] if case < len(GEMM_CASES) else _many_tiles()
    g = _g(10 + case)
    xq, xs, wq, ws, t, bcat, b = _operands(B, M, N, K, r_pad, g)
    b = b if bias else None
    buf, out = _nan_view((B, M, N))
    ops.linear_fp8_lora(xq, xs, wq, ws, b, t, bcat, out=out)
    emu, floor, _ = LQ.linear_fp8_lora_emu(xq, xs, wq, ws, t, bcat, b, p=P_ACC)
    c = R.Checker(f"gemm fp8 lora B{B} M{M} N{N} K{K} r_pad{r_pad} bias={bias}")
    c.bf16("out", out, emu, floor, dims=("b", "row", "col"), **TH_GEMM)
    _outside_untouched(c, buf, _slices(buf, M, N))
    c.finish()


@pytest.mark.parametrize("epi", [R.EPI_BIAS, R.EPI_GELU_TANH, R.EPI_GELU_ERF, R.EPI_SILU, R.EPI_QUICK_GELU,
                                 R.EPI_GATE_RESID, R.EPI_RESID])
def test_gemm_fp8_lora_every_epilogue(epi):
    """Every forward epilogue, batched with pitched views, residual ones in place."""
    from gpt_image_edit_b200 import ops

    B, M, N, K, r_pad = 2, 200, 384, 336, 64
    g = _g(100 + epi)
    xq, xs, wq, ws, t, bcat, b = _operands(B, M, N, K, r_pad, g)
    resid, gate = _bf(B, M, N, g=g), _bf(B, N, g=g)
    out = torch.empty(B, M, N, device="cuda", dtype=bf16)
    if epi in (R.EPI_GATE_RESID, R.EPI_RESID):
        out.copy_(resid)
        ops.linear_fp8_lora(xq, xs, wq, ws, b, t, bcat, epilogue=epi, resid=out,
                            gate=gate if epi == R.EPI_GATE_RESID else None, out=out)
    else:
        ops.linear_fp8_lora(xq, xs, wq, ws, b, t, bcat, epilogue=epi, out=out)
    emu, floor, _ = LQ.linear_fp8_lora_emu(xq, xs, wq, ws, t, bcat, b, epi, p=P_ACC, resid=resid, gate=gate)
    c = R.Checker(f"gemm fp8 lora epi{epi}")
    c.bf16("out", out, emu, floor, dims=("b", "row", "col"), **TH_GEMM)
    c.finish()


@pytest.mark.parametrize("extra", [False, True])
def test_gemm_qkv_norm_rope_fp8_lora(extra):
    from gpt_image_edit_b200 import ops

    B, H, K, M, row0, r_pad = 2, 3, 336, 300, 24, 128
    d = H * 128
    n_extra = 4 * d if extra else 0
    g = _g(300 + extra)
    xq, xs, wq, ws, t, bcat, b = _operands(B, M, 3 * d + n_extra, K, r_pad, g)
    nq, nk = (_bf(128, g=g, scale=0.1) + 1).bfloat16(), (_bf(128, g=g, scale=0.1) + 1).bfloat16()
    cos, sin = _rope(row0 + M + 3, g)
    buf, out = _nan_view((B, M, 3 * d))
    cat = out_extra = None
    if extra:
        cat_buf, cat = _nan_view((B, M, d + n_extra))
        out_extra = cat[:, :, d:]
    ops.linear_qkv_norm_rope_fp8_lora(xq, xs, wq, ws, b, nq, nk, cos, sin, t, bcat, rope_row0=row0, out=out,
                                      out_extra=out_extra, epi_extra=ops.EPI_GELU_TANH)
    emu, floor, _ = LQ.qkv_fp8_lora_emu(xq, xs, wq, ws, t, bcat, b, nq, nk, cos, sin, p=P_ACC, rope_row0=row0,
                                        n_extra=n_extra, epi_extra=R.EPI_GELU_TANH)
    c = R.Checker(f"qkv fp8 lora B{B} M{M} H{H} extra={n_extra}")
    dims = ("b", "row", "col")
    c.bf16("QKV", out, emu[..., :3 * d], floor[..., :3 * d], dims=dims, **TH_GEMM)
    _outside_untouched(c, buf, _slices(buf, M, 3 * d))
    if extra:
        c.bf16("mlp", out_extra, emu[..., 3 * d:], floor[..., 3 * d:], dims=dims, **TH_GEMM)
        c.equal("attn columns (still NaN)", torch.isnan(cat[:, :, :d]), torch.ones_like(cat[:, :, :d], dtype=torch.bool))
        _outside_untouched(c, cat_buf, _slices(cat_buf, M, d + n_extra), "outside [attn|mlp]")
    c.finish()


def test_gemm_fp8_lora_refusals():
    from gpt_image_edit_b200 import _lib, ops

    g = _g(9)
    xq, xs, wq, ws, t, bcat, b = _operands(1, 64, 128, 256, 64, g)
    for r in (32, 96):                                        # r_pad not a multiple of 64
        tt = _bf(1, 64, r, g=g)
        with pytest.raises(_lib.B2FError):
            ops.linear_fp8_lora(xq, xs, wq, ws, b, tt, _bf(128, r, g=g))
    with pytest.raises(_lib.B2FError):                       # r_pad 0
        ops.linear_fp8_lora(xq, xs, wq, ws, b, t[..., :0], bcat[:, :0])
    tbuf = _bf(1, 64, 80, g=g)
    with pytest.raises(_lib.B2FError):                       # T's base not 16-byte aligned
        ops.linear_fp8_lora(xq, xs, wq, ws, b, tbuf[..., 4:68], bcat)
    tbuf = _bf(1, 64, 68, g=g)
    with pytest.raises(_lib.B2FError):                       # T's row pitch 68: not a multiple of 8
        ops.linear_fp8_lora(xq, xs, wq, ws, b, tbuf[..., :64], bcat)
    with pytest.raises(_lib.B2FError):                       # e4m3 row pitch 72 bytes
        ops.linear_fp8_lora(torch.zeros(64, 72, device="cuda", dtype=Q.E4M3)[:, :64], xs, wq[:, :64], ws, b,
                            t[0], bcat)
    with pytest.raises(_lib.B2FError):                       # the QKV epilogue only through the QKV entry point
        ops.linear_fp8_lora(xq, xs, wq, ws, b, t, bcat, epilogue=6)
    with pytest.raises(_lib.B2FError):                       # T rows do not match x
        ops.linear_fp8_lora(xq, xs, wq, ws, b, t[:, :32], bcat)


# ---------------------------------------------------------------------------------------------------- fidelity
@pytest.mark.parametrize("rel_dw", [0.003, 0.01, 0.03])
def test_update_fidelity_unfused_vs_fused(rel_dw):
    """One 3072 x 3072 linear, 512 tokens, a rank-16 update with |dW| / |W| = rel_dw.  The change the adapter makes to
    the output, y_A - y_0, against the fp64 update x dW^T: unfused in FP8 (b2f_gemm_fp8_lora), fused into the weight and
    re-quantized (FP8), and unfused in bf16 (b2f_gemm_bf16_lora)."""
    from gpt_image_edit_b200 import ops

    g = _g(500)
    M, K, N, r = 512, 3072, 3072, 16
    x, w = _bf(M, K, g=g), _bf(N, K, g=g, scale=K ** -0.5)
    a, bm = _bf(r, K, g=g, scale=K ** -0.5), _bf(N, r, g=g)
    dw0 = R.d64(bm) @ R.d64(a)
    s = rel_dw * R.d64(w).norm().item() / dw0.norm().item()
    acat = torch.zeros(64, K, device="cuda", dtype=bf16)
    bcat = torch.zeros(N, 64, device="cuda", dtype=bf16)
    acat[:r], bcat[:, :r] = a, bm
    cs = torch.zeros(64, device="cuda")
    cs[:r] = s
    ref = R.d64(x) @ (s * dw0).T
    t = ops.lora_down(x, acat, cs)
    xq, xs = ops.quant_fp8_rows(x)
    wq, ws = ops.quant_fp8_rows(w)
    y0 = ops.linear_fp8(xq, xs, wq, ws)
    e_unf8 = R.rel_l2(R.d64(ops.linear_fp8_lora(xq, xs, wq, ws, None, t, bcat)) - R.d64(y0), ref)
    wf = w.clone()
    ops.lora_fuse_(wf, bcat[:, :r].contiguous(), acat[:r].contiguous(), cs[:r].contiguous())
    wfq, wfs = ops.quant_fp8_rows(wf)
    e_fus8 = R.rel_l2(R.d64(ops.linear_fp8(xq, xs, wfq, wfs)) - R.d64(y0), ref)
    yb0 = ops.linear(x, w)
    e_unfb = R.rel_l2(R.d64(ops.linear_lora(x, w, None, t, bcat)) - R.d64(yb0), ref)
    print(f"KREF lora fp8 fidelity |dW|/|W|={rel_dw:g}: update rel-L2 unfused fp8 {e_unf8:.4g}, fused-then-quantized "
          f"fp8 {e_fus8:.4g}, unfused bf16 {e_unfb:.4g}")
    assert e_unf8 <= 2 * e_unfb and e_unf8 < e_fus8


# ---------------------------------------------------------------------------------------------------- the model
def _with_adapters(s, scale=0.7, wb=0.5):
    """Two adapters on every target (every linear, the AdaLN ones and the embedders included), set as in the LoRA
    stage tests, at call scale `scale`."""
    la = LR.make_lora(s.ocfg, rank=16, seed=11, alpha=32.0, a_std=0.03, b_std=0.03)
    lb = LR.make_lora(s.ocfg, rank=8, seed=12, alpha=None, a_std=0.03, b_std=0.03)
    s.model.load_lora_adapter(LR.to_diffusers(la), adapter_name="a")
    s.model.load_lora_adapter(LR.to_bfl(s.ocfg, lb), adapter_name="b")
    s.model.set_adapters(["a", "b"], [1.0, wb])
    s.scale = scale
    return [(la, scale), (lb, scale * wb)]


@pytest.mark.parametrize("attention", [False, True])
def test_fp8_lora_forward_stagewise(attention):
    """Each block's output against the fp64 FP8 emulation with PEFT-style unfused adapters (fp8_lora_linears(), with
    fp8_attention() when the attention runs in FP8 too) from the engine's own input to that block, at d = 3072 with
    ragged S_txt / S_img and B = 2; the gates of test_fp8_forward_stagewise_matches_fp8_emulation."""
    import contextlib

    s = _setup(*CASES["ragged"])
    loras = _with_adapters(s)
    s.model.enable_fp8(attention=attention, unfused_lora=True)
    assert s.model.fp8_unfused_lora and s.model.lora_unfused_active()
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
        with (A.fp8_attention() if attention else contextlib.nullcontext()), LQ.fp8_lora_linears(loras):
            Rf, Yf = f(s.sd, f64), f(s.sd, bf16)
        checks += IB.token_gates(name, "h", K["h"], Rf["h"], Yf["h"], s.S_txt, base=h_in)
        for n in ("qkv", "attn"):
            checks += IB.token_gates(name, n, K[n], Rf[n], Yf[n], s.S_txt, heads=True)
        checks += IB.token_gates(name, "mlp", K["mlp"], Rf["mlp"], Yf["mlp"], s.S_txt)
        del K, Rf, Yf
    bad = _report(f"fp8 + unfused lora stagewise (attention {attention})", s, checks)
    assert not bad, "\n".join(bad)


def _inputs(s):
    return dict(hidden_states=s.hs, encoder_hidden_states=s.enc, pooled_projections=s.pooled, timestep=s.t,
                img_ids=s.img_ids, txt_ids=s.txt_ids, guidance=s.gd, return_dict=False)


def test_fp8_unfused_lora_contract():
    """enable_fp8(unfused_lora=True) before or after loading gives the same bits; adapter, weight and scale changes leave
    the e4m3 weights alone and invalidate the first-block cache; cache threshold 0 == cache off; disable_fp8() gives
    the bf16 unfused bits; the default enable_fp8() keeps refusing; training refuses."""
    from gpt_image_edit_b200 import _lib
    from gpt_image_edit_b200.flux_transformer import FirstBlockCacheConfig
    from gpt_image_edit_b200.training import FluxTrainGraph

    s = _setup(*CASES["toy_text_of_one"])
    m, inp = s.model, _inputs(s)
    run = lambda sc=0.7: m(**inp, joint_attention_kwargs={"scale": sc})[0].clone()
    base = run()
    _with_adapters(s)
    bf16_unfused = run()
    m.enable_fp8(unfused_lora=True)                          # adapters loaded before
    assert m.fp8_enabled and m.fp8_unfused_lora and not m.fp8_attention_enabled
    after = run()
    assert not torch.equal(after, bf16_unfused)
    m.disable_fp8()
    assert not m.fp8_unfused_lora and torch.equal(run(), bf16_unfused), "disable_fp8() != the bf16 unfused bits"
    m.unload_lora()
    assert torch.equal(run(), base)
    m.enable_fp8(unfused_lora=True)                          # adapters loaded after
    _with_adapters(s)
    assert torch.equal(run(), after), "enable_fp8(unfused_lora=True) before / after loading differ"
    # mode 1 -> mode 2 with the adapters already loaded: the same bits again
    m.disable_fp8()
    m.unload_lora()
    m.enable_fp8()
    _with_adapters(s)
    with pytest.raises(_lib.B2FError, match="fuse_lora"):
        m(**inp)
    m.enable_fp8(unfused_lora=True)
    assert torch.equal(run(), after)
    m.enable_fp8()                                           # leaves mode 2 as it is
    assert m.fp8_unfused_lora and torch.equal(run(), after)

    # adapter, weight and scale changes touch no e4m3 weight
    snap = {k: (w8.view(torch.uint8).clone(), ws.clone()) for k, (w8, ws) in m._fp8.items()}
    outs = [run(0.3)]
    m.set_adapters(["a", "b"], [0.5, 2.0])
    outs.append(run())
    m.disable_lora()
    outs.append(run())
    m.enable_lora()
    m.delete_adapters("b")
    outs.append(run())
    assert all(not torch.equal(outs[i], outs[i - 1]) for i in range(1, len(outs))), "a change had no effect"
    for k, (w8, ws) in m._fp8.items():
        assert torch.equal(w8.view(torch.uint8), snap[k][0]) and torch.equal(ws, snap[k][1]), k

    # first-block cache: threshold 0 == off; an adapter change invalidates the state
    ref = run()
    m.enable_cache(FirstBlockCacheConfig(0.0))
    assert torch.equal(run(), ref) and torch.equal(run(), ref)
    m.enable_cache(FirstBlockCacheConfig(float("inf")))
    run()
    run()
    assert m.cache_log[-1]["hit"]
    m.set_adapters(["a"], [0.25])
    run()
    assert not m.cache_log[-1]["hit"], "an adapter change must invalidate the first-block cache"
    run(0.1)
    assert not m.cache_log[-1]["hit"], "a scale change must invalidate the first-block cache"
    m.disable_cache()

    # training refuses
    holder = type("M", (), {})()
    holder.denoise_tower = type("Tower", (), {})()
    holder.denoise_tower.denoiser = m
    with pytest.raises(_lib.B2FError):
        FluxTrainGraph(holder, [])
    m.unload_lora()
    with pytest.raises(_lib.B2FError, match="disable_fp8"):
        FluxTrainGraph(holder, [])


@pytest.mark.parametrize("true_cfg", [False, True])
def test_pipeline_fp8_unfused_lora_scale(true_cfg):
    """A pipeline call with joint_attention_kwargs={"scale": s} on FP8 linears with an unfused adapter: its latents are
    closer to the bf16 run with the same adapter than to the FP8 run without it."""
    from gpt_image_edit_b200.flux_transformer import B200FluxTransformer2DModel, FluxTransformerConfig
    from gpt_image_edit_b200.pipeline import FluxKontextPipeline
    from gpt_image_edit_b200.scheduler import FlowMatchEulerDiscreteScheduler
    from gpt_image_edit_b200.vae import B200AutoencoderKL, VaeConfig
    from oracle import flux_oracle as fo
    from oracle import vae_oracle as vo

    TOY = dict(num_layers=2, num_single_layers=2, attention_head_dim=128, num_attention_heads=2,
               joint_attention_dim=256, pooled_projection_dim=64)
    BOC = (64, 128, 256, 256)
    fcfg, vcfg = fo.FluxConfig(**TOY), vo.VaeConfig(block_out_channels=BOC)
    tr = B200FluxTransformer2DModel(FluxTransformerConfig(**TOY))
    tr.load_state_dict(fo.make_synthetic_state_dict(fcfg, seed=3, dtype=torch.bfloat16, device="cuda"))
    vae = B200AutoencoderKL(VaeConfig(block_out_channels=BOC))
    vae.load_state_dict(vo.make_synthetic_state_dict(vcfg, seed=4, dtype=torch.bfloat16, device="cuda"))
    pipe = FluxKontextPipeline(transformer=tr, vae=vae, scheduler=FlowMatchEulerDiscreteScheduler())
    g = torch.Generator().manual_seed(13)
    H = W = 128
    image = (torch.randint(0, 256, (1, 3, H, W), generator=g).float() / 127.5 - 1.0).cuda()
    pe = torch.randn(1, 24, 256, generator=g).bfloat16().cuda()
    pooled = torch.randn(1, 64, generator=g).bfloat16().cuda()
    npe = torch.randn(1, 9, 256, generator=g).bfloat16().cuda()
    npooled = torch.randn(1, 64, generator=g).bfloat16().cuda()
    noise = torch.randn(1, 64, 64, generator=g).bfloat16().cuda()
    common = dict(height=H, width=W, num_inference_steps=3, guidance_scale=3.5, max_area=H * W)
    if true_cfg:
        common.update(negative_prompt_embeds=npe, negative_pooled_prompt_embeds=npooled, true_cfg_scale=4.0)

    def call():
        return pipe(image=image, prompt_embeds=pe, pooled_prompt_embeds=pooled, latents=noise.clone(),
                    _auto_resize=False, output_type="latent", joint_attention_kwargs={"scale": 0.5},
                    **common).images.float()

    pipe.load_lora_weights(LR.to_kohya(fcfg, LR.make_lora(fcfg, rank=8, seed=9, alpha=8.0, a_std=0.1, b_std=0.1)))
    bf16_lora = call()
    tr.enable_fp8(unfused_lora=True)
    fp8_lora = call()
    tr.disable_lora()
    fp8_none = call()
    e_lora, e_none = R.rel_l2(fp8_lora, bf16_lora), R.rel_l2(fp8_none, bf16_lora)
    print(f"pipeline fp8 + unfused lora (true_cfg={true_cfg}): rel-L2 to bf16 + lora {e_lora:.3e}, "
          f"FP8 without the adapter {e_none:.3e}")
    assert torch.isfinite(fp8_lora).all() and e_lora < 0.5 * e_none
