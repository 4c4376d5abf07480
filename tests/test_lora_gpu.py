"""LoRA on the GPU: the K-extended GEMM element by element, exact properties of whole forwards, the model against the
fp64 oracle on merged weights, the pipeline surface, and the training refusal.

K-extended GEMM: the down projection T = bf16(fp32(x Acat^T) * fp32(colscale * cs_mul)) is checked against its own
emulation, then out = epi(x W^T + T Bcat^T + b) against kernel_ref's emulation of the plain GEMM on the concatenated
operands [x | T] and [W | Bcat] — the K-extension is exactly that contraction, in one fp32 accumulation.
"""
import pytest
import torch

import kernel_ref as R
import lora_ref as LR
import train_block_ref as TB

pytestmark = pytest.mark.gpu

TH_GEMM = dict(max_ulp=2, share_gt1=1e-3, mean_ulp=0.1)   # as in test_sm90_edges_gpu.py
TOY = dict(num_layers=2, num_single_layers=2, attention_head_dim=128, num_attention_heads=2,
           joint_attention_dim=256, pooled_projection_dim=64)
FULL = dict(num_layers=2, num_single_layers=2)            # d = 3072, the real embedder widths


def _g(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _bf(*shape, g, scale=1.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).bfloat16()


def _adapters(K, N, ranks, scales, g):
    """Two (or more) adapters concatenated: Acat [r_pad, K], Bcat [N, r_pad], colscale [r_pad] (zero padded)."""
    R_ = sum(ranks)
    r_pad = -(-R_ // 64) * 64
    acat = torch.zeros(r_pad, K, device="cuda", dtype=torch.bfloat16)
    bcat = torch.zeros(N, r_pad, device="cuda", dtype=torch.bfloat16)
    cs = torch.zeros(r_pad, device="cuda")
    c = 0
    for r, s in zip(ranks, scales):
        acat[c:c + r] = _bf(r, K, g=g, scale=K ** -0.5)
        bcat[:, c:c + r] = _bf(N, r, g=g, scale=r ** -0.5)
        cs[c:c + r] = s
        c += r
    return acat, bcat, cs


def _down_checked(c, x, acat, cs, cs_mul):
    from gpt_image_edit_b200 import ops
    t = ops.lora_down(x, acat, cs, cs_mul=cs_mul)
    s_eff = (cs * cs_mul).double()                      # fp32(colscale * cs_mul), as the kernel forms it
    acc = R.linear_math(x, acat)
    floor = R.acc_floor(x.shape[-1], R.linear_absref(x, acat)) * s_eff.abs()
    c.bf16("T", t, R.bf16r(acc * s_eff), floor, dims=("b", "row", "rank")[-t.dim():], **TH_GEMM)
    return t


GEMM_CASES = [  # (ranks of the adapters, batch, M, K, N)
    ((1,), 1, 1, 200, 136),
    ((8,), 1, 127, 136, 256),
    ((24, 16), 2, 129, 192, 384),          # two adapters, total rank 40
    ((64,), 1, 8736, 3072, 384),
    ((40, 25), 3, 129, 72, 264),           # 65: r_pad 128
    ((120, 80), 2, 300, 264, 520),         # 200: r_pad 256
]


@pytest.mark.parametrize("case", range(len(GEMM_CASES)))
@pytest.mark.parametrize("bias", [True, False])
def test_lora_gemm_ranks_and_shapes(case, bias):
    from gpt_image_edit_b200 import ops
    ranks, B, M, K, N = GEMM_CASES[case]
    g = _g(10 + case)
    x, w = _bf(B, M, K, g=g), _bf(N, K, g=g, scale=K ** -0.5)
    b = _bf(N, g=g, scale=0.5) if bias else None
    acat, bcat, cs = _adapters(K, N, ranks, [0.75, -1.5, 2.0][:len(ranks)], g)
    c = R.Checker(f"lora gemm ranks{ranks} B{B} M{M} K{K} N{N} bias={bias}")
    t = _down_checked(c, x, acat, cs, 0.5)
    buf = torch.full((B, M + 2, N + 16), float("nan"), device="cuda", dtype=torch.bfloat16)
    out = buf[:, 1:1 + M, 8:8 + N]
    ops.linear_lora(x, w, b, t, bcat, out=out)
    emu, floor, acc = R.linear_emu(torch.cat([x, t], -1), torch.cat([w, bcat], -1), b)
    c.bf16("out", out, emu, floor, math_ref=acc, rel_l2_max=4e-3, dims=("b", "row", "col"), **TH_GEMM)
    mask = torch.ones_like(buf, dtype=torch.bool)
    mask[:, 1:1 + M, 8:8 + N] = False
    c.equal("outside the view (still NaN)", torch.isnan(buf[mask]), torch.ones_like(buf[mask], dtype=torch.bool))
    c.finish()


@pytest.mark.parametrize("epi", [R.EPI_BIAS, R.EPI_GELU_TANH, R.EPI_GELU_ERF, R.EPI_SILU, R.EPI_QUICK_GELU,
                                 R.EPI_GATE_RESID, R.EPI_RESID])
def test_lora_gemm_every_epilogue(epi):
    """Every forward epilogue on the K-extended GEMM, batched with strided views, residual ones in place."""
    from gpt_image_edit_b200 import ops
    g = _g(100 + epi)
    B, M, K, N = 2, 200, 328, 384
    xb = _bf(B, M, K + 8, g=g)
    x = xb[..., :K]                                       # pitched rows
    w, b = _bf(N, K, g=g, scale=K ** -0.5 * 2), _bf(N, g=g, scale=0.5)
    acat, bcat, cs = _adapters(K, N, (16, 24), (1.0, 0.5), g)
    resid, gate = _bf(B, M, N, g=g), _bf(B, N, g=g)
    c = R.Checker(f"lora gemm epi{epi}")
    t = _down_checked(c, x, acat, cs, 1.0)
    out = torch.empty(B, M, N, device="cuda", dtype=torch.bfloat16)
    if epi in (R.EPI_GATE_RESID, R.EPI_RESID):
        out.copy_(resid)
        ops.linear_lora(x, w, b, t, bcat, epilogue=epi, resid=out, gate=gate if epi == R.EPI_GATE_RESID else None,
                        out=out)
    else:
        ops.linear_lora(x, w, b, t, bcat, epilogue=epi, out=out)
    emu, floor, _ = R.linear_emu(torch.cat([x, t], -1), torch.cat([w, bcat], -1), b, epi, resid=resid, gate=gate)
    c.bf16("out", out, emu, floor, dims=("b", "row", "col"), **TH_GEMM)
    c.finish()


@pytest.mark.parametrize("extra", [False, True])
def test_lora_gemm_qkv_norm_rope(extra):
    """QKV RMSNorm + RoPE (and the single block's GELU'd MLP block with n_extra) on the K-extended GEMM."""
    from gpt_image_edit_b200 import ops
    g = _g(300 + extra)
    B, H, K, M, row0 = 2, 2, 256, 137, 16
    d = H * 128
    n_extra = 4 * d if extra else 0
    x = _bf(B, M, K, g=g)
    w, b = _bf(3 * d + n_extra, K, g=g, scale=K ** -0.5), _bf(3 * d + n_extra, g=g, scale=0.5)
    nq, nk = (_bf(128, g=g, scale=0.1).float() + 1).bfloat16(), (_bf(128, g=g, scale=0.1).float() + 1).bfloat16()
    ang = torch.rand(row0 + M, 64, device="cuda", generator=g) * 6.28
    cos, sin = ang.cos().repeat_interleave(2, 1).contiguous(), ang.sin().repeat_interleave(2, 1).contiguous()
    acat, bcat, cs = _adapters(K, 3 * d + n_extra, (8, 32), (2.0, -0.5), g)
    c = R.Checker(f"lora qkv extra={n_extra}")
    t = _down_checked(c, x, acat, cs, 0.5)
    out = torch.empty(B, M, 3 * d, device="cuda", dtype=torch.bfloat16)
    cat = torch.empty(B, M, d + n_extra, device="cuda", dtype=torch.bfloat16) if extra else None
    ops.linear_qkv_norm_rope_lora(x, w, b, nq, nk, cos, sin, t, bcat, rope_row0=row0, out=out,
                                  out_extra=cat[:, :, d:] if extra else None, epi_extra=ops.EPI_GELU_TANH)
    emu, floor, mth = R.qkv_norm_rope_emu(torch.cat([x, t], -1), torch.cat([w, bcat], -1), b, nq, nk, cos, sin,
                                          rope_row0=row0, n_extra=n_extra, epi_extra=R.EPI_GELU_TANH)
    dims = ("b", "row", "col")
    c.bf16("QKV", out, emu[..., :3 * d], floor[..., :3 * d], dims=dims, **TH_GEMM)
    if extra:
        c.bf16("mlp", cat[:, :, d:], emu[..., 3 * d:], floor[..., 3 * d:], dims=dims, **TH_GEMM)
    c.finish()


def test_lora_fuse_kernel():
    """W' = bf16(W + sum_k fp32(B_k s_k) A_k): within one bf16 rounding of the fp64 merge."""
    from gpt_image_edit_b200 import ops
    g = _g(400)
    w = _bf(300, 200, g=g, scale=0.05)
    acat, bcat, cs = _adapters(200, 300, (16, 5), (1.0, -2.0), g)
    w2 = w.clone()
    ops.lora_fuse_(w2, bcat[:, :21].contiguous(), acat[:21].contiguous(), cs[:21].contiguous(), cs_mul=0.5)
    ref = R.d64(w) + R.d64(bcat[:, :21]) @ (R.d64(acat[:21]) * (cs[:21] * 0.5).double()[:, None])
    d = R.ulp_diff(w2, ref, R.acc_floor(21, R.d64(bcat[:, :21]).abs() @ R.d64(acat[:21]).abs()))
    assert d.max().item() <= 1.0, d.max().item()


# ---------------------------------------------------------------------------------------------------- the model
def _model(cfg_kw, seed=3):
    from gpt_image_edit_b200.flux_transformer import B200FluxTransformer2DModel, FluxTransformerConfig
    from oracle import flux_oracle as fo
    fcfg = fo.FluxConfig(**cfg_kw)
    sd = fo.make_synthetic_state_dict(fcfg, seed=seed, dtype=torch.bfloat16, device="cuda")
    m = B200FluxTransformer2DModel(FluxTransformerConfig(**cfg_kw))
    m.load_state_dict(sd)
    return m, sd, fcfg


def _inputs(fcfg, B=1, n=64, S_txt=24, seed=5):
    g = torch.Generator().manual_seed(seed)
    side = int(n ** 0.5)
    ids = torch.stack([torch.zeros(n), torch.arange(n) // side, torch.arange(n) % side], 1)
    ctx = ids.clone()
    ctx[:, 0] = 1
    return dict(hidden_states=torch.randn(B, 2 * n, fcfg.in_channels, generator=g).bfloat16().cuda(),
                encoder_hidden_states=torch.randn(B, S_txt, fcfg.joint_attention_dim, generator=g).bfloat16().cuda(),
                pooled_projections=torch.randn(B, fcfg.pooled_projection_dim, generator=g).bfloat16().cuda(),
                # t = 0.5 and guidance 4.0 survive the bf16 `x * 1000` chain exactly, so the fp64 reference sees the same
                # sinusoid inputs as the bf16 runs (see test_flux_gpu._setup)
                timestep=torch.full((B,), 0.5).bfloat16().cuda(), img_ids=torch.cat([ids, ctx]).bfloat16().cuda(),
                txt_ids=torch.zeros(S_txt, 3).bfloat16().cuda(), guidance=torch.full((B,), 4.0).cuda())


def _run(m, inp, scale=None):
    jak = None if scale is None else {"scale": scale}
    return m(**inp, joint_attention_kwargs=jak, return_dict=False)[0].clone()


def test_exact_properties_whole_forward():
    """Bit for bit over whole toy forwards: B = 0, call scale 0, load -> unload, fuse -> unfuse, three layouts."""
    m, sd, fcfg = _model(TOY)
    inp = _inputs(fcfg)
    base = _run(m, inp)
    lora = LR.make_lora(fcfg, rank=8, seed=1, alpha=16.0)
    zero_b = {n: (A, torch.zeros_like(B), a) for n, (A, B, a) in lora.items()}
    m.load_lora_adapter(LR.to_diffusers(zero_b), adapter_name="zero")
    assert m.lora_unfused_active()
    assert torch.equal(_run(m, inp), base), "an adapter with B = 0 changed the output"
    m.delete_adapters("zero")
    m.load_lora_adapter(LR.to_diffusers(lora), adapter_name="a")
    on = _run(m, inp)
    assert not torch.equal(on, base)
    assert torch.equal(_run(m, inp, scale=0.0), base), "call scale 0 changed the output"
    assert torch.equal(_run(m, inp, scale=1.0), on)
    m.unload_lora()
    assert not m.lora_unfused_active()
    assert torch.equal(_run(m, inp), base), "load -> unload changed the output"
    # fuse -> unfuse restores every weight bit for bit
    before = {k: v.clone() for k, v in m.state_dict().items()}
    m.load_lora_adapter(LR.to_diffusers(lora), adapter_name="a")
    m.fuse_lora(lora_scale=0.8)
    assert not m.lora_unfused_active()
    changed = [k for k, v in m.state_dict().items() if not torch.equal(v, before[k])]
    assert len(changed) == len(lora), (len(changed), len(lora))      # every adapted weight, nothing else
    m.unfuse_lora()
    for k, v in m.state_dict().items():
        assert torch.equal(v, before[k]), k
    assert torch.equal(_run(m, inp), on)
    m.unload_lora()
    # the same adapter in the three layouts: equal outputs
    outs = []
    for sd_l in (LR.to_diffusers(lora), LR.to_bfl(fcfg, lora), LR.to_kohya(fcfg, lora)):
        m.load_lora_adapter(sd_l, adapter_name="x")
        outs.append(_run(m, inp, scale=0.7))
        m.delete_adapters("x")
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


def test_adapter_bookkeeping_rules():
    """A second load joins the active set with weight 1; set_adapters replaces it; disable / enable; weights scale."""
    m, sd, fcfg = _model(TOY)
    inp = _inputs(fcfg)
    la = LR.make_lora(fcfg, rank=4, seed=1, modules=["transformer_blocks.0.attn.to_q", "proj_out"])
    lb = LR.make_lora(fcfg, rank=4, seed=2, modules=["single_transformer_blocks.1.proj_out", "norm_out.linear"])
    m.load_lora_adapter(LR.to_diffusers(la), adapter_name="a")
    only_a = _run(m, inp)
    m.load_lora_adapter(LR.to_diffusers(lb), adapter_name="b")
    assert m.get_active_adapters() == ["a", "b"] and m.get_list_adapters() == {"transformer": ["a", "b"]}
    both = _run(m, inp)
    m.set_adapters(["a"])
    assert m.get_active_adapters() == ["a"] and torch.equal(_run(m, inp), only_a)
    m.set_adapters(["a", "b"], [1.0, 1.0])
    assert torch.equal(_run(m, inp), both)
    m.disable_lora()
    base = _run(m, inp)
    m.enable_lora()
    assert torch.equal(_run(m, inp), both) and not torch.equal(base, both)
    with pytest.raises(ValueError):
        m.set_adapters(["nope"])
    with pytest.raises(ValueError):
        m.load_lora_adapter(LR.to_diffusers(la), adapter_name="a")


def _model_case(cfg_kw, n, S_txt, rank, std):
    from oracle import flux_oracle as fo
    m, sd, fcfg = _model(cfg_kw)
    inp = _inputs(fcfg, B=2, n=n, S_txt=S_txt)
    base = _run(m, inp)
    la = LR.make_lora(fcfg, rank=rank, seed=11, alpha=2.0 * rank, a_std=std, b_std=std)   # every linear target
    lb = LR.make_lora(fcfg, rank=rank // 2, seed=12, alpha=None, a_std=std, b_std=std, modules=[
        "transformer_blocks.0.attn.add_k_proj", "transformer_blocks.1.norm1_context.linear", "x_embedder",
        "time_text_embed.guidance_embedder.linear_2", "single_transformer_blocks.0.proj_mlp", "norm_out.linear"])
    s, wb = 0.6, 0.5
    m.load_lora_adapter(LR.to_diffusers(la), adapter_name="a")
    m.load_lora_adapter(LR.to_bfl(fcfg, lb), adapter_name="b")
    m.set_adapters(["a", "b"], [1.0, wb])
    K_unf = _run(m, inp, scale=s)
    m.fuse_lora(lora_scale=s)
    K_fus = _run(m, inp)
    m.unfuse_lora()
    loras = [(la, s), (lb, s * wb)]
    args = [inp[k] for k in ("hidden_states", "encoder_hidden_states", "pooled_projections", "timestep", "img_ids",
                             "txt_ids")]
    sd64 = LR.merged({k: v.double() for k, v in sd.items()}, loras)
    Rf = fo.flux_forward(sd64, fcfg, *[a.double() for a in args[:3]], args[3].double(), args[4].double(),
                         args[5].double(), guidance=inp["guidance"].double())
    with LR.peft_linear(loras):
        Y = fo.flux_forward(sd, fcfg, *args, guidance=inp["guidance"])
    checks = TB.gate("model", "out unfused", K_unf, Rf, Y, ["rows"]) + \
        TB.gate("model", "out fused", K_fus, Rf, Y, ["rows"])
    for ch in checks:
        print(ch)
    assert all(ch.ok for ch in checks), "\n".join(str(ch) for ch in checks if not ch.ok)
    # the adapters move the output by far more than the bf16 error the comparison allows
    moved, allowed = TB.rel(base, Rf), 2 * TB.rel(Y, Rf) + TB.TENSOR_SLACK
    print(f"no-LoRA output vs the merged reference: {moved:.3e}; allowed error {allowed:.3e}")
    assert moved > 3 * allowed


def test_model_every_target_toy():
    _model_case(TOY, n=64, S_txt=24, rank=8, std=0.05)


def test_model_every_target_full_width():
    _model_case(FULL, n=64, S_txt=32, rank=16, std=0.03)


# ---------------------------------------------------------------------------------------------------- pipeline
@pytest.mark.parametrize("true_cfg", [False, True])
def test_pipeline_load_lora_weights_scale(true_cfg):
    from gpt_image_edit_b200.flux_transformer import B200FluxTransformer2DModel, FluxTransformerConfig
    from gpt_image_edit_b200.pipeline import FluxKontextPipeline
    from gpt_image_edit_b200.scheduler import FlowMatchEulerDiscreteScheduler
    from gpt_image_edit_b200.vae import B200AutoencoderKL, VaeConfig
    from oracle import flux_oracle as fo
    from oracle import pipeline_oracle as po
    from oracle import vae_oracle as vo

    BOC = (64, 128, 256, 256)
    fcfg, vcfg = fo.FluxConfig(**TOY), vo.VaeConfig(block_out_channels=BOC)
    fsd = fo.make_synthetic_state_dict(fcfg, seed=3, dtype=torch.bfloat16, device="cuda")
    vsd = vo.make_synthetic_state_dict(vcfg, seed=4, dtype=torch.bfloat16, device="cuda")
    tr = B200FluxTransformer2DModel(FluxTransformerConfig(**TOY))
    tr.load_state_dict(fsd)
    vae = B200AutoencoderKL(VaeConfig(block_out_channels=BOC))
    vae.load_state_dict(vsd)
    pipe = FluxKontextPipeline(transformer=tr, vae=vae, scheduler=FlowMatchEulerDiscreteScheduler())
    lora = LR.make_lora(fcfg, rank=8, seed=9, alpha=8.0, a_std=0.1, b_std=0.1)
    pipe.load_lora_weights(LR.to_kohya(fcfg, lora))
    with pytest.raises(ValueError):
        pipe.fuse_lora(components=["transformer", "text_encoder"])
    g = torch.Generator().manual_seed(13)
    H = W = 128
    image = (torch.randint(0, 256, (1, 3, H, W), generator=g).float() / 127.5 - 1.0).cuda()
    pe = torch.randn(1, 24, 256, generator=g).bfloat16().cuda()
    pooled = torch.randn(1, 64, generator=g).bfloat16().cuda()
    npe = torch.randn(1, 9, 256, generator=g).bfloat16().cuda()
    npooled = torch.randn(1, 64, generator=g).bfloat16().cuda()
    noise = torch.randn(1, 64, 64, generator=g).bfloat16().cuda()
    common = dict(height=H, width=W, num_inference_steps=3, guidance_scale=3.5, max_area=H * W)
    cfg_kw = dict(negative_prompt_embeds=npe, negative_pooled_prompt_embeds=npooled, true_cfg_scale=4.0) if true_cfg \
        else {}
    lat = pipe(image=image, prompt_embeds=pe, pooled_prompt_embeds=pooled, latents=noise.clone(), _auto_resize=False,
               output_type="latent", joint_attention_kwargs={"scale": 0.5}, **cfg_kw, **common).images
    merged = {k: v.bfloat16() for k, v in LR.merged({k: v.double() for k, v in fsd.items()}, [(lora, 0.5)]).items()}
    ocfg = dict(true_cfg_scale=4.0, negative_prompt_embeds=npe, negative_pooled=npooled) if true_cfg else {}
    ref = po.sample(merged, fcfg, vsd, vcfg, image.bfloat16(), pe, pooled, latents=noise.clone(), output="latent",
                    **ocfg, **common)
    base = po.sample(fsd, fcfg, vsd, vcfg, image.bfloat16(), pe, pooled, latents=noise.clone(), output="latent",
                     **ocfg, **common)
    e = ((lat.float() - ref.float()).norm() / ref.float().norm()).item()
    e_base = ((base.float() - ref.float()).norm() / ref.float().norm()).item()
    print(f"pipeline + LoRA (true_cfg={true_cfg}): latents rel-L2 vs oracle on merged weights {e:.3e}; "
          f"the adapter moves the oracle by {e_base:.3e}")
    assert e < 2e-2 and e_base > 3 * e


def test_training_refuses_unfused_adapters():
    from types import SimpleNamespace

    from gpt_image_edit_b200 import training as tr
    from gpt_image_edit_b200._lib import B2FError
    m, sd, fcfg = _model(TOY)
    m.load_lora_adapter(LR.to_diffusers(LR.make_lora(fcfg, rank=4, modules=["proj_out"])), adapter_name="a")
    holder = SimpleNamespace(denoise_tower=SimpleNamespace(denoiser=m))
    with pytest.raises(B2FError, match="unfused LoRA"):
        tr.FluxTrainGraph(holder, [])
    m.fuse_lora()                      # fused weights are just weights
    tr.FluxTrainGraph(holder, [])
