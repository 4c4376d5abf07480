"""Per-item text windows in the FLUX joint attention, on the GPU: the window kernels (bf16 and FP8), the model's
encoder_attention_mask and the pipeline's prompt_attention_mask.

What a window promises: a batch item computes what it computes alone on its unpadded text, and nothing in its masked
text rows, NaN included, reaches an unmasked output.  So every check here compares an item of a padded batch with the
same code run on that item alone, and both with float64:

  * exact, bit for bit: the full window against the unwindowed kernels; NaN-filled against zero-filled pad rows; the FP8
    scales of an item against those of its run alone;
  * allowance: rel-L2(batch item, alone) <= 1.5 e_alone + 1e-3 and rel-L2(batch item, fp64) <= 1.25 e_alone + 1e-3,
    where e_alone = rel-L2(alone, fp64).  The windowed item may differ from its run alone only in where its 128-key
    blocks start (and so in the order of its fp32 sums and, in FP8, in the running max its probabilities are rounded
    against); an item must be no worse than its run alone against float64.
"""
import math

import pytest
import torch

import lora_ref as LR
from oracle import flux_oracle as fo
from test_train_blocks_gpu import _ids, _synthetic_sd

pytestmark = pytest.mark.gpu

f64, bf16 = torch.float64, torch.bfloat16
H, DH = 2, 128
S_TXT, S_IMG = 300, 200                         # S_txt % 128 != 0, S = 500
# (lo, hi) per item: edges at 0, 1, 127, 128, 129, S_txt - 1 and S_txt, left, right and two-sided padding
WINDOW_SETS = {
    "left_and_two_sided": [(1, S_TXT), (127, 129), (128, S_TXT - 1)],
    "right_and_tiny": [(0, 127), (129, S_TXT), (0, 1)],
}


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-300)).item()


def _gate(name, got, alone, ref):
    e_alone, e_ref, e_diff = _rel(alone, ref), _rel(got, ref), _rel(got, alone)
    print(f"{name}: vs alone {e_diff:.3e} ({'bit-identical' if torch.equal(got, alone) else 'differs'}), "
          f"vs fp64 {e_ref:.3e}, alone vs fp64 {e_alone:.3e}")
    assert torch.isfinite(got).all(), name
    assert e_diff <= 1.5 * e_alone + 1e-3, name
    assert e_ref <= 1.25 * e_alone + 1e-3, name


def _qkv(B, S, g):
    """One qkv [B, S, 3 H 128] buffer as the model holds it (_views splits it into head-split column slices)."""
    return torch.randn(B, S, 3 * H * DH, device="cuda", generator=g).bfloat16()


def _valid_rows(lo, hi):
    return torch.cat([torch.arange(lo, hi), torch.arange(S_TXT, S_TXT + S_IMG)]).cuda()


def _fill_pads(qkv, wins, value):
    out = qkv.clone()
    for b, (lo, hi) in enumerate(wins):
        out[b, :lo] = value
        out[b, hi:S_TXT] = value
    return out


def _attn64(q, k, v):
    """fp64 softmax attention of [S, H, 128] operands."""
    q, k, v = (t.double().transpose(0, 1) for t in (q, k, v))
    p = torch.softmax(q @ k.transpose(1, 2) / math.sqrt(DH), dim=-1)
    return (p @ v).transpose(0, 1).reshape(q.shape[1], H * DH)


def _views(qkv):
    return [qkv[:, :, i * H * DH:(i + 1) * H * DH].unflatten(-1, (H, DH)) for i in range(3)]


def _bf16_attn(qkv, win=None, S_txt=None):
    from gpt_image_edit_b200 import ops

    return ops.attention(*_views(qkv), win=win, S_txt=S_txt)


def _fp8_attn(qkv, win=None, S_txt=None):
    from gpt_image_edit_b200 import ops

    bufs = ops.attn_quant_fp8(*_views(qkv), win=win, S_txt=S_txt)
    return ops.attention_fp8(*bufs, win=win, S_txt=S_txt), bufs


# ---------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
def test_full_window_is_bit_identical_to_the_unwindowed_kernels(fp8):
    g = torch.Generator(device="cuda").manual_seed(1)
    qkv = _qkv(3, S_TXT + S_IMG, g)
    full = torch.tensor([[0, S_TXT]] * 3, dtype=torch.int32, device="cuda")
    if not fp8:
        assert torch.equal(_bf16_attn(qkv, full, S_TXT), _bf16_attn(qkv))
        return
    o_w, b_w = _fp8_attn(qkv, full, S_TXT)
    o, b = _fp8_attn(qkv)
    for x, y in zip(b_w, b):
        assert torch.equal(x.view(torch.uint8), y.view(torch.uint8))
    assert torch.equal(o_w, o)


@pytest.mark.parametrize("wset", list(WINDOW_SETS))
@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
def test_window_items_match_their_runs_alone(fp8, wset):
    wins = WINDOW_SETS[wset]
    B = len(wins)
    g = torch.Generator(device="cuda").manual_seed(2)
    qkv = _qkv(B, S_TXT + S_IMG, g)
    win = torch.tensor(wins, dtype=torch.int32, device="cuda")
    run = (lambda x, *a: _fp8_attn(x, *a)[0]) if fp8 else _bf16_attn
    o_nan = run(_fill_pads(qkv, wins, float("nan")), win, S_TXT)
    o_zero = run(_fill_pads(qkv, wins, 0.0), win, S_TXT)
    o_inf = run(_fill_pads(qkv, wins, float("inf")), win, S_TXT)
    for b, (lo, hi) in enumerate(wins):
        rows = _valid_rows(lo, hi)
        got = o_zero[b, rows]
        assert torch.isfinite(o_nan[b, rows]).all()
        assert torch.equal(o_nan[b, rows], got), f"item {b}: NaN pads reached a valid output"
        assert torch.equal(o_inf[b, rows], got), f"item {b}: Inf pads reached a valid output"
        alone_qkv = qkv[b:b + 1, rows].contiguous()
        alone = run(alone_qkv)[0]
        ref = _attn64(*(t[0] for t in _views(alone_qkv)))
        _gate(f"{'fp8' if fp8 else 'bf16'} {wset} item {b} window ({lo}, {hi})", got, alone, ref)


@pytest.mark.parametrize("wset", list(WINDOW_SETS))
def test_fp8_scales_equal_those_of_the_run_alone(wset):
    from gpt_image_edit_b200 import ops

    wins = WINDOW_SETS[wset]
    g = torch.Generator(device="cuda").manual_seed(3)
    qkv = _qkv(len(wins), S_TXT + S_IMG, g)
    qkv = _fill_pads(qkv, wins, 1e4)          # pads far above every valid value: they must not enter an amax
    win = torch.tensor(wins, dtype=torch.int32, device="cuda")
    q8, k8, sq, sk, v8t, sv = ops.attn_quant_fp8(*_views(qkv), win=win, S_txt=S_TXT)
    for b, (lo, hi) in enumerate(wins):
        rows = _valid_rows(lo, hi)
        _, _, sq1, sk1, _, sv1 = ops.attn_quant_fp8(*_views(qkv[b:b + 1, rows].contiguous()))
        assert torch.equal(sq[b], sq1[0]) and torch.equal(sk[b], sk1[0]) and torch.equal(sv[b], sv1[0])
        pads = torch.cat([torch.arange(0, lo), torch.arange(hi, S_TXT)]).cuda()
        assert not q8.view(torch.uint8)[b, pads].any() and not k8.view(torch.uint8)[b, pads].any()
        # v8t holds the tokens of each 32-token group permuted; masked tokens are +0 wherever they sit
        assert int((v8t.view(torch.uint8)[b] != 0).sum()) <= H * DH * len(rows)


# ---------------------------------------------------------------------------------------------------- model
FULL = dict(attention_head_dim=128, num_attention_heads=24, joint_attention_dim=4096, pooled_projection_dim=768,
            num_layers=2, num_single_layers=2)
LENS = (77, 130, 201)                    # distinct text lengths: S_txt = 201, windows (124, 201), (71, 201), (0, 201)
HL = WL = 8                              # S_img = 128 (target + context image), n_out = 64


def _model(variant):
    from gpt_image_edit_b200.flux_transformer import B200FluxTransformer2DModel, FirstBlockCacheConfig, \
        FluxTransformerConfig

    ocfg = fo.FluxConfig(**FULL)
    model = B200FluxTransformer2DModel(FluxTransformerConfig(**FULL))
    sd = _synthetic_sd(ocfg, 0)
    model.load_state_dict(sd)
    sd64, scale = {k: v.double() for k, v in sd.items()}, None
    if variant == "lora":
        la = LR.make_lora(ocfg, rank=16, seed=11, alpha=32.0, a_std=0.03, b_std=0.03)
        model.load_lora_adapter(LR.to_diffusers(la), adapter_name="a")
        model.set_adapters(["a"], [1.0])
        scale = 0.7
        sd64 = LR.merged(sd, [(la, scale)])
    elif variant == "fp8_linears":
        model.enable_fp8(linears=True)
    elif variant == "fp8_attention":
        model.enable_fp8(linears=False, attention=True)
    elif variant == "cache":
        model.enable_cache(FirstBlockCacheConfig(threshold=0.0))
    return ocfg, model, sd64, scale


def _inputs(ocfg):
    g = torch.Generator(device="cuda").manual_seed(5)
    B, S_img = len(LENS), 2 * HL * WL
    return dict(hs=torch.randn(B, S_img, ocfg.in_channels, device="cuda", generator=g).bfloat16(),
                encs=[torch.randn(1, n, ocfg.joint_attention_dim, device="cuda", generator=g).bfloat16() for n in LENS],
                pooled=torch.randn(B, ocfg.pooled_projection_dim, device="cuda", generator=g).bfloat16(),
                # the engine takes timestep and guidance * 1000 in bf16: values whose products are exact there, so that
                # the fp64 oracle embeds the same numbers
                t=torch.tensor([0.5, 0.25, 0.125], device="cuda").bfloat16(),
                gd=torch.tensor([4.0, 2.0, 1.0], device="cuda"))


def _call(model, hs, enc, pooled, t, gd, mask=None, scale=None):
    jak = {"_b2f_out_rows": HL * WL}
    if scale is not None:
        jak["scale"] = scale
    kw = {} if mask is None else {"encoder_attention_mask": mask}
    return model(hidden_states=hs, encoder_hidden_states=enc, pooled_projections=pooled, timestep=t, guidance=gd,
                 img_ids=_ids(HL, WL), txt_ids=torch.zeros(enc.shape[1], 3, device="cuda", dtype=bf16),
                 joint_attention_kwargs=jak, return_dict=False, **kw)[0]


@pytest.mark.parametrize("variant", ["bf16", "fp8_linears", "fp8_attention", "lora", "cache"])
def test_model_items_match_their_forwards_alone(variant):
    from gpt_image_edit_b200.pipeline import stack_prompt_embeds

    ocfg, model, sd64, scale = _model(variant)
    x = _inputs(ocfg)
    enc, mask = stack_prompt_embeds(x["encs"])
    nan_enc = enc.masked_fill(mask[..., None] == 0, float("nan"))
    with torch.no_grad():
        out = _call(model, x["hs"], enc, x["pooled"], x["t"], x["gd"], mask, scale)
        out_nan = _call(model, x["hs"], nan_enc, x["pooled"], x["t"], x["gd"], mask, scale)
    assert torch.equal(out_nan, out), "NaN pad rows changed an output"
    for b, e in enumerate(x["encs"]):
        one = dict(hs=x["hs"][b:b + 1], pooled=x["pooled"][b:b + 1], t=x["t"][b:b + 1], gd=x["gd"][b:b + 1])
        alone = _call(model, one["hs"], e, one["pooled"], one["t"], one["gd"], scale=scale)[0]
        ref = fo.flux_forward(sd64, ocfg, one["hs"].double(), e.double(), one["pooled"].double(), one["t"],
                              _ids(HL, WL).double(), torch.zeros(e.shape[1], 3, device="cuda", dtype=f64),
                              guidance=one["gd"].double())[0, :HL * WL]
        _gate(f"model {variant} item {b} (L = {e.shape[1]})", out[b], alone, ref)


def test_training_forward_and_batch_mismatch_refuse_a_set_window():
    from gpt_image_edit_b200 import _lib

    from gpt_image_edit_b200.pipeline import stack_prompt_embeds

    ocfg, model, _, _ = _model("bf16")
    x = _inputs(ocfg)
    enc, mask = stack_prompt_embeds(x["encs"])
    lib = _lib.lib
    win = torch.tensor([[124, 201], [71, 201], [0, 201]], dtype=torch.int32, device="cuda")
    dummy = torch.zeros(256, dtype=torch.uint8, device="cuda")
    p = dummy.data_ptr()
    _call(model, x["hs"], enc, x["pooled"], x["t"], x["gd"], mask)      # sets the RoPE tables of S = 201 + 128
    torch.cuda.synchronize()
    # the model clears its window after the forward: the training forward gets as far as the workspace size
    assert lib.b2f_flux_train_forward(model._h, p, p, p, 0, p, 3, 128, 201, 64, p, 0, None) == -6
    assert lib.b2f_flux_set_text_window(model._h, win.data_ptr(), 3) == 0
    try:
        # a set window is refused before the workspace size is looked at
        assert lib.b2f_flux_train_forward(model._h, p, p, p, 0, p, 3, 128, 201, 64, p, 0, None) == -3
        # a forward over another batch size than the window's
        assert lib.b2f_flux_forward(model._h, p, p, p, 0, p, 2, 128, 201, 64, p, 1 << 40, 0, -1, None) == -1
    finally:
        assert lib.b2f_flux_set_text_window(model._h, None, 0) == 0
    assert lib.b2f_flux_train_forward(model._h, p, p, p, 0, p, 3, 128, 201, 64, p, 0, None) == -6
    assert lib.b2f_flux_set_text_window(model._h, win.data_ptr(), 0) == -1
    with pytest.raises(_lib.B2FError, match="encoder_attention_mask"):   # refused before anything is set
        _call(model, x["hs"], enc, x["pooled"], x["t"], x["gd"], mask[:2])


# ---------------------------------------------------------------------------------------------------- pipeline
TOY = dict(num_layers=2, num_single_layers=2, attention_head_dim=128, num_attention_heads=2,
           joint_attention_dim=256, pooled_projection_dim=64)
BOC = (64, 128, 256, 256)
PH = PW = 128
STEPS = 3


def _pipe():
    from gpt_image_edit_b200.flux_transformer import B200FluxTransformer2DModel, FluxTransformerConfig
    from gpt_image_edit_b200.pipeline import FluxKontextPipeline
    from gpt_image_edit_b200.scheduler import FlowMatchEulerDiscreteScheduler
    from gpt_image_edit_b200.vae import B200AutoencoderKL, VaeConfig
    from oracle import vae_oracle as vo

    tr = B200FluxTransformer2DModel(FluxTransformerConfig(**TOY))
    tr.load_state_dict(fo.make_synthetic_state_dict(fo.FluxConfig(**TOY), seed=3, dtype=bf16, device="cuda"))
    vae = B200AutoencoderKL(VaeConfig(block_out_channels=BOC))
    vae.load_state_dict(vo.make_synthetic_state_dict(vo.VaeConfig(block_out_channels=BOC), seed=4, dtype=bf16,
                                                     device="cuda"))
    return FluxKontextPipeline(transformer=tr, vae=vae, scheduler=FlowMatchEulerDiscreteScheduler())


def _pipe_inputs(n, seed, lens):
    g = torch.Generator().manual_seed(seed)
    n_tgt = (PH // 16) * (PW // 16)
    return dict(image=(torch.randint(0, 256, (n, 3, PH, PW), generator=g).float() / 127.5 - 1.0).cuda(),
                embeds=[torch.randn(1, L, 256, generator=g).bfloat16().cuda() for L in lens],
                pooled=torch.randn(n, 64, generator=g).bfloat16().cuda(),
                noise=torch.randn(n, n_tgt, 64, generator=g).bfloat16().cuda())


def _sample(pipe, image, pe, pooled, noise, **kw):
    return pipe(image=image, prompt_embeds=pe, pooled_prompt_embeds=pooled, height=PH, width=PW,
                num_inference_steps=STEPS, guidance_scale=3.5, latents=noise.clone(), max_area=PH * PW,
                _auto_resize=False, output_type="latent", **kw).images


def test_pipeline_all_ones_mask_is_bit_identical_to_no_mask():
    pipe = _pipe()
    x = _pipe_inputs(2, 21, (24, 24))
    pe = torch.cat(x["embeds"])
    plain = _sample(pipe, x["image"], pe, x["pooled"], x["noise"])
    ones = _sample(pipe, x["image"], pe, x["pooled"], x["noise"],
                   prompt_attention_mask=torch.ones(2, 24, dtype=torch.int64, device="cuda"))
    assert torch.equal(ones, plain)


@pytest.mark.parametrize("true_cfg", [1.0, 4.0], ids=["plain", "true_cfg"])
def test_pipeline_ragged_batch_matches_separate_calls(true_cfg):
    """B = 3 instructions of lengths 24, 9 and 17 in one call against three calls; with true CFG the negative prompts
    are ragged too (lengths 5, 12, 12) and take their own mask."""
    from gpt_image_edit_b200.pipeline import stack_prompt_embeds

    pipe = _pipe()
    x = _pipe_inputs(3, 22, (24, 9, 17))
    neg = _pipe_inputs(3, 23, (5, 12, 12))
    pe, mask = stack_prompt_embeds(x["embeds"])
    kw = {}
    if true_cfg > 1:
        npe, nmask = stack_prompt_embeds(neg["embeds"])
        kw = dict(true_cfg_scale=true_cfg, negative_prompt_embeds=npe, negative_pooled_prompt_embeds=neg["pooled"],
                  negative_prompt_attention_mask=nmask)
    batch = _sample(pipe, x["image"], pe, x["pooled"], x["noise"], prompt_attention_mask=mask, **kw)
    for b in range(3):
        kb = {}
        if true_cfg > 1:
            kb = dict(true_cfg_scale=true_cfg, negative_prompt_embeds=neg["embeds"][b],
                      negative_pooled_prompt_embeds=neg["pooled"][b:b + 1])
        alone = _sample(pipe, x["image"][b:b + 1], x["embeds"][b], x["pooled"][b:b + 1], x["noise"][b:b + 1], **kb)
        e = _rel(batch[b], alone[0])
        print(f"pipeline {'true-CFG' if true_cfg > 1 else 'plain'} item {b}: latents rel-L2 vs the call alone {e:.3e} "
              f"({'bit-identical' if torch.equal(batch[b], alone[0]) else 'differs'})")
        assert torch.isfinite(batch[b]).all()
        assert e <= 5e-3, "a ragged batch item drifted from its call alone beyond the allowance"
    if true_cfg > 1:   # the negative branch really used its windows: without them the pads join its attention
        unmasked = _sample(pipe, x["image"], pe, x["pooled"], x["noise"], prompt_attention_mask=mask,
                           true_cfg_scale=true_cfg, negative_prompt_embeds=kw["negative_prompt_embeds"],
                           negative_pooled_prompt_embeds=neg["pooled"])
        assert not torch.equal(unmasked, batch)


def test_pipeline_mask_shape_is_checked():
    pipe = _pipe()
    x = _pipe_inputs(1, 24, (24,))
    with pytest.raises(ValueError, match="prompt_attention_mask"):
        _sample(pipe, x["image"], x["embeds"][0], x["pooled"], x["noise"],
                prompt_attention_mask=torch.ones(1, 23, dtype=torch.int64, device="cuda"))
