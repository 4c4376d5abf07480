"""The FLUX VAE at every preferred Kontext resolution, and the pipeline resizing a context image onto one.

Six of the seventeen resolutions (720x1456, 752x1392, 944x1104 and their transposes) have a latent pixel count that is
not a multiple of 8 (P = 16380, 16356, 16284), so the mid-block attention runs on padded keys there.
"""
import numpy as np
import pytest
import torch

from gpt_image_edit_b200.pipeline import PREFERRED_KONTEXT_RESOLUTIONS
from oracle import vae_oracle as vo

pytestmark = pytest.mark.gpu


def _rel_l2(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-20)).item()


@pytest.fixture(scope="module")
def full_vae():
    from gpt_image_edit_b200.vae import B200AutoencoderKL, VaeConfig

    ocfg = vo.VaeConfig()
    sd = vo.make_synthetic_state_dict(ocfg, seed=0, dtype=torch.bfloat16, device="cuda")
    vae = B200AutoencoderKL(VaeConfig())
    vae.load_state_dict(sd)
    return ocfg, sd, {k: v.float() for k, v in sd.items()}, vae


@pytest.mark.parametrize("W,H", PREFERRED_KONTEXT_RESOLUTIONS, ids=[f"{w}x{h}" for w, h in PREFERRED_KONTEXT_RESOLUTIONS])
def test_vae_at_preferred_kontext_resolutions(full_vae, W, H):
    from gpt_image_edit_b200.pipeline import VaeImageProcessor

    ocfg, sd, sd32, vae = full_vae
    g = torch.Generator(device="cuda").manual_seed(W)
    x = (torch.rand(1, 3, H, W, device="cuda", generator=g) * 2 - 1).bfloat16()
    z = torch.randn(1, 16, H // 8, W // 8, device="cuda", generator=g).bfloat16()
    mean = vae.encode(x).latent_dist.mode()
    img = vae.decode(z, return_dict=False)[0]
    u8 = vae.decode_u8(z)
    m32 = vo.encode_mode(sd32, ocfg, x.float())
    e_m, t_m = _rel_l2(mean, m32), _rel_l2(vo.encode_mode(sd, ocfg, x), m32)
    del m32
    i32 = vo.decode(sd32, ocfg, z.float())
    e_i, t_i = _rel_l2(img, i32), _rel_l2(vo.decode(sd, ocfg, z), i32)
    print(f"{W}x{H} P={(H // 8) * (W // 8)}: encode {e_m:.3e} (bf16 {t_m:.3e})  decode {e_i:.3e} (bf16 {t_i:.3e})")
    assert e_m <= 2.0 * t_m + 3e-3 and e_i <= 2.0 * t_i + 3e-3
    assert u8.shape == (1, H, W, 3) and np.array_equal(np.asarray(VaeImageProcessor.postprocess(img, "pil")[0]),
                                                       u8[0].cpu().numpy())


def test_pipeline_auto_resizes_context_onto_a_ragged_latent_grid():
    """A 2:1 context image with `_auto_resize` on is resized to 1456 x 720 (latent 90 x 182) and encoded there."""
    from gpt_image_edit_b200.flux_transformer import B200FluxTransformer2DModel, FluxTransformerConfig
    from gpt_image_edit_b200.pipeline import FluxKontextPipeline
    from gpt_image_edit_b200.scheduler import FlowMatchEulerDiscreteScheduler
    from gpt_image_edit_b200.vae import B200AutoencoderKL, VaeConfig
    from oracle import flux_oracle as fo

    toy = dict(num_layers=1, num_single_layers=1, attention_head_dim=128, num_attention_heads=2,
               joint_attention_dim=256, pooled_projection_dim=64)
    boc = (64, 128, 256, 256)
    fcfg, vcfg = fo.FluxConfig(**toy), vo.VaeConfig(block_out_channels=boc)
    tr = B200FluxTransformer2DModel(FluxTransformerConfig(**toy))
    tr.load_state_dict(fo.make_synthetic_state_dict(fcfg, seed=3, dtype=torch.bfloat16, device="cuda"))
    vae = B200AutoencoderKL(VaeConfig(block_out_channels=boc))
    vae.load_state_dict(vo.make_synthetic_state_dict(vcfg, seed=4, dtype=torch.bfloat16, device="cuda"))
    seen = []
    encode = vae.encode
    vae.encode = lambda x, *a, **k: (seen.append(tuple(x.shape)), encode(x, *a, **k))[1]
    pipe = FluxKontextPipeline(transformer=tr, vae=vae, scheduler=FlowMatchEulerDiscreteScheduler())
    g = torch.Generator().manual_seed(5)
    image = (torch.rand(1, 3, 128, 256, generator=g) * 2 - 1).cuda()
    pe = torch.randn(1, 24, 256, generator=g).bfloat16().cuda()
    pooled = torch.randn(1, 64, generator=g).bfloat16().cuda()
    lat = pipe(image=image, prompt_embeds=pe, pooled_prompt_embeds=pooled, height=128, width=256, num_inference_steps=2,
               max_area=128 * 256, output_type="latent").images
    assert seen and seen[0][-2:] == (720, 1456), seen
    assert lat.shape == (1, 8 * 16, 64) and torch.isfinite(lat.float()).all()
