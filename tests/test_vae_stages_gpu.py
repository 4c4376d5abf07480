"""The FLUX VAE's encode and decode checked stage by stage, at full width and at ragged latent sizes, against float64
references of the oracle per pixel, per channel and per GroupNorm group (tests/vae_stage_ref.py).

`B200AutoencoderKL.stage_output` runs the engine's own encode / decode and stops after stage k (`b2f_vae_set_stop_stage`).
Stage k's reference is fed the engine's stage k - 1 output, with torch-bf16 of the same stage as the yardstick: the
per-tensor rule rel-L2(engine) <= 2 rel-L2(bf16) + 1e-2 and the per-slice gate max_s e_s <= 2 max_s y_s + 1e-3
(`infer_block_ref.BETA`).  Stages whose input and output have the same shape (the ResnetBlock2Ds without a shortcut
GEMM and the mid-block attention) are also gated on their own share, output - input.
"""
import pytest
import torch
import torch.nn.functional as F

import vae_stage_ref as VS
from oracle import vae_oracle as vo

pytestmark = pytest.mark.gpu

f64, bf16 = torch.float64, torch.bfloat16
FULL = (128, 256, 512, 512)
TOY = (64, 128, 256, 256)

# name: (block_out_channels, N, H, W)
CASES = {
    "ragged_13x21": (FULL, 2, 104, 168),       # latent 13 x 21, P = 273: odd grids after every downsample
    "kontext_720x1456": (FULL, 1, 720, 1456),  # a preferred Kontext resolution: latent 90 x 182, P = 16380
    "toy_40x56": (TOY, 1, 40, 56),             # P = 35, padded to 40
    "toy_64x96": (TOY, 1, 64, 96),             # P = 96, no padding
}


def _vae(boc, seed=0):
    from gpt_image_edit_b200.vae import B200AutoencoderKL, VaeConfig

    ocfg = vo.VaeConfig(block_out_channels=boc)
    sd = vo.make_synthetic_state_dict(ocfg, seed=seed, dtype=bf16, device="cuda")
    vae = B200AutoencoderKL(VaeConfig(block_out_channels=boc))
    vae.load_state_dict(sd)
    return ocfg, sd, vae


def _inputs(side, N, H, W, g):
    """items of different scale and offset"""
    if side == "encoder":
        x = torch.rand(N, 3, H, W, device="cuda", generator=g) * 2 - 1
        a, b = (1.0, 0.4), (0.0, 0.3)
    else:
        x = torch.randn(N, 16, H // 8, W // 8, device="cuda", generator=g)
        a, b = (1.0, 2.5), (0.0, -0.7)
    return (x * torch.tensor(a[:N], device="cuda").view(N, 1, 1, 1) +
            torch.tensor(b[:N], device="cuda").view(N, 1, 1, 1)).bfloat16()


def _report(title, checks):
    print(f"\n[{title}]")
    print("\n".join(str(c) for c in checks))
    return [str(c) for c in checks if not c.ok]


@pytest.mark.parametrize("case,side", [(c, s) for c in CASES for s in ("encoder", "decoder")])
def test_stagewise_vae_matches_fp64(case, side):
    boc, N, H, W = CASES[case]
    ocfg, sd, vae = _vae(boc)
    x = _inputs(side, N, H, W, torch.Generator(device="cuda").manual_seed(3))
    checks = []
    x_in = x
    for k, st in enumerate(VS.stages(ocfg, side), 1):
        K = vae.stage_output(x, side, k)
        R = VS.run_stage(sd, st, x_in, f64)
        Y = VS.run_stage(sd, st, x_in, bf16)
        assert K.shape == R.shape, (st[0], K.shape, R.shape)
        checks += VS.stage_gates(f"{side[:3]} {k}", st[0], K, R, Y, base=x_in if x_in.shape == K.shape else None)
        del R, Y
        x_in = K
    # the stagewise runs end where one call ends
    full = vae.encode(x).latent_dist.parameters if side == "encoder" else vae.decode(x, return_dict=False)[0]
    assert torch.equal(full, x_in)
    bad = _report(f"{case} {side} N={N} {H}x{W} widths {boc}", checks)
    assert not bad, "\n".join(bad)


def test_peaked_mid_attention_matches_fp64():
    """The decoder's mid-block attention alone at latent 90 x 182 (P = 16380), with to_q and to_k scaled so the scaled
    logits have a standard deviation of about 4: peaked softmax rows, where rounding the logits shows most.  The weights
    are constructed, not taken from a checkpoint."""
    ocfg, sd, vae = _vae(FULL)
    z = _inputs("decoder", 1, 720, 1456, torch.Generator(device="cuda").manual_seed(4))
    x_in = vae.stage_output(z, "decoder", 2)                     # mid_block.resnets.0: the attention's input
    a, C = "decoder.mid_block.attentions.0", FULL[-1]

    def logits(w):
        h = F.group_norm(x_in.double().flatten(2), 32, w[f"{a}.group_norm.weight"].double(),
                         w[f"{a}.group_norm.bias"].double(), eps=1e-6).transpose(1, 2)
        q = F.linear(h, w[f"{a}.to_q.weight"].double(), w[f"{a}.to_q.bias"].double())
        k = F.linear(h, w[f"{a}.to_k.weight"].double(), w[f"{a}.to_k.bias"].double())
        return (q @ k.transpose(1, 2)) * C ** -0.5

    s0 = logits(sd).std().item()
    f = (4.0 / s0) ** 0.5
    sd = dict(sd)
    for n in ("to_q", "to_k"):
        for p in ("weight", "bias"):
            sd[f"{a}.{n}.{p}"] = (sd[f"{a}.{n}.{p}"].double() * f).bfloat16()
    vae.load_state_dict(sd)
    s = logits(sd)
    std, peak = s.std().item(), torch.softmax(s, -1).amax(-1).mean().item()
    del s
    st = VS.stages(ocfg, "decoder")[2]
    assert st[0] == a
    K = vae.stage_output(z, "decoder", 3)
    R = VS.run_stage(sd, st, x_in, f64)
    Y = VS.run_stage(sd, st, x_in, bf16)
    h = F.group_norm(x_in.flatten(2), 32, sd[f"{a}.group_norm.weight"], sd[f"{a}.group_norm.bias"], eps=1e-6).transpose(1, 2)
    qkv = [F.linear(h, sd[f"{a}.{n}.weight"], sd[f"{a}.{n}.bias"])[:, None] for n in ("to_q", "to_k", "to_v")]
    print(f"\nscaled logits: std {std:.2f} (unscaled weights {s0:.2f}), mean row max of the softmax {peak:.3f}; "
          f"yardstick SDPA backend: {VS.sdpa_backend(*qkv)}")
    assert 3.5 < std < 4.5
    checks = VS.stage_gates("attn", a, K, R, Y, base=x_in)
    bad = _report("peaked decoder mid attention, latent 90x182", checks)
    assert not bad, "\n".join(bad)
