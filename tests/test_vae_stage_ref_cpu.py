"""The VAE's stage references (tests/vae_stage_ref.py) on the CPU: chained in float64 they are the oracle's encode and
decode exactly, they follow the engine's stage numbering, and their gates catch one wrong pixel or one wrong GroupNorm
group that a rel-L2 over the whole activation lets through."""
import torch

import vae_stage_ref as VS
from gpt_image_edit_b200.vae import stage_shapes
from oracle import vae_oracle as vo

CFG = vo.VaeConfig(block_out_channels=(32, 64, 64, 64), layers_per_block=1, latent_channels=4)


def _sd():
    return vo.make_synthetic_state_dict(CFG, seed=2, dtype=torch.float64)


def test_chained_stages_are_the_oracle():
    sd = _sd()
    g = torch.Generator().manual_seed(0)
    x = torch.rand(2, 3, 40, 24, generator=g, dtype=torch.float64) * 2 - 1
    enc = VS.chain(sd, CFG, "encoder", x)
    mean, logvar = vo.encode_moments(sd, CFG, x)
    assert torch.equal(enc[-1][:, :4], mean) and torch.equal(enc[-1][:, 4:].clamp(-30.0, 20.0), logvar)
    z = torch.randn(2, 4, 5, 3, generator=g, dtype=torch.float64)
    assert torch.equal(VS.chain(sd, CFG, "decoder", z)[-1], vo.decode(sd, CFG, z))


def test_stage_numbering_matches_the_engine():
    full = vo.VaeConfig()
    for cfg in (CFG, full):
        L = cfg.layers_per_block
        for side, n, hw in (("encoder", 4 * L + 8, (40, 56)), ("decoder", 4 * L + 12, (5, 7))):
            ref = VS.stages(cfg, side)
            eng = stage_shapes(cfg, side, *hw)
            assert len(ref) == len(eng) == n, (side, len(ref), len(eng))
            assert [s[0] for s in ref] == [e[0] for e in eng]
    # the shapes the engine's helper reads back are the shapes the references produce
    sd = _sd()
    x = torch.rand(1, 3, 40, 56, dtype=torch.float64)
    for out, (_, c, h, w) in zip(VS.chain(sd, CFG, "encoder", x), stage_shapes(CFG, "encoder", 40, 56)):
        assert tuple(out.shape) == (1, c, h, w)
    z = torch.randn(1, 4, 5, 7, dtype=torch.float64)
    for out, (_, c, h, w) in zip(VS.chain(sd, CFG, "decoder", z), stage_shapes(CFG, "decoder", 5, 7)):
        assert tuple(out.shape) == (1, c, h, w)


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def test_gates_catch_one_pixel_and_one_group():
    """An 'engine' that is the reference rounded to bf16 passes every gate; the same with one border pixel or one
    GroupNorm group of one item off by a few percent fails its slice gate, while the whole-tensor rel-L2 rule that
    test_vae_gpu.py applies (e <= 2 y + 3e-3) still passes it."""
    sd = _sd()
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(2, 64, 24, 40, generator=g) * torch.tensor([1.0, 3.0]).view(2, 1, 1, 1)).bfloat16()
    st = VS.stages(CFG, "decoder")[2]                    # decoder.mid_block.attentions.0
    assert st[0] == "decoder.mid_block.attentions.0"
    R = VS.run_stage(sd, st, x, torch.float64)
    Y = VS.run_stage(sd, st, x, torch.bfloat16)
    K = R.bfloat16()
    assert all(c.ok for c in VS.stage_gates("attn", "x", K, R, Y, base=x)), "bf16 rounding must pass"
    scale = R.pow(2).mean().sqrt()
    bad_pixel = K.clone()
    bad_pixel[1, :, 23, 39] += (0.05 * scale).bfloat16()              # bottom-right corner of item 1
    bad_group = K.clone()
    bad_group[0, 2 * 5:2 * 6] *= 1.03                                 # group 5 of item 0 (2 channels per group)
    for what, Kb, kind in (("pixel", bad_pixel, "rows"), ("group", bad_group, "chunks")):
        e_k, e_t = _rel(Kb, R), _rel(Y, R)
        assert e_k <= 2 * e_t + 3e-3, f"{what}: the whole-tensor rule should not see it ({e_k:.2e} vs {e_t:.2e})"
        failed = [c for c in VS.stage_gates("attn", "x", Kb, R, Y, base=x) if not c.ok]
        assert any(c.kind == kind for c in failed), f"{what}: " + "\n".join(map(str, failed))
        if what == "pixel":
            assert any("item 1 pixel (y 23, x 39)" in c.where for c in failed)
        else:
            assert any("item 0 group 5" in c.where for c in failed)
