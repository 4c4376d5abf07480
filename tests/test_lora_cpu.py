"""LoRA state-dict parsing (gpt_image_edit_b200/lora.py) and the merged-vs-unfused identity, on the host.

  - one synthetic adapter written in the diffusers, BFL and kohya layouts parses to the same (Acat, Bcat, colscale) for
    every engine target: q/k/v given separately (diffusers) and fused (BFL / kohya), a subset (to_q only), the
    norm_out half swap, alpha present and absent;
  - every refusal names the offending keys;
  - the fp64 oracle on merged weights W + s B A equals the unfused form x W^T + s (x A^T) B^T to fp64 round-off.
"""
import pytest
import torch

import lora_ref as LR
from oracle import flux_oracle as fo

pytestmark = pytest.mark.filterwarnings("ignore")


def _cfg(**kw):
    return fo.FluxConfig.toy(num_layers=1, num_single_layers=1, **kw)


def _parse(sd, cfg):
    from gpt_image_edit_b200 import lora as L
    return L.parse(sd, cfg)


def _same(a, b):
    assert list(a) == list(b), (list(a), list(b))
    for t in a:
        for f in ("A", "B", "scale"):
            x, y = getattr(a[t], f), getattr(b[t], f)
            assert x.shape == y.shape and torch.equal(x, y), (t, f)


@pytest.mark.parametrize("alpha", [8.0, None])
def test_three_layouts_parse_identically_every_linear(alpha):
    cfg = _cfg()
    lora = LR.make_lora(cfg, rank=4, seed=1, alpha=alpha)
    d = _parse(LR.to_diffusers(lora), cfg)
    _same(d, _parse(LR.to_diffusers(lora, prefix=""), cfg))
    _same(d, _parse(LR.to_bfl(cfg, lora), cfg))
    _same(d, _parse(LR.to_kohya(cfg, lora), cfg))
    from gpt_image_edit_b200 import lora as L
    assert list(d) == list(L.targets(cfg))              # every linear, AdaLN and embedders included
    dd = cfg.inner_dim
    qkv = d["transformer_blocks.0.attn.qkv"]            # q/k/v given separately -> one block-structured target
    assert qkv.A.shape == (12, dd) and qkv.B.shape == (3 * dd, 12)
    for j, n in enumerate(("to_q", "to_k", "to_v")):
        A, B, _ = lora[f"transformer_blocks.0.attn.{n}"]
        assert torch.equal(qkv.A[4 * j:4 * j + 4], A)
        assert torch.equal(qkv.B[j * dd:(j + 1) * dd, 4 * j:4 * j + 4], B)
        blk = qkv.B[j * dd:(j + 1) * dd].clone()
        blk[:, 4 * j:4 * j + 4] = 0
        assert not blk.any()
    sm = d["single_transformer_blocks.0.qkv_mlp"]
    assert sm.A.shape == (16, dd) and sm.B.shape == (7 * dd, 16)
    want = 1.0 if alpha is None else alpha / 4
    assert torch.equal(qkv.scale, torch.full((12,), want))
    # norm_out: the BFL rows are swapped back to diffusers' (scale, shift)
    assert torch.equal(d["norm_out.linear"].B, lora["norm_out.linear"][1])


def test_subset_to_q_only_and_alpha_mix():
    cfg = _cfg()
    lora = LR.make_lora(cfg, rank=8, seed=2, alpha=4.0,
                        modules=["transformer_blocks.0.attn.to_q", "single_transformer_blocks.0.proj_mlp",
                                 "norm_out.linear", "x_embedder"])
    lora["x_embedder"] = (*lora["x_embedder"][:2], None)
    d = _parse(LR.to_diffusers(lora), cfg)
    _same(d, _parse(LR.to_bfl(cfg, lora), cfg))
    _same(d, _parse(LR.to_kohya(cfg, lora), cfg))
    dd = cfg.inner_dim
    q = d["transformer_blocks.0.attn.qkv"]
    assert q.A.shape == (8, dd) and q.B.shape == (3 * dd, 8) and not q.B[dd:].any()
    m = d["single_transformer_blocks.0.qkv_mlp"]
    assert not m.B[:3 * dd].any() and torch.equal(m.B[3 * dd:], lora["single_transformer_blocks.0.proj_mlp"][1])
    assert torch.equal(d["x_embedder"].scale, torch.ones(8)) and torch.equal(q.scale, torch.full((8,), 0.5))


def _refused(sd, cfg, *needles):
    from gpt_image_edit_b200._lib import B2FError
    with pytest.raises(B2FError) as e:
        _parse(sd, cfg)
    for n in needles:
        assert n in str(e.value), str(e.value)


def test_refusals_name_keys():
    cfg = _cfg()
    base = LR.to_diffusers(LR.make_lora(cfg, rank=4, modules=["proj_out"]))
    t = torch.zeros(4, 8)
    _refused({**base, "text_encoder.text_model.encoder.layers.0.self_attn.q_proj.lora_A.weight": t}, cfg,
             "text-encoder", "text_encoder.text_model")
    _refused({**base, "text_encoder_2.encoder.block.0.layer.0.SelfAttention.q.lora_A.weight": t}, cfg, "text_encoder_2.")
    _refused({**base, "lora_te1_text_model_encoder_layers_0_mlp_fc1.lora_down.weight": t}, cfg, "lora_te1_")
    _refused({**base, "transformer.proj_out.lora_magnitude_vector": torch.zeros(64)}, cfg, "DoRA",
             "lora_magnitude_vector")
    _refused({**base, "diffusion_model.img_in.diff": t}, cfg, ".diff", "img_in.diff")
    _refused({**base, "diffusion_model.img_in.diff_b": t}, cfg, "diffusion_model.img_in.diff_b")
    _refused({**base, "transformer.transformer_blocks.0.attn.norm_q.lora_A.weight": t}, cfg, "norm weights", "norm_q")
    _refused({**base, "diffusion_model.double_blocks.0.img_attn.norm.query_norm.lora_A.weight": t}, cfg, "query_norm")
    _refused({**base, "transformer.transformer_blocks.7.attn.to_q.lora_A.weight": t}, cfg, "not a LoRA",
             "transformer_blocks.7")
    _refused({**base, "transformer.proj_out.lora_A.bias": t}, cfg, "proj_out.lora_A.bias")
    A, B = base["transformer.proj_out.lora_A.weight"], base["transformer.proj_out.lora_B.weight"]
    _refused({"transformer.proj_out.lora_A.weight": A, "transformer.proj_out.lora_B.weight": B[:, :3]}, cfg,
             "ranks disagree", "proj_out")
    _refused({"transformer.proj_out.lora_A.weight": A[:, :64], "transformer.proj_out.lora_B.weight": B}, cfg,
             "do not match", "proj_out")
    _refused({"transformer.proj_out.lora_A.weight": A}, cfg, "without both", "proj_out")


def test_merged_equals_unfused_fp64():
    """fp64 oracle: W + s B A merged == x W^T + s (x A^T) B^T on every linear, to fp64 round-off."""
    cfg = _cfg()
    sd = fo.make_synthetic_state_dict(cfg, seed=3, dtype=torch.float64)
    la = LR.make_lora(cfg, rank=4, seed=4, alpha=8.0)
    lb = LR.make_lora(cfg, rank=3, seed=5, alpha=None, modules=["transformer_blocks.0.attn.to_k", "proj_out",
                                                                 "single_transformer_blocks.0.norm.linear"])
    loras = [(la, 0.7), (lb, -1.3)]
    g = torch.Generator().manual_seed(6)
    B, n, S_txt = 1, 16, 8
    hs = torch.randn(B, n, 64, generator=g, dtype=torch.float64)
    enc = torch.randn(B, S_txt, 256, generator=g, dtype=torch.float64)
    pooled = torch.randn(B, 64, generator=g, dtype=torch.float64)
    img_ids = torch.stack([torch.zeros(n), torch.arange(n) // 4, torch.arange(n) % 4], 1).double()
    txt_ids = torch.zeros(S_txt, 3, dtype=torch.float64)
    t = torch.full((B,), 0.5, dtype=torch.float64)
    gd = torch.full((B,), 3.5, dtype=torch.float64)
    ref = fo.flux_forward(LR.merged(sd, loras), cfg, hs, enc, pooled, t, img_ids, txt_ids, guidance=gd)
    with LR.peft_linear(loras):
        unf = fo.flux_forward(sd, cfg, hs, enc, pooled, t, img_ids, txt_ids, guidance=gd)
    base = fo.flux_forward(sd, cfg, hs, enc, pooled, t, img_ids, txt_ids, guidance=gd)
    err = ((unf - ref).norm() / ref.norm()).item()
    assert err < 1e-12, err
    assert ((base - ref).norm() / ref.norm()).item() > 1e-2      # the adapters do change the output
