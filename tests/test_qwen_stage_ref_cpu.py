"""The Qwen2.5-VL stage references (tests/qwen_stage_ref.py) on the CPU: the float64 oracle is transformers'
Qwen2_5_VLModel in float64 at ragged image grids, the float64 stages chain to the oracle bit for bit, the bf16 yardstick
passes its own gates, and the per-slice gates catch five planted faults of the kinds the engine's host code could make.
"""
import pytest
import torch

import qwen_stage_ref as QS
from gpt_image_edit_b200.qwen2p5vl import QwenTextConfig, QwenVisionConfig, get_rope_index
from oracle import qwen_oracle as qo

hf = pytest.importorskip("transformers.models.qwen2_5_vl.modeling_qwen2_5_vl")

f64, bf16 = torch.float64, torch.bfloat16
IMG, VSTART, VEND = 900, 902, 903
TC = QwenTextConfig(hidden_size=256, num_hidden_layers=2, num_attention_heads=2, num_key_value_heads=1, intermediate_size=512,
                    vocab_size=1000, image_token_id=IMG, video_token_id=901, vision_start_token_id=VSTART)
VC = QwenVisionConfig(depth=4, hidden_size=320, num_heads=4, intermediate_size=340, out_hidden_size=256,
                      fullatt_block_indexes=(1, 3))
GRIDS = {
    "1000x1500": [(1, 26, 38)],            # windows of 64, 48, 16 and 12 patches
    "1456x720": [(1, 44, 22)],             # windows of 64, 48, 32 and 24 patches
    "two_images": [(1, 26, 38), (1, 2, 2)],  # a 4-patch image: one window of 4, one merged token
}


def _prompt(grid, text=(11, 12, 13), tail=(20, 21, 22, 23)):
    ids = list(text)
    for t, h, w in grid:
        ids += [VSTART] + [IMG] * (t * h * w // 4) + [VEND, 5]
    return torch.tensor([ids + list(tail)])


def _pixels(grid, seed=0):
    T = sum(t * h * w for t, h, w in grid)
    return torch.randn(T, 3 * 2 * 14 * 14, generator=torch.Generator().manual_seed(seed), dtype=f64)


def _pos(ids, grid):
    return get_rope_index(ids, torch.tensor(grid), None, spatial_merge_size=2, image_token_id=IMG,
                          vision_start_token_id=VSTART)[0]


def _transformers_fp64(monkeypatch, sd):
    """transformers' Qwen2_5_VLModel in float64 with the oracle's weights.  Its RMSNorm, vision RoPE and rotary angles
    compute in float32 whatever the model's dtype; those casts are lifted to the input dtype here, so that the
    comparison is float64 throughout."""
    from transformers.models.qwen2_5_vl.configuration_qwen2_5_vl import Qwen2_5_VLConfig

    def rms(self, x):
        return self.weight * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + self.variance_epsilon))

    def rope_vision(q, k, cos, sin):
        cos, sin = cos.unsqueeze(-2), sin.unsqueeze(-2)
        return q * cos + hf.rotate_half(q) * sin, k * cos + hf.rotate_half(k) * sin

    def rope_text(self, x, position_ids):
        inv = self.inv_freq[None, None, :, None].expand(3, position_ids.shape[1], -1, 1)
        freqs = (inv @ position_ids[:, :, None, :].to(inv.dtype)).transpose(2, 3)
        emb = torch.cat((freqs, freqs), dim=-1)
        return emb.cos().to(x.dtype), emb.sin().to(x.dtype)

    monkeypatch.setattr(hf.Qwen2_5_VLRMSNorm, "forward", rms)
    monkeypatch.setattr(hf, "apply_rotary_pos_emb_vision", rope_vision)
    monkeypatch.setattr(hf.Qwen2_5_VLRotaryEmbedding, "forward", rope_text)
    tcd = dict(hidden_size=TC.hidden_size, num_hidden_layers=TC.num_hidden_layers, num_attention_heads=TC.num_attention_heads,
               num_key_value_heads=TC.num_key_value_heads, intermediate_size=TC.intermediate_size, vocab_size=TC.vocab_size,
               rms_norm_eps=TC.rms_norm_eps, rope_parameters=dict(rope_type="default", rope_theta=TC.rope_theta,
                                                                  mrope_section=list(TC.mrope_section)))
    vcd = dict(depth=VC.depth, hidden_size=VC.hidden_size, num_heads=VC.num_heads, intermediate_size=VC.intermediate_size,
               out_hidden_size=VC.out_hidden_size, fullatt_block_indexes=list(VC.fullatt_block_indexes))
    cfg = Qwen2_5_VLConfig(text_config=tcd, vision_config=vcd, image_token_id=IMG, video_token_id=901,
                           vision_start_token_id=VSTART, vision_end_token_id=VEND)
    cfg._attn_implementation = "sdpa"
    cfg.vision_config._attn_implementation = cfg.text_config._attn_implementation = "sdpa"
    ref = hf.Qwen2_5_VLModel(cfg).eval().double()
    hsd = {(k.replace("model.", "language_model.", 1) if k.startswith("model.") else k): v for k, v in sd.items()
           if k != "lm_head.weight"}
    missing, unexpected = ref.load_state_dict(hsd, strict=False)
    assert not unexpected and not [k for k in missing if "inv_freq" not in k], (missing, unexpected)
    vd = VC.hidden_size // VC.num_heads // 2
    ref.visual.rotary_pos_emb.inv_freq = 1.0 / 10000.0 ** (torch.arange(0, vd, 2, dtype=f64) / vd)
    hd = TC.hidden_size // TC.num_attention_heads
    ref.language_model.rotary_emb.inv_freq = 1.0 / TC.rope_theta ** (torch.arange(0, hd, 2, dtype=f64) / hd)
    return ref


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


@pytest.mark.parametrize("case", list(GRIDS))
def test_oracle_is_transformers_in_fp64(monkeypatch, case):
    grid = GRIDS[case]
    sd = qo.make_synthetic_state_dict(TC, VC, seed=1, dtype=f64)
    ref = _transformers_fp64(monkeypatch, sd)
    pix, ids = _pixels(grid), _prompt(grid)
    pos = _pos(ids, grid)
    with torch.no_grad():
        v_ref = ref.visual(pix, grid_thw=torch.tensor(grid)).pooler_output
        h_ref = ref(input_ids=ids, pixel_values=pix, image_grid_thw=torch.tensor(grid), position_ids=pos).last_hidden_state
    v = qo.vision_forward(sd, VC, pix, grid)
    h = qo.prefill(sd, TC, VC, ids, pos, pix, grid)
    print(f"\n{case}: vision rel {_rel(v, v_ref):.2e}, prefill rel {_rel(h, h_ref):.2e}")
    assert v.shape == v_ref.shape and _rel(v, v_ref) < 1e-12
    assert h.shape == h_ref.shape and _rel(h, h_ref) < 1e-12
    # the oracle's window order is transformers'
    widx, cu = qo.window_index(grid)
    t_idx, t_cu = ref.visual.get_window_index(torch.tensor(grid))
    assert torch.equal(widx, t_idx) and cu == torch.unique_consecutive(torch.tensor(t_cu)).tolist()


def test_stage_chain_is_the_oracle():
    grid = GRIDS["two_images"]
    sd = qo.make_synthetic_state_dict(TC, VC, seed=2, dtype=f64)
    pix, ids = _pixels(grid, 1), _prompt(grid)
    x = QS.vit_embed_stage(sd, VC, pix, grid, f64)
    for i in range(VC.depth):
        x = QS.vit_block_stage(sd, VC, i, x, grid, f64)["h"]
    emb = QS.vit_merge_stage(sd, VC, x, grid, f64)["out"]
    assert torch.equal(emb, qo.vision_forward(sd, VC, pix, grid))
    pos = _pos(ids, grid)
    h = qo.embed_prompt(sd, ids, emb, IMG)
    for i in range(TC.num_hidden_layers):
        h = QS.decoder_stage(sd, TC, i, h, pos, f64)["h"]
    assert torch.equal(QS.norm_stage(sd, TC, h, f64), qo.prefill(sd, TC, VC, ids, pos, pix, grid))


def _fails_slice(checks):
    return [c for c in checks if not c.ok and c.kind != "tensor"]


def _tensor_misses(checks):
    return all(c.ok for c in checks if c.kind == "tensor")


def test_yardstick_passes_its_own_gates():
    grid = GRIDS["1000x1500"]
    sd = qo.make_synthetic_state_dict(TC, VC, seed=3, dtype=f64)
    x = QS.vit_embed_stage(sd, VC, _pixels(grid, 2), grid, f64).to(bf16)
    cu = QS.vit_context(VC, grid)[1]
    R, Y = QS.vit_block_stage(sd, VC, 0, x, grid, f64), QS.vit_block_stage(sd, VC, 0, x, grid, bf16)
    for K in (Y, {k: v.to(bf16) for k, v in R.items()}):
        checks = QS.vit_gates("vit 0", "h", K["h"], R["h"], Y["h"], cu, base=x)
        checks += QS.vit_gates("vit 0", "attn", K["attn"], R["attn"], Y["attn"], cu, heads=(VC.num_heads, 80))
        assert all(c.ok for c in checks), "\n".join(map(str, checks))
    ids = _prompt(grid)
    xd = qo.embed_prompt(sd, ids, torch.randn(247, 256, dtype=f64), IMG).to(bf16)
    pos = _pos(ids, grid)
    R, Y = QS.decoder_stage(sd, TC, 0, xd, pos, f64), QS.decoder_stage(sd, TC, 0, xd, pos, bf16)
    parts = {"text": ids != IMG, "image": ids == IMG}
    for K in (Y, {k: v.to(bf16) for k, v in R.items()}):
        checks = QS.dec_gates("dec 0", "h", K["h"], R["h"], Y["h"], parts, base=xd)
        checks += QS.dec_gates("dec 0", "qkv", K["qkv"], R["qkv"], Y["qkv"], parts, heads=(QS.qkv_head_labels(2, 1), 128))
        assert all(c.ok for c in checks), "\n".join(map(str, checks))


# ------------------------------------------------------------------------------------------------ planted faults
def _report(name, checks):
    bad = _fails_slice(checks)
    print(f"\n[{name}] per-tensor rule {'misses it' if _tensor_misses(checks) else 'catches it'}; per-slice failures:")
    print("\n".join(map(str, bad)))
    assert bad, f"{name}: the per-slice gate passed the planted fault"


def test_fault_window_attends_into_its_neighbour():
    """one ViT window's cu_seqlens boundary dropped: windows 2 and 3 of a (1, 26, 38) grid attend as one"""
    grid = GRIDS["1000x1500"]
    sd = qo.make_synthetic_state_dict(TC, VC, seed=4, dtype=f64)
    x = QS.vit_embed_stage(sd, VC, _pixels(grid, 3), grid, f64).to(bf16)
    cu = QS.vit_context(VC, grid)[1]
    R, Y = QS.vit_block_stage(sd, VC, 0, x, grid, f64), QS.vit_block_stage(sd, VC, 0, x, grid, bf16)
    _, cos, sin = None, *qo.vision_rope(grid, 80)
    perm = QS.vit_context(VC, grid)[3]
    bad_cu = cu[:3] + cu[4:]
    K = qo.vision_block(sd, 0, x.double(), cos[perm], sin[perm], bad_cu, VC)
    _report("window boundary", QS.vit_gates("vit 0", "attn", K["attn"].to(bf16), R["attn"], Y["attn"], cu,
                                            heads=(VC.num_heads, 80)))


def test_fault_unwindowing_gather_wrong_for_one_window():
    """the merger output un-permuted with one window's tokens in reverse order"""
    grid = GRIDS["1456x720"]
    sd = qo.make_synthetic_state_dict(TC, VC, seed=5, dtype=f64)
    x = torch.randn(sum(t * h * w for t, h, w in grid), VC.hidden_size, dtype=f64).to(bf16)
    R, Y = QS.vit_merge_stage(sd, VC, x, grid, f64), QS.vit_merge_stage(sd, VC, x, grid, bf16)
    widx = QS.vit_context(VC, grid)[0].clone()
    widx[16:32] = widx[16:32].flip(0)                                  # the second window (16 merged tokens)
    K = R["merged"][torch.argsort(widx)].to(bf16)
    _report("un-windowing gather", QS.TB.gate("merge", "out", K, R["out"], Y["out"], ("rows", "cols"), beta=QS.IB.BETA))


def test_fault_query_head_reads_the_wrong_kv_head(monkeypatch):
    """GQA 28 : 4 at the decoder's width, query head h reading KV head h % 4 instead of h // 7"""
    tc = QwenTextConfig(hidden_size=3584, num_hidden_layers=1, intermediate_size=256, vocab_size=1000)
    sd = qo.make_synthetic_state_dict(tc, VC, seed=6, dtype=f64)
    x = torch.randn(1, 40, 3584, dtype=f64).to(bf16)
    pos = torch.arange(40).view(1, 1, -1).expand(3, 1, -1)
    R, Y = QS.decoder_stage(sd, tc, 0, x, pos, f64), QS.decoder_stage(sd, tc, 0, x, pos, bf16)
    good = qo.attention

    def wrong(q, k, v, mask=None, scale=None):
        idx = torch.arange(q.shape[1]) % k.shape[1]
        return good(q, k[:, idx], v[:, idx], mask, scale)

    monkeypatch.setattr(qo, "attention", wrong)
    K = QS.decoder_stage(sd, tc, 0, x, pos, f64)
    parts = {"text": torch.ones(1, 40, dtype=torch.bool)}
    _report("GQA head map", QS.dec_gates("dec 0", "attn", K["attn"].to(bf16), R["attn"], Y["attn"], parts,
                                         heads=([f"head {h}" for h in range(28)], 128)))


def test_fault_mrope_h_w_swapped_on_image_rows():
    grid = GRIDS["1000x1500"]
    sd = qo.make_synthetic_state_dict(TC, VC, seed=7, dtype=f64)
    ids = _prompt(grid)
    x = qo.embed_prompt(sd, ids, torch.randn(247, 256, dtype=f64), IMG).to(bf16)
    pos = _pos(ids, grid)
    R, Y = QS.decoder_stage(sd, TC, 0, x, pos, f64), QS.decoder_stage(sd, TC, 0, x, pos, bf16)
    img = ids == IMG
    bad = pos.clone()
    bad[1][img], bad[2][img] = pos[2][img], pos[1][img]
    K = QS.decoder_stage(sd, TC, 0, x, bad, f64)
    parts = {"text": ~img, "image": img}
    _report("M-RoPE h / w", QS.dec_gates("dec 0", "qkv", K["qkv"].to(bf16), R["qkv"], Y["qkv"], parts,
                                         heads=(QS.qkv_head_labels(2, 1), 128)))


def test_fault_decode_drops_the_oldest_cache_row():
    """a decode step over a left-padded pair whose second sequence starts one row late in the cache"""
    sd = qo.make_synthetic_state_dict(TC, VC, seed=8, dtype=f64)
    P, lo = 24, [0, 9]
    kv = [torch.randn(2, P, 1, 128, dtype=f64).to(bf16) for _ in range(2)]
    x = torch.randn(2, 1, 256, dtype=f64).to(bf16)
    pos = torch.tensor([P + 3, P - 6]).view(1, 2, 1).expand(3, 2, 1)
    R = QS.decoder_stage(sd, TC, 0, x, pos, f64, past_kv=kv, past_lo=lo)
    Y = QS.decoder_stage(sd, TC, 0, x, pos, bf16, past_kv=kv, past_lo=lo)
    K = QS.decoder_stage(sd, TC, 0, x, pos, f64, past_kv=kv, past_lo=[0, 10])
    lab = lambda kind, i: f"sequence {i}" if kind == "rows" else f"{kind[:-1]} {i}"
    _report("decode cache row", QS.TB.gate("decode", "attn", K["attn"][:, 0].to(bf16), R["attn"][:, 0], Y["attn"][:, 0],
                                           ("rows", "cols"), lab, beta=QS.IB.BETA))
