"""The T5-XXL and CLIP-L prompt encoders (gpt_image_edit_b200/text_encoders.py) checked stage by stage at full width
against float64 references of the oracle per token, per channel and per head (tests/text_encoder_stage_ref.py), at the
lengths the edit path runs them: T5 at 512 (the pipeline's default), 256 (bench and the CLI, an empty prompt included),
77 and 300; CLIP at 77 with EOS early, in the middle and last, padded with EOS or with 0.

Every stage runs through the engine's own methods (`_t5_embed`, `_t5_layer`, `_t5_final`; `_clip_embed`, `_clip_layer`,
`_clip_final`); its reference is fed the engine's input to that stage, with the same oracle stage in bf16 as the
yardstick: the per-tensor rule rel-L2(engine) <= 2 rel-L2(bf16) + 1e-2 and the per-slice gate max_s e_s <= 2 max_s y_s +
1e-3.  Exact checks: the stagewise run is forward() bit for bit, the padding columns 64..127 of every head slot stay zero,
the embeddings are the bf16 gathers (and sum), the pooled row is the last hidden state at the first EOS, and the T5
position bias is the layer-0 table gathered by transformers' own bucket function run on the device.
"""
import pytest
import torch

import text_encoder_stage_ref as SR
from oracle import text_encoder_oracle as to

pytestmark = pytest.mark.gpu

f64, bf16 = torch.float64, torch.bfloat16
XXL = dict(vocab_size=32128, d_model=4096, d_kv=64, num_heads=64, d_ff=10240)
TOY_T5 = dict(vocab_size=128, d_model=256, d_kv=64, num_heads=4, d_ff=512)
CLIP_L = dict(vocab_size=49408, hidden_size=768, intermediate_size=3072, num_attention_heads=12)
TOY_CLIP = dict(vocab_size=49408, hidden_size=256, intermediate_size=1024, num_attention_heads=4)
BOS, EOS = 49406, 49407          # CLIP's <|startoftext|> and <|endoftext|> (also its padding)


def _report(title, checks):
    print(f"\n[{title}]")
    print("\n".join(str(c) for c in checks))
    return [str(c) for c in checks if not c.ok]


def _summary(title, checks):
    """worst e / y and the smallest margin 2y + beta - e per tensor family"""
    fam = {}
    for c in checks:
        if c.kind == "tensor":
            continue
        k = f"{c.tensor} {c.kind}"
        r = c.e / c.y if c.y > 0 else 0.0
        m = 2 * c.y + SR.IB.BETA - c.e
        a, b = fam.get(k, (0.0, float("inf")))
        fam[k] = (max(a, r), min(b, m))
    print(f"\n[{title} summary] " + "; ".join(f"{k}: e/y {a:.2f} margin {b:.2e}" for k, (a, b) in sorted(fam.items())))


# ------------------------------------------------------------------------------------------------ T5
def _t5(kw, layers, seed, peaked=False):
    from gpt_image_edit_b200.text_encoders import B200T5Encoder, T5EncoderConfig

    cfg = T5EncoderConfig(**kw, num_layers=layers)
    sd = to.make_t5_state_dict(cfg, seed=seed, dtype=bf16, device="cuda")
    if peaked:
        # logits of std ~30 (q and k each 1.93x) and a bias table of std 4: the online softmax rescales often
        for n in "qk":
            w = sd[f"encoder.block.0.layer.0.SelfAttention.{n}.weight"]
            w.copy_(w.float() * 1.93)
        rb = sd["encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"]
        rb.copy_(rb.float() * 4)
    m = B200T5Encoder(cfg)
    m.load_state_dict(sd)
    return cfg, sd, m


def _t5_ids(B, L, vocab, seed):
    return torch.randint(2, vocab, (B, L), generator=torch.Generator().manual_seed(seed))


def _outliers(rows, d, seed):
    """a residual stream [rows, d] of N(0, 1) with four channels at +-1e4 (a bf16 ulp there is 64)"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    y = torch.randn(rows, d, device="cuda", generator=g)
    for c, s in ((11, 1e4), (907, -1e4), (2050, 1e4), (3999, -1e4)):
        y[:, c] = s * (1 + 0.01 * torch.randn(rows, device="cuda", generator=g))
    return y.bfloat16()


def _t5_run(cfg, sd, m, ids, x0=None):
    """the engine's stages on ids [B, L], each gated against the oracle's stage fed the engine's input; x0 replaces the
    embedding as block 0's input"""
    B, L = ids.shape
    H = cfg.num_heads
    idc = ids.cuda()
    x = m._t5_embed(idc)
    assert torch.equal(x.view(B, L, -1), SR.t5_embed_stage(sd, idc, bf16)), "embedding gather"
    if x0 is not None:
        x = x0
    bias = m.position_bias(L)
    attn = torch.empty((B, L, H * SR.HP), device="cuda", dtype=bf16)
    checks = []
    v3 = lambda t: t.view(B, L, -1)
    for i in range(cfg.num_layers):
        x_in = x
        keep = {}
        x = m._t5_layer(i, x_in, bias, attn, B, L, keep)
        for name, t in SR.padding(keep).items():
            assert not bool(t.any()), f"block {i}: {name} is not zero"
        K = {n: v3(keep[n]) for n in ("xn1", "x_mid", "xn2", "gu", "h")}
        K.update(qkv=SR.strip_heads(v3(keep["qkv"])), attn_out=SR.strip_heads(v3(keep["attn_out"])), x=v3(x))
        R = SR.t5_layer_stage(sd, cfg, i, v3(x_in), f64)
        Y = SR.t5_layer_stage(sd, cfg, i, v3(x_in), bf16)
        checks += SR.layer_gates(f"B{B} L{L} t5 {i}", K, R, Y, v3(x_in))
        del R, Y
    out = m._t5_final(x)
    checks += SR.enc_gates(f"B{B} L{L} final", "out", v3(out), SR.t5_final_stage(sd, cfg, v3(x), f64),
                           SR.t5_final_stage(sd, cfg, v3(x), bf16))
    if x0 is None:
        assert torch.equal(m(idc).last_hidden_state, v3(out)), "the stagewise run is not forward()"
    return checks


# name: (width, layers, [(B, L)] or explicit ids, peaked, outliers)
T5_CASES = {
    "t5_512": (XXL, 2, [(1, 512)], False, False),                 # the pipeline's default; bias [64, 512, 512]
    "t5_256_pair": (XXL, 2, [(2, 256)], False, False),            # bench's and the CLI's length; one bias for the batch
    "t5_empty_prompt": (XXL, 2, [torch.tensor([[1] + [0] * 255])], False, False),   # "</s>" then <pad> x 255
    "t5_ragged": (XXL, 2, [(2, 77), (1, 300)], False, False),     # odd bias row stride, partial query and key tiles
    "t5_full_depth": (XXL, 24, [(1, 256)], False, False),         # bench's shape; the layer-0 table in every layer
    "t5_peaked": (XXL, 1, [(1, 512)], True, False),
    "t5_outliers": (XXL, 1, [(1, 256)], False, True),
    "toy_t5": (TOY_T5, 2, [(3, 1), (2, 77)], False, False),       # compute-sanitizer's shapes
}


def _t5_case(case):
    kw, layers, shapes, peaked, outliers = T5_CASES[case]
    cfg, sd, m = _t5(kw, layers, seed=1, peaked=peaked)
    checks = []
    for j, s in enumerate(shapes):
        ids = s if torch.is_tensor(s) else _t5_ids(*s, cfg.vocab_size, seed=10 + j)
        x0 = _outliers(ids.numel(), cfg.d_model, 3) if outliers else None
        if peaked:
            R = SR.t5_layer_stage(sd, cfg, 0, SR.t5_embed_stage(sd, ids.cuda(), bf16), f64)
            q, k = (t.view(*ids.shape, cfg.num_heads, 64).transpose(1, 2) for t in R["qkv"].split(cfg.num_heads * 64, -1)[:2])
            print(f"\nt5_peaked: logit std {(q @ k.transpose(-1, -2)).std().item():.1f}")
            del R, q, k
        checks += _t5_run(cfg, sd, m, ids, x0)
    return checks


# ------------------------------------------------------------------------------------------------ CLIP
def _clip(kw, layers, seed):
    from gpt_image_edit_b200.text_encoders import B200CLIPTextModel, CLIPTextConfig

    cfg = CLIPTextConfig(**kw, num_hidden_layers=layers)
    sd = to.make_clip_state_dict(cfg, seed=seed, dtype=bf16, device="cuda")
    m = B200CLIPTextModel(cfg)
    m.load_state_dict(sd)
    return cfg, sd, m


def _clip_ids(eos_at, pad_zero=(), seed=0):
    """[B, 77]: BOS, body tokens, EOS at eos_at[b], then EOS as padding (FLUX's CLIP tokenizer), or 0 for pad_zero rows"""
    ids = torch.randint(1, BOS, (len(eos_at), 77), generator=torch.Generator().manual_seed(seed))
    ids[:, 0] = BOS
    for b, e in enumerate(eos_at):
        ids[b, e] = EOS
        ids[b, e + 1:] = 0 if b in pad_zero else EOS
    return ids


CLIP_CASES = {
    "clip_l": (CLIP_L, 12, ([1, 40, 76, 20], (3,))),
    "toy_clip": (TOY_CLIP, 2, ([9, 76], ())),
}


def _clip_case(case):
    kw, layers, (eos_at, pad_zero) = CLIP_CASES[case]
    cfg, sd, m = _clip(kw, layers, seed=2)
    ids = _clip_ids(eos_at, pad_zero, seed=4)
    B, L = ids.shape
    H = cfg.num_attention_heads
    idc = ids.cuda()
    v3 = lambda t: t.view(B, L, -1)
    x = m._clip_embed(idc)
    assert torch.equal(v3(x), SR.clip_embed_stage(sd, idc, bf16)), "token + position embedding"
    attn = torch.empty((B, L, H * SR.HP), device="cuda", dtype=bf16)
    checks = []
    for i in range(layers):
        x_in = x
        keep = {}
        x = m._clip_layer(i, x_in, attn, B, L, keep)
        for name, t in SR.padding(keep).items():
            assert not bool(t.any()), f"layer {i}: {name} is not zero"
        K = {n: v3(keep[n]) for n in ("xn1", "x_mid", "xn2", "fc1")}
        K.update(qkv=SR.strip_heads(v3(keep["qkv"])), attn_out=SR.strip_heads(v3(keep["attn_out"])), x=v3(x))
        R = SR.clip_layer_stage(sd, cfg, i, v3(x_in), f64)
        Y = SR.clip_layer_stage(sd, cfg, i, v3(x_in), bf16)
        checks += SR.layer_gates(f"clip {i}", K, R, Y, v3(x_in))
    last, pooled = m._clip_final(x, idc)
    R, Y = SR.clip_final_stage(sd, cfg, v3(x), ids, f64), SR.clip_final_stage(sd, cfg, v3(x), ids, bf16)
    checks += SR.enc_gates("final", "last", v3(last), R["last"], Y["last"])
    checks += SR.pooled_gates("final", pooled, R["pooled"], Y["pooled"])
    # the pooled row is the hidden state at argmax(ids), and that is the first EOS even where the padding is EOS too
    first_eos = torch.tensor([r.index(EOS) for r in ids.tolist()])
    assert ids.argmax(-1).tolist() == first_eos.tolist() == eos_at
    assert torch.equal(pooled, v3(last)[torch.arange(B), first_eos.cuda()])
    out = m(idc)
    assert torch.equal(out.last_hidden_state, v3(last)) and torch.equal(out.pooler_output, pooled)
    return checks


@pytest.mark.parametrize("case", list(T5_CASES) + list(CLIP_CASES))
def test_stagewise_encoder_matches_fp64(case):
    checks = _t5_case(case) if case in T5_CASES else _clip_case(case)
    _summary(case, checks)
    bad = _report(case, checks)
    assert not bad, "\n".join(bad)


# ------------------------------------------------------------------------------------------------ exact checks
@pytest.mark.parametrize("L", [1, 77, 256, 300, 512])
def test_position_bias_is_transformers_buckets_on_device(L):
    """`position_bias(L)` is rel_bias at transformers' own `_relative_position_bucket` of (key - query), computed on the
    CUDA device as T5Attention.compute_bias does.  The float32 log at the exact bucket edges (distances 16, 32, 64 and
    128) is where a device's rounding could move a distance into the next bucket."""
    t5_hf = pytest.importorskip("transformers.models.t5.modeling_t5")
    from gpt_image_edit_b200.text_encoders import B200T5Encoder, T5EncoderConfig

    m = B200T5Encoder(T5EncoderConfig(**TOY_T5, num_layers=1)).randomize_(seed=5)
    pos = torch.arange(L, dtype=torch.long, device="cuda")
    idx = t5_hf.T5Attention._relative_position_bucket(pos[None, :] - pos[:, None], bidirectional=True, num_buckets=32,
                                                      max_distance=128)
    moved = (idx.cpu() != to.bucket_grid(L)).nonzero()
    print(f"\nL {L}: {len(moved)} (query, key) pairs whose device bucket differs from the exact one: {moved[:8].tolist()}")
    assert torch.equal(m.position_bias(L), m.W["rel_bias"][idx].permute(2, 0, 1))


def test_encoder_gemm_tiles():
    """Records the GEMM tile (t128 / t256) of every T5-XXL and CLIP-L linear at the encoders' real shapes.  T5's qkv
    (M 512) and wi (M 300) projections run on the wide tile, so its plain epilogue reaches both tiles; its residual
    epilogues (o, wo) and every CLIP linear (bias, quick-GELU and residual epilogues at M <= 308) stay on the 128 tile at
    these shapes.  Those epilogues are checked on the wide tile by test_gemm_wide_gpu.py's forced-tile tests."""
    from test_gemm_wide_gpu import _tags

    _, _, t5 = _t5(XXL, 1, seed=6)
    seen = set()
    for B, L in ((1, 512), (2, 256), (1, 256), (2, 77), (1, 300)):
        tags = _tags(lambda: t5(_t5_ids(B, L, XXL["vocab_size"], 1).cuda()))
        print(f"\nT5 B {B} L {L}: " + ", ".join(tags))
        assert tags
        seen |= {t.rsplit(" ", 1)[-1] for t in tags}
    assert {"t128", "t256"} <= seen, seen
    _, _, clip = _clip(CLIP_L, 1, seed=7)
    for B in (1, 2, 4):
        tags = _tags(lambda: clip(_clip_ids([20] * B).cuda()))
        print(f"\nCLIP B {B} L 77: " + ", ".join(tags))
        assert tags and all(t.endswith((" t128", " t256")) for t in tags), tags
