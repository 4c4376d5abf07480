"""The T5 / CLIP stage references (tests/text_encoder_stage_ref.py) on the CPU: the float64 oracle is transformers'
T5EncoderModel and CLIPTextModel in float64 at the encoders' real lengths and EOS layouts, the float64 stages chain to
the oracle bit for bit, the bf16 yardstick passes its own gates, and the per-slice gates catch five planted faults of the
kinds the engine's kernels or host code could make.
"""
import pytest
import torch

import text_encoder_stage_ref as SR
from gpt_image_edit_b200.text_encoders import CLIPTextConfig, T5EncoderConfig
from oracle import text_encoder_oracle as to

t5_hf = pytest.importorskip("transformers.models.t5.modeling_t5")
clip_hf = pytest.importorskip("transformers.models.clip.modeling_clip")

f64, bf16 = torch.float64, torch.bfloat16
T5C = T5EncoderConfig(vocab_size=300, d_model=256, d_kv=64, num_heads=4, d_ff=512, num_layers=2)
CLIPC = CLIPTextConfig(vocab_size=400, hidden_size=256, intermediate_size=1024, num_hidden_layers=2, num_attention_heads=4)
EOS = CLIPC.vocab_size - 1            # FLUX's CLIP tokenizer pads with <|endoftext|>, the largest id


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def _t5_ids(B, L, seed):
    return torch.randint(2, T5C.vocab_size, (B, L), generator=torch.Generator().manual_seed(seed))


def _clip_ids(eos_at, pad_zero=(), seed=0):
    """[B, 77]: BOS, body tokens, EOS at eos_at[b], then EOS padding (or 0 for the rows in pad_zero)"""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(1, EOS - 1, (len(eos_at), 77), generator=g)
    ids[:, 0] = EOS - 1
    for b, e in enumerate(eos_at):
        ids[b, e] = EOS
        ids[b, e + 1:] = 0 if b in pad_zero else EOS
    return ids


def _t5_fp64(monkeypatch, sd):
    """transformers' T5EncoderModel in float64 with the oracle's weights.  T5LayerNorm's variance and the attention's
    softmax over `scores.float()` run in float32 whatever the model's dtype; those casts are lifted to float64 here."""
    from transformers import T5Config

    def norm(self, x):
        return self.weight * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + self.variance_epsilon))

    monkeypatch.setattr(t5_hf.T5LayerNorm, "forward", norm)
    to_float = torch.Tensor.float
    monkeypatch.setattr(torch.Tensor, "float", lambda t: t if t.dtype == f64 else to_float(t))
    cfg = T5Config(vocab_size=T5C.vocab_size, d_model=T5C.d_model, d_kv=T5C.d_kv, num_heads=T5C.num_heads, d_ff=T5C.d_ff,
                   num_layers=T5C.num_layers, feed_forward_proj="gated-gelu", dropout_rate=0.0, is_encoder_decoder=False,
                   use_cache=False, relative_attention_num_buckets=32, relative_attention_max_distance=128)
    ref = t5_hf.T5EncoderModel(cfg).eval().double()
    missing, unexpected = ref.load_state_dict(sd, strict=False)
    assert not unexpected and set(missing) <= {"encoder.embed_tokens.weight"}, (missing, unexpected)
    return ref


def _clip_fp64(monkeypatch, sd, eos_token_id):
    """transformers' CLIPTextModel in float64 with the oracle's weights.  Its eager attention takes the softmax in
    float32; that cast is lifted to float64 here."""
    from transformers import CLIPTextConfig as HFCfg

    def eager(module, query, key, value, attention_mask, scaling, dropout=0.0, **kw):
        w = torch.matmul(query, key.transpose(-1, -2)) * scaling
        if attention_mask is not None:
            w = w + attention_mask
        w = torch.softmax(w, dim=-1)
        return torch.matmul(w, value).transpose(1, 2).contiguous(), w

    monkeypatch.setattr(clip_hf, "eager_attention_forward", eager)
    cfg = HFCfg(vocab_size=CLIPC.vocab_size, hidden_size=CLIPC.hidden_size, intermediate_size=CLIPC.intermediate_size,
                num_hidden_layers=CLIPC.num_hidden_layers, num_attention_heads=CLIPC.num_attention_heads,
                max_position_embeddings=77, hidden_act="quick_gelu", eos_token_id=eos_token_id, bos_token_id=EOS - 1,
                pad_token_id=EOS, attn_implementation="eager")
    ref = clip_hf.CLIPTextModel(cfg).eval().double()
    missing, unexpected = ref.load_state_dict(sd, strict=False)
    assert not unexpected and all("position_ids" in k for k in missing), (missing, unexpected)
    return ref


# ------------------------------------------------------------------------------------------------ oracle = transformers
def test_buckets_are_transformers():
    """the oracle's integer bucket rule equals transformers' float32-log rule (on the host) at every distance up to 511,
    the exact bucket edges 16, 32, 64 and 128 included"""
    L = 512
    rel = torch.arange(L)[None, :] - torch.arange(L)[:, None]
    want = t5_hf.T5Attention._relative_position_bucket(rel, bidirectional=True, num_buckets=32, max_distance=128)
    assert torch.equal(to.bucket_grid(L), want)
    assert [to.relative_position_bucket(n) for n in (15, 16, 32, 64, 127, 128, -16, -64)] == [25, 26, 28, 30, 31, 31, 10, 14]


@pytest.mark.parametrize("B,L", [(2, 40), (1, 77), (1, 300)])
def test_t5_oracle_is_transformers_in_fp64(monkeypatch, B, L):
    sd = to.make_t5_state_dict(T5C, seed=1, dtype=f64)
    ref = _t5_fp64(monkeypatch, sd)
    ids = _t5_ids(B, L, seed=L)
    with torch.no_grad():
        want = ref(input_ids=ids).last_hidden_state
    got = to.t5_forward(sd, T5C, ids)
    print(f"\nT5 B {B} L {L}: rel {_rel(got, want):.2e}")
    assert got.shape == want.shape and _rel(got, want) < 1e-13


@pytest.mark.parametrize("eos_token_id", [2, EOS], ids=["argmax_rule", "first_eos_rule"])
def test_clip_oracle_is_transformers_in_fp64(monkeypatch, eos_token_id):
    """a batch whose rows end at different positions, padded with EOS (ties for the argmax) or with 0"""
    cfg = CLIPTextConfig(**{**vars(CLIPC), "eos_token_id": eos_token_id})
    sd = to.make_clip_state_dict(cfg, seed=2, dtype=f64)
    ref = _clip_fp64(monkeypatch, sd, eos_token_id)
    ids = _clip_ids([1, 40, 76, 20], pad_zero=(3,))
    with torch.no_grad():
        want = ref(input_ids=ids)
    last, pooled = to.clip_forward(sd, cfg, ids)
    print(f"\nCLIP {eos_token_id}: last rel {_rel(last, want.last_hidden_state):.2e}, "
          f"pooled rel {_rel(pooled, want.pooler_output):.2e}")
    assert _rel(last, want.last_hidden_state) < 1e-13 and _rel(pooled, want.pooler_output) < 1e-13
    assert to.eos_positions(ids, eos_token_id).tolist() == [1, 40, 76, 20]


def test_stage_chain_is_the_oracle():
    sd = to.make_t5_state_dict(T5C, seed=3, dtype=f64)
    ids = _t5_ids(2, 77, seed=4)
    x = SR.t5_embed_stage(sd, ids, f64)
    for i in range(T5C.num_layers):
        x = SR.t5_layer_stage(sd, T5C, i, x, f64)["x"]
    assert torch.equal(SR.t5_final_stage(sd, T5C, x, f64), to.t5_forward(sd, T5C, ids))
    sd = to.make_clip_state_dict(CLIPC, seed=4, dtype=f64)
    ids = _clip_ids([5, 60])
    x = SR.clip_embed_stage(sd, ids, f64)
    for i in range(CLIPC.num_hidden_layers):
        x = SR.clip_layer_stage(sd, CLIPC, i, x, f64)["x"]
    out = SR.clip_final_stage(sd, CLIPC, x, ids, f64)
    last, pooled = to.clip_forward(sd, CLIPC, ids)
    assert torch.equal(out["last"], last) and torch.equal(out["pooled"], pooled)


def test_layout_helpers():
    H = 3
    t = torch.arange(2 * 5 * 3 * H * 128, dtype=f64).view(2, 5, 3 * H * 128)
    real = SR.strip_heads(t)
    assert real.shape == (2, 5, 3 * H * 64)
    assert torch.equal(real[..., 64:128], t[..., 128:192])
    pad = SR.padding({"qkv": t, "attn_out": t[..., :H * 128]})
    assert torch.equal(pad["qkv[..., 64:128]"][..., 1, :], t[..., 192:256])


def _t5_layer_case(seed, L=300, d=4096, H=64, d_ff=512):
    """one T5 block at T5-XXL's head count (64 heads of 64) and a narrow feed-forward"""
    cfg = T5EncoderConfig(vocab_size=300, d_model=d, d_kv=64, num_heads=H, d_ff=d_ff, num_layers=1)
    sd = to.make_t5_state_dict(cfg, seed=seed, dtype=f64)
    noise = torch.randn(1, L, d, dtype=f64, generator=torch.Generator().manual_seed(seed))
    x = (SR.t5_embed_stage(sd, _t5_ids(1, L, seed), f64) + noise).to(bf16)
    return cfg, sd, x


def test_yardstick_passes_its_own_gates():
    cfg, sd, x = _t5_layer_case(5, L=200, d=256, H=4)
    R, Y = SR.t5_layer_stage(sd, cfg, 0, x, f64), SR.t5_layer_stage(sd, cfg, 0, x, bf16)
    for K in (Y, {k: v.to(bf16) for k, v in R.items()}):
        checks = SR.layer_gates("t5 0", K, R, Y, x)
        assert all(c.ok for c in checks), "\n".join(map(str, checks))
    sd = to.make_clip_state_dict(CLIPC, seed=6, dtype=f64)
    x = SR.clip_embed_stage(sd, _clip_ids([9, 33]), f64).to(bf16)
    R, Y = SR.clip_layer_stage(sd, CLIPC, 0, x, f64), SR.clip_layer_stage(sd, CLIPC, 0, x, bf16)
    for K in (Y, {k: v.to(bf16) for k, v in R.items()}):
        checks = SR.layer_gates("clip 0", K, R, Y, x)
        assert all(c.ok for c in checks), "\n".join(map(str, checks))


# ------------------------------------------------------------------------------------------------ planted faults
def _report(name, checks):
    bad = [c for c in checks if not c.ok and c.kind != "tensor"]
    misses = all(c.ok for c in checks if c.kind == "tensor")
    print(f"\n[{name}] per-tensor rule {'misses it' if misses else 'catches it'}; per-slice failures:")
    print("\n".join(map(str, bad)))
    assert bad, f"{name}: the per-slice gate passed the planted fault"


def _t5_fault(name, seed, edit, keys=("attn_out",)):
    """a T5 block whose position bias is edited by `edit(bias)`, gated against the right one"""
    cfg, sd, x = _t5_layer_case(seed)
    R, Y = SR.t5_layer_stage(sd, cfg, 0, x, f64), SR.t5_layer_stage(sd, cfg, 0, x, bf16)
    K = SR.t5_layer_stage(sd, cfg, 0, x, f64, bias=edit(to.position_bias(sd, cfg, x.shape[1]).clone()))
    checks = []
    for k in keys:
        checks += SR.enc_gates("t5 0", k, K[k].to(bf16), R[k], Y[k], heads=64 if k == "attn_out" else None)
    _report(name, checks)


def test_fault_one_query_row_reads_the_wrong_bias_row():
    """query row 128 (the first row of the second query tile) adds the bias row of query 127"""
    def edit(b):
        b[:, 128] = b[:, 127]
        return b
    _t5_fault("bias row at a tile edge", 7, edit, keys=("attn_out", "x"))


def test_fault_one_head_reads_the_next_heads_bias():
    def edit(b):
        b[5] = b[6]
        return b
    _t5_fault("one head's bias", 8, edit, keys=("attn_out", "x"))


def test_fault_transposed_position_bias():
    """bias[h, key, query] for bias[h, query, key]: the table is asymmetric (+16 buckets for keys after the query)"""
    _t5_fault("transposed bias", 9, lambda b: b.transpose(-1, -2))


def test_fault_clip_query_sees_the_next_key(monkeypatch):
    sd = to.make_clip_state_dict(CLIPC, seed=10, dtype=f64)
    x = SR.clip_embed_stage(sd, _clip_ids([30, 76, 12]), f64).to(bf16)
    R, Y = SR.clip_layer_stage(sd, CLIPC, 0, x, f64), SR.clip_layer_stage(sd, CLIPC, 0, x, bf16)
    monkeypatch.setattr(to, "causal_mask", lambda L, device=None: torch.ones(L, L, dtype=torch.bool, device=device).tril(1))
    K = SR.clip_layer_stage(sd, CLIPC, 0, x, f64)
    _report("causal mask off by one", SR.enc_gates("clip 0", "attn_out", K["attn_out"].to(bf16), R["attn_out"],
                                                   Y["attn_out"], heads=64))


def test_fault_pooled_one_token_late():
    sd = to.make_clip_state_dict(CLIPC, seed=11, dtype=f64)
    ids = _clip_ids([3, 40, 76, 20], pad_zero=(3,))
    x = torch.randn(4, 77, CLIPC.hidden_size, dtype=f64, generator=torch.Generator().manual_seed(12)).to(bf16)
    R, Y = SR.clip_final_stage(sd, CLIPC, x, ids, f64), SR.clip_final_stage(sd, CLIPC, x, ids, bf16)
    pos = (to.eos_positions(ids, 2) + 1).clamp_max(76)
    K = R["last"][torch.arange(4), pos].to(bf16)
    _report("pooled one token late", SR.pooled_gates("final", K, R["pooled"], Y["pooled"]))
