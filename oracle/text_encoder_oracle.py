"""ORACLE — TEST INFRASTRUCTURE ONLY (see oracle/flux_oracle.py for the rules).

PyTorch restatement of the two prompt encoders the reference reaches through transformers (`T5EncoderModel`,
`CLIPTextModel`), written from the models' math:

  T5 v1.1 encoder   token embedding; pre-RMSNorm blocks of unscaled multi-head attention plus a bucketed relative-position
                    bias (one table, owned by block 0, shared by every block) and no mask, then a gated-GELU (tanh)
                    feed-forward wo(gelu(wi_0 x) * wi_1 x); final RMSNorm
  CLIP text         token + learned position embedding; pre-LayerNorm layers of causal attention at d_h^-0.5 with biases,
                    then fc2(quick_gelu(fc1 x)); final LayerNorm; the pooled row at argmax(ids) (eos_token_id == 2) or
                    at the first eos_token_id

It takes weights under the transformers names at their true shapes (head_dim 64, no head slots), so it knows nothing of
the engine's kernel layout.

Every function runs in the dtype of its inputs: float64 gives the exact-math answer, bfloat16 what transformers does in
bf16.  Where transformers computes in float32 inside a bf16 model (T5LayerNorm's variance, T5's softmax over
`scores.float()`, CLIP's eager softmax) a bf16 run does the same, so the bf16 run is the yardstick the engine is held to.
Pinned against transformers in float64 by tests/test_text_encoder_stage_ref_cpu.py.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F


def _up(dtype):
    """the compute dtype of a step transformers runs in float32 (float64 stays float64)."""
    return torch.promote_types(dtype, torch.float32)


def _lin(sd, name, x):
    return F.linear(x, sd[name + ".weight"], sd.get(name + ".bias"))


def _heads(t, H):
    """[B, L, H * dh] -> [B, H, L, dh]"""
    B, L, _ = t.shape
    return t.view(B, L, H, -1).transpose(1, 2)


def _flat(t):
    """[B, H, L, dh] -> [B, L, H * dh]"""
    B, H, L, dh = t.shape
    return t.transpose(1, 2).reshape(B, L, H * dh)


# ------------------------------------------------------------------------------------------------ T5
def relative_position_bucket(n: int, num_buckets: int = 32, max_distance: int = 128) -> int:
    """Bidirectional T5 bucket of the signed distance n = key - query.  Half the buckets are for n > 0.  Within a half,
    distances below e = half / 2 get a bucket each; a larger distance m gets e + floor((half - e) log(m / e) /
    log(max_distance / e)), at most half - 1.  The floor is taken exactly, in integers: with s = half - e, bucket e + j
    is reached when (m / e)^s >= (max_distance / e)^j, i.e. m^s e^j >= e^s max_distance^j."""
    half = num_buckets // 2
    e = half // 2
    m = abs(n)
    base = half if n > 0 else 0
    if m < e:
        return base + m
    s = half - e
    j = 0
    while j + 1 < s and m ** s * e ** (j + 1) >= e ** s * max_distance ** (j + 1):
        j += 1
    return base + e + j


def bucket_grid(L: int, num_buckets: int = 32, max_distance: int = 128) -> torch.Tensor:
    """int64 [L, L]: bucket of (key - query) for query row i, key column j"""
    table = torch.tensor([relative_position_bucket(n, num_buckets, max_distance) for n in range(-(L - 1), L)],
                         dtype=torch.long)
    rel = torch.arange(L)[None, :] - torch.arange(L)[:, None]
    return table[rel + L - 1]


def position_bias(sd, cfg, L, dtype=None):
    """[H, L, L]: the layer-0 relative_attention_bias table at the bucket of every (query, key)"""
    w = sd["encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"]
    w = w if dtype is None else w.to(dtype)
    idx = bucket_grid(L, cfg.relative_attention_num_buckets, cfg.relative_attention_max_distance).to(w.device)
    return w[idx].permute(2, 0, 1)


def t5_layer_norm(x, w, eps=1e-6):
    """x / rms(x) * w, no mean and no bias; the mean square in `_up`"""
    xf = x.to(_up(x.dtype))
    return w * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)).to(x.dtype)


def t5_attention(q, k, v, bias):
    """softmax(q k^T + bias) v over [B, H, L, dh] with bias [H, L, L]: no 1/sqrt(dh), no mask; softmax in `_up`"""
    s = q @ k.transpose(-1, -2) + bias
    p = torch.softmax(s.to(_up(s.dtype)), dim=-1).to(s.dtype)
    return p @ v


def gelu_tanh(x):
    """0.5 x (1 + tanh(sqrt(2 / pi) (x + 0.044715 x^3))), one elementwise step at a time in the dtype of x"""
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * torch.pow(x, 3.0))))


def t5_layer(sd, cfg, i, x, bias):
    """Block i on x [B, L, d] with the position bias [H, L, L].  -> {"xn1", "qkv" [B, L, 3 H dk] (q heads, then k, then
    v), "attn_out" [B, L, H dk], "x_mid" (after o + residual), "xn2", "gu" [B, L, 2 d_ff] ([wi_0 x | wi_1 x]), "h" (gated
    GELU), "x" (the block's output)}"""
    p = f"encoder.block.{i}.layer."
    H, eps = cfg.num_heads, cfg.layer_norm_epsilon
    xn1 = t5_layer_norm(x, sd[p + "0.layer_norm.weight"], eps)
    a = p + "0.SelfAttention."
    q, k, v = (_lin(sd, a + n, xn1) for n in "qkv")
    o = _flat(t5_attention(_heads(q, H), _heads(k, H), _heads(v, H), bias))
    x_mid = x + _lin(sd, a + "o", o)
    xn2 = t5_layer_norm(x_mid, sd[p + "1.layer_norm.weight"], eps)
    f = p + "1.DenseReluDense."
    g, u = _lin(sd, f + "wi_0", xn2), _lin(sd, f + "wi_1", xn2)
    h = gelu_tanh(g) * u
    out = x_mid + _lin(sd, f + "wo", h)
    return {"xn1": xn1, "qkv": torch.cat([q, k, v], -1), "attn_out": o, "x_mid": x_mid, "xn2": xn2,
            "gu": torch.cat([g, u], -1), "h": h, "x": out}


def t5_embed(sd, ids):
    return sd["shared.weight"][ids]


def t5_final(sd, cfg, x):
    return t5_layer_norm(x, sd["encoder.final_layer_norm.weight"], cfg.layer_norm_epsilon)


def t5_forward(sd, cfg, ids):
    """last_hidden_state [B, L, d] of ids [B, L]"""
    x = t5_embed(sd, ids)
    bias = position_bias(sd, cfg, ids.shape[1])
    for i in range(cfg.num_layers):
        x = t5_layer(sd, cfg, i, x, bias)["x"]
    return t5_final(sd, cfg, x)


def t5_state_dict_spec(cfg) -> dict[str, tuple]:
    d, inner, ff = cfg.d_model, cfg.num_heads * cfg.d_kv, cfg.d_ff
    s = {"shared.weight": (cfg.vocab_size, d),
         "encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight": (cfg.relative_attention_num_buckets,
                                                                                  cfg.num_heads)}
    for i in range(cfg.num_layers):
        p = f"encoder.block.{i}.layer."
        for n in "qkv":
            s[p + f"0.SelfAttention.{n}.weight"] = (inner, d)
        s[p + "0.SelfAttention.o.weight"] = (d, inner)
        s[p + "0.layer_norm.weight"] = s[p + "1.layer_norm.weight"] = (d,)
        s[p + "1.DenseReluDense.wi_0.weight"] = s[p + "1.DenseReluDense.wi_1.weight"] = (ff, d)
        s[p + "1.DenseReluDense.wo.weight"] = (d, ff)
    s["encoder.final_layer_norm.weight"] = (d,)
    return s


# ------------------------------------------------------------------------------------------------ CLIP
def layer_norm(x, w, b, eps=1e-5):
    return F.layer_norm(x, (x.shape[-1],), w, b, eps)


def causal_mask(L, device=None):
    """[L, L] boolean: query i sees keys 0..i"""
    return torch.ones(L, L, dtype=torch.bool, device=device).tril()


def clip_attention(q, k, v, scale):
    """causal softmax(q k^T * scale) v over [B, H, L, dh]; softmax in `_up`.  bf16 on a GPU goes through
    F.scaled_dot_product_attention."""
    if q.is_cuda and q.dtype != torch.float64:
        return F.scaled_dot_product_attention(q, k, v, is_causal=True, scale=scale)
    s = (q @ k.transpose(-1, -2)) * scale
    s = s.masked_fill(~causal_mask(q.shape[2], q.device), float("-inf"))
    return torch.softmax(s.to(_up(s.dtype)), dim=-1).to(s.dtype) @ v


def quick_gelu(x):
    return x * torch.sigmoid(1.702 * x)


def clip_layer(sd, cfg, i, x):
    """Layer i on x [B, L, d].  -> {"xn1", "qkv" [B, L, 3 d] (q heads, then k, then v), "attn_out", "x_mid" (after
    out_proj + residual), "xn2", "fc1" (after quick-GELU), "x" (the layer's output)}"""
    p = f"text_model.encoder.layers.{i}."
    H, eps = cfg.num_attention_heads, cfg.layer_norm_eps
    hd = cfg.hidden_size // H
    xn1 = layer_norm(x, sd[p + "layer_norm1.weight"], sd[p + "layer_norm1.bias"], eps)
    a = p + "self_attn."
    q, k, v = (_lin(sd, a + n, xn1) for n in ("q_proj", "k_proj", "v_proj"))
    o = _flat(clip_attention(_heads(q, H), _heads(k, H), _heads(v, H), hd ** -0.5))
    x_mid = x + _lin(sd, a + "out_proj", o)
    xn2 = layer_norm(x_mid, sd[p + "layer_norm2.weight"], sd[p + "layer_norm2.bias"], eps)
    fc1 = quick_gelu(_lin(sd, p + "mlp.fc1", xn2))
    out = x_mid + _lin(sd, p + "mlp.fc2", fc1)
    return {"xn1": xn1, "qkv": torch.cat([q, k, v], -1), "attn_out": o, "x_mid": x_mid, "xn2": xn2, "fc1": fc1, "x": out}


def clip_embed(sd, ids):
    L = ids.shape[1]
    return sd["text_model.embeddings.token_embedding.weight"][ids] + sd["text_model.embeddings.position_embedding.weight"][:L]


def eos_positions(ids, eos_token_id):
    """the pooled token of each row of ids [B, L]: argmax(ids) under the legacy eos_token_id == 2 rule (the largest id
    marks the end of text), else the first position holding eos_token_id; a tie goes to the first position"""
    ids = ids.cpu()
    if eos_token_id == 2:
        return torch.tensor([max(range(len(r)), key=lambda j: (r[j], -j)) for r in ids.tolist()])
    return torch.tensor([r.index(eos_token_id) for r in ids.tolist()])


def clip_final(sd, cfg, x, ids):
    """(last_hidden_state [B, L, d], pooler_output [B, d])"""
    last = layer_norm(x, sd["text_model.final_layer_norm.weight"], sd["text_model.final_layer_norm.bias"],
                      cfg.layer_norm_eps)
    pos = eos_positions(ids, cfg.eos_token_id).to(last.device)
    return last, last[torch.arange(last.shape[0], device=last.device), pos]


def clip_forward(sd, cfg, ids):
    x = clip_embed(sd, ids)
    for i in range(cfg.num_hidden_layers):
        x = clip_layer(sd, cfg, i, x)["x"]
    return clip_final(sd, cfg, x, ids)


def clip_state_dict_spec(cfg) -> dict[str, tuple]:
    d, I = cfg.hidden_size, cfg.intermediate_size
    s = {"text_model.embeddings.token_embedding.weight": (cfg.vocab_size, d),
         "text_model.embeddings.position_embedding.weight": (cfg.max_position_embeddings, d)}
    for i in range(cfg.num_hidden_layers):
        p = f"text_model.encoder.layers.{i}."
        for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
            s[p + f"self_attn.{n}.weight"], s[p + f"self_attn.{n}.bias"] = (d, d), (d,)
        for n in ("layer_norm1", "layer_norm2"):
            s[p + f"{n}.weight"] = s[p + f"{n}.bias"] = (d,)
        s[p + "mlp.fc1.weight"], s[p + "mlp.fc1.bias"] = (I, d), (I,)
        s[p + "mlp.fc2.weight"], s[p + "mlp.fc2.bias"] = (d, I), (d,)
    s["text_model.final_layer_norm.weight"] = s["text_model.final_layer_norm.bias"] = (d,)
    return s


# ------------------------------------------------------------------------------------------------ weights
def _synthetic(spec, seed, dtype, device):
    """Random weights at fan_in^-1/2 (activations stay O(1) and every block's own share of the residual stream is a
    visible part of it), norm weights 1 + 0.1 N(0, 1), biases 0.1 N(0, 1), embeddings and the T5 bias table N(0, 1).
    Drawn on `device` in float32, one tensor at a time, then cast."""
    sd = {}
    g = torch.Generator(device=device).manual_seed(seed)
    for name, shape in spec.items():
        t = torch.randn(shape, generator=g, device=device)
        if name.endswith(".bias"):
            t.mul_(0.1)
        elif len(shape) == 1:
            t.mul_(0.1).add_(1.0)
        elif "embed" not in name and "shared" not in name and "relative_attention_bias" not in name:
            t.mul_(shape[1] ** -0.5)
        sd[name] = t.to(dtype)
    return sd


def make_t5_state_dict(cfg, seed: int = 0, dtype=torch.float32, device="cpu"):
    return _synthetic(t5_state_dict_spec(cfg), seed, dtype, device)


def make_clip_state_dict(cfg, seed: int = 0, dtype=torch.float32, device="cpu"):
    return _synthetic(clip_state_dict_spec(cfg), seed, dtype, device)
