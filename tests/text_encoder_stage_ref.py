"""Float64 references of the T5-XXL and CLIP-L prompt encoders one stage at a time, and the gates that compare a stage's
tensors with them.

`B200T5Encoder` and `B200CLIPTextModel` (gpt_image_edit_b200/text_encoders.py) run in stages a test can drive one at a
time: `_t5_embed`, `_t5_layer(i)` and `_t5_final`; `_clip_embed`, `_clip_layer(i)` and `_clip_final` (final LayerNorm and
the pooled gather).  Each function here is the oracle's stage (oracle/text_encoder_oracle.py), run in the dtype it is
given: float64 for the reference, bfloat16 for the yardstick (what transformers in bf16 makes of the same inputs: T5
attention in its eager form, CLIP attention through F.scaled_dot_product_attention on a GPU).  The stage inputs are the
engine's bf16 tensors, so an error stays inside the stage that made it.  The oracle builds its own bucket grid and
causal mask, so the engine's are checked, not reused.

The engine lays every 64-wide head out in a 128-wide slot: `strip_heads` takes the 64 real columns out of `qkv` and
`attn_out` before gating, and `padding` returns the other 64 for an exact zero check.

The gates are train_block_ref's per-tensor rule and per-slice gate at `infer_block_ref.BETA`, over token rows, channels
and heads (the 64 real columns of each q, k, v and attention-output head), and for the residual outputs again on the
stage's own share, output - input.
"""
from __future__ import annotations

import torch

import infer_block_ref as IB
import train_block_ref as TB
from oracle import text_encoder_oracle as to

HP = 128  # the engine's head slot


# ------------------------------------------------------------------------------------------------ engine layout
def strip_heads(t, hd=64):
    """[..., n * 128] in head slots -> [..., n * hd], the real columns"""
    return t.unflatten(-1, (-1, HP))[..., :hd].flatten(-2)


def padding(keep, hd=64):
    """the padding columns of a layer's head-slot buffers: {name: tensor} that must all be exactly zero"""
    return {f"qkv[..., {hd}:128]": keep["qkv"].unflatten(-1, (-1, HP))[..., hd:],
            f"attn_out[..., {hd}:128]": keep["attn_out"].unflatten(-1, (-1, HP))[..., hd:]}


# ------------------------------------------------------------------------------------------------ stages
_sub = IB._sub


def t5_embed_stage(sd, ids, dtype):
    """the rows of the table gathered in its own dtype, then cast (a float64 copy of the table is never made)"""
    return to.t5_embed(sd, ids.to(sd["shared.weight"].device)).to(dtype)


def t5_layer_stage(sd, cfg, i, x_in, dtype, bias=None):
    """block i on the engine's block input x_in [B, L, d] -> the oracle's {"xn1", "qkv", "attn_out", "x_mid", "xn2",
    "gu", "h", "x"}; `bias` [H, L, L] replaces the oracle's own position bias (planted faults)"""
    if bias is None:
        bias = to.position_bias(sd, cfg, x_in.shape[1], dtype)
    w = _sub(sd, f"encoder.block.{i}.", dtype)
    return to.t5_layer(w, cfg, i, x_in.to(dtype), bias.to(dtype))


def t5_final_stage(sd, cfg, x_in, dtype):
    return to.t5_final(_sub(sd, "encoder.final_layer_norm.", dtype), cfg, x_in.to(dtype))


def clip_embed_stage(sd, ids, dtype):
    """token rows gathered in the table's own dtype, the sum in `dtype`"""
    tok = sd["text_model.embeddings.token_embedding.weight"]
    w = {"text_model.embeddings.token_embedding.weight": tok[ids.reshape(-1).to(tok.device)].to(dtype),
         "text_model.embeddings.position_embedding.weight": sd["text_model.embeddings.position_embedding.weight"].to(dtype)}
    return to.clip_embed(w, torch.arange(ids.numel(), device=tok.device).view(ids.shape))


def clip_layer_stage(sd, cfg, i, x_in, dtype):
    """layer i on the engine's layer input x_in [B, L, d] -> the oracle's {"xn1", "qkv", "attn_out", "x_mid", "xn2",
    "fc1", "x"}"""
    return to.clip_layer(_sub(sd, f"text_model.encoder.layers.{i}.", dtype), cfg, i, x_in.to(dtype))


def clip_final_stage(sd, cfg, x_in, ids, dtype):
    """{"last" [B, L, d], "pooled" [B, d]}"""
    last, pooled = to.clip_final(_sub(sd, "text_model.final_layer_norm.", dtype), cfg, x_in.to(dtype), ids)
    return {"last": last, "pooled": pooled}


# ------------------------------------------------------------------------------------------------ gates
def _by_head(t, hd):
    t = t.double()
    n = t.shape[-1] // hd
    return t.reshape(-1, n, hd).transpose(0, 1).reshape(n, -1)


def head_labels(name, n):
    """labels of the heads of `qkv` (n = 3 H: q heads, then k, then v) or of an attention output (n = H)"""
    if name == "qkv":
        return [f"{'qkv'[j // (n // 3)]} head {j % (n // 3)}" for j in range(n)]
    return [f"head {j}" for j in range(n)]


def enc_gates(stage, name, K, R, Y, heads=None, base=None):
    """gates of an activation [B, L, n]: token rows and channels, with heads = head_dim one slice per head, and with
    `base` (the stage input) the rows and channels again on the stage's own share K - base."""
    L = K.shape[1]
    flat = lambda t: t.double().reshape(-1, t.shape[-1])
    lab = lambda kind, i: f"batch {i // L} token {i % L}" if kind == "rows" else f"{kind[:-1]} {i}"
    k, r, y = flat(K), flat(R), flat(Y)
    out = TB.gate(stage, name, k, r, y, ("rows", "cols"), lab, beta=IB.BETA)
    if base is not None:
        b = flat(base)
        out += TB.gate(stage, f"{name} - {name}_in", k - b, r - b, y - b, ("rows", "cols"), lab, beta=IB.BETA)
    if heads is not None:
        names = head_labels(name, K.shape[-1] // heads)
        out += [c for c in TB.gate(stage, f"{name} heads", _by_head(k, heads), _by_head(r, heads), _by_head(y, heads),
                                   ("rows",), lambda kind, i: names[i], beta=IB.BETA) if c.kind != "tensor"]
    return out


def layer_gates(stage, K, R, Y, x_in, hd=64):
    """every gate of a T5 block or a CLIP layer: K the engine's buffers (head slots stripped), R / Y the oracle's"""
    out = []
    for name in K:
        heads = hd if name in ("qkv", "attn_out") else None
        base = x_in if name in ("x", "x_mid") else None
        out += enc_gates(stage, name, K[name], R[name], Y[name], heads=heads, base=base)
    return out


def pooled_gates(stage, K, R, Y):
    """gates of the pooled rows [B, d]: one slice per batch row and per channel"""
    lab = lambda kind, i: f"batch {i}" if kind == "rows" else f"{kind[:-1]} {i}"
    return TB.gate(stage, "pooled", K, R, Y, ("rows", "cols"), lab, beta=IB.BETA)
