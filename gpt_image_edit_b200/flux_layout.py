"""The FLUX denoiser's weights as the engine stores them, written out once.

Every engine target (the name b2f_flux_bind_weight / b2f_flux_bind_lora / b2f_flux_bind_fp8 take) with its
(out, in) shape and the diffusers nn.Linear rows it holds, in the order lora.targets lists them.  A target is an
embedder ("embedder": the embedders and proj_out), a block linear ("block": the FP8-capable linears; q/k/v and the
single block's q/k/v/proj_mlp are fused into one) or an AdaLN linear ("adaln": rows of the fused `adaln` weight, which
concatenates them in this order).  flux_transformer builds its storage and state-dict views from this list, lora its
targets and diffusers parts.  The engine's own list is for_each_linear in csrc/flux_model.cu.
"""
from __future__ import annotations

from typing import NamedTuple


class Target(NamedTuple):
    name: str
    kind: str     # "embedder", "block" or "adaln"
    out: int
    inp: int
    parts: tuple  # ((diffusers name, row0, rows), ...) in row order


def layout(cfg) -> "list[Target]":
    d = cfg.num_attention_heads * cfg.attention_head_dim
    out = []

    def add(kind, name, o, k, parts=None):
        if parts is None:
            parts = ((name, 0, o),)
        else:   # (diffusers name, rows) -> (diffusers name, row0, rows)
            row0 = [sum(n for _, n in parts[:j]) for j in range(len(parts))]
            parts = tuple((p, r, n) for (p, n), r in zip(parts, row0))
        out.append(Target(name, kind, o, k, parts))

    add("embedder", "x_embedder", d, cfg.in_channels)
    add("embedder", "context_embedder", d, cfg.joint_attention_dim)
    for e, k in [("timestep_embedder", 256), ("text_embedder", cfg.pooled_projection_dim)] + \
            ([("guidance_embedder", 256)] if cfg.guidance_embeds else []):
        add("embedder", f"time_text_embed.{e}.linear_1", d, k)
        add("embedder", f"time_text_embed.{e}.linear_2", d, d)
    for i in range(cfg.num_layers):
        p = f"transformer_blocks.{i}."
        add("block", p + "attn.qkv", 3 * d, d, [(p + "attn.to_" + n, d) for n in "qkv"])
        add("block", p + "attn.add_qkv", 3 * d, d, [(p + f"attn.add_{n}_proj", d) for n in "qkv"])
        for n, o, k in (("attn.to_out.0", d, d), ("attn.to_add_out", d, d), ("ff.net.0.proj", 4 * d, d),
                        ("ff.net.2", d, 4 * d), ("ff_context.net.0.proj", 4 * d, d), ("ff_context.net.2", d, 4 * d)):
            add("block", p + n, o, k)
        add("adaln", p + "norm1.linear", 6 * d, d)
        add("adaln", p + "norm1_context.linear", 6 * d, d)
    for i in range(cfg.num_single_layers):
        p = f"single_transformer_blocks.{i}."
        add("block", p + "qkv_mlp", 7 * d, d, [(p + "attn.to_" + n, d) for n in "qkv"] + [(p + "proj_mlp", 4 * d)])
        add("block", p + "proj_out", d, 5 * d)
        add("adaln", p + "norm.linear", 3 * d, d)
    add("adaln", "norm_out.linear", 2 * d, d)
    add("embedder", "proj_out", cfg.out_channels, d)
    return out


def norm_weights(cfg) -> "list[str]":
    """The blocks' per-head RMSNorm weights, [attention_head_dim] each."""
    out = []
    for i in range(cfg.num_layers):
        p = f"transformer_blocks.{i}.attn."
        out += [p + n + ".weight" for n in ("norm_q", "norm_k", "norm_added_q", "norm_added_k")]
    for i in range(cfg.num_single_layers):
        p = f"single_transformer_blocks.{i}.attn."
        out += [p + "norm_q.weight", p + "norm_k.weight"]
    return out
