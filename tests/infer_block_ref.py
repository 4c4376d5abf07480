"""Float64 references of the FLUX inference forward one stage at a time, and the gates that compare a stage's tensors
with them.

The engine's forward (`b2f_flux_forward`, csrc/flux_model.cu) runs in stages that `_b2f_block_range` can drive one at a
time: the embedders (`(0, 0)`), each transformer block (`(blk, blk + 1)`) and the tail (`(nblk, nblk)`, norm_out +
proj_out over the first n_out image rows).  The time-text embedding and the AdaLN modulation run before it
(`b2f_flux_temb`, `b2f_flux_modulation[_ws]`).  Each function here is the oracle's composition of one stage, built from
its pieces (`fo._lin`, `fo.layer_norm`, `fo.rms_norm`, `fo.apply_rotary_emb`, `fo.attention`, `fo.time_text_embed`) in
the oracle's op order, run in the dtype it is given: float64 for the reference, bfloat16 for the yardstick (what torch
in bf16 makes of the same inputs).  The stage inputs are the engine's bf16 tensors, so an error stays inside the stage
that made it.

Besides its output, each block stage returns the intermediates the engine's workspace still holds when the block
returns (`B200FluxTransformer2DModel.debug_buffers`), in the engine's layout:
  qkv  [B, S, 3d]  Q and K after RMSNorm + RoPE, and V; rows in the joint [txt; img] order, head-major columns
  attn [B, S, d]   the attention output
  mlp  [B, S, 4d]  the GELU'd MLP activations (a double block: text rows from ff_context, image rows from ff)
  xn   [B, S, d]   the modulated LayerNorm the MLP reads (a double block's second one; a single block's only one)

The gates are train_block_ref's: the per-tensor rule and the per-slice gate max_s e_s <= 2 max_s y_s + beta, over token
rows (text and image apart), channels, attention heads and modulation chunks.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

import train_block_ref as TB
from oracle import flux_oracle as fo

# additive allowance of the forward's per-slice gate, a tenth of the backward's.  Measured on an H100 over every case of
# test_flux_blocks_gpu.py, the engine's worst slice is within 1.17x the yardstick's and e - 2y <= -1.5e-3 in every
# family, so the forward passes even at beta = 0; 1e-3 keeps a floor for slices whose yardstick is exact.  At 1e-2 the
# gate would pass a 1 % error in one modulation chunk (e 1.1e-2 against y 1.8e-3, test_infer_block_ref_cpu.py).
BETA = 1e-3


def _sub(sd, prefix, dtype):
    """the weights under `prefix`, in `dtype` (one block at a time: a whole full-size model in float64 does not fit)."""
    return {k: v.to(dtype) for k, v in sd.items() if k.startswith(prefix)}


def _lin(sd, name, x):
    return fo._lin(_sub(sd, name + ".", x.dtype), name, x)


def _modulate(x, shift, scale):
    return fo.layer_norm(x) * (1 + scale[:, None]) + shift[:, None]


def _flat(t):
    """[B, H, S, dh] -> [B, S, H * dh]"""
    B, H, S, dh = t.shape
    return t.transpose(1, 2).reshape(B, S, H * dh)


def adaln_names(cfg):
    """the AdaLN linears in the column order of `mod` (b2f_flux_modulation)."""
    out = []
    for i in range(cfg.num_layers):
        out += [f"transformer_blocks.{i}.norm1.linear", f"transformer_blocks.{i}.norm1_context.linear"]
    out += [f"single_transformer_blocks.{i}.norm.linear" for i in range(cfg.num_single_layers)]
    return out + ["norm_out.linear"]


def chunk_names(cfg):
    """one label per d-wide chunk of `mod`: block, stream and chunk name."""
    out = []
    for i in range(cfg.num_layers):
        out += [f"double{i} img {n}" for n in TB.CHUNKS["double"]] + [f"double{i} txt {n}" for n in TB.CHUNKS["double"]]
    for i in range(cfg.num_single_layers):
        out += [f"single{i} {n}" for n in TB.CHUNKS["single"]]
    return out + [f"norm_out {n}" for n in TB.CHUNKS["norm_out"]]


# ------------------------------------------------------------------------------------------------ stages
def embed_stage(sd, hidden, enc, dtype):
    """x_embedder(hidden) and context_embedder(enc) as the joint buffer h = [c; x]."""
    c = _lin(sd, "context_embedder", enc.to(dtype))
    x = _lin(sd, "x_embedder", hidden.to(dtype))
    return {"h": torch.cat([c, x], 1)}


def temb_stage(sd, cfg, t1000, g1000, pooled, dtype):
    """time_text_embed of the values the engine receives (`_times1000`: bf16(t) * 1000 in bf16, as fp32)."""
    temb = fo.time_text_embed(_sub(sd, "time_text_embed.", dtype), cfg, t1000, g1000, pooled.to(dtype))
    return {"temb": temb, "silu": F.silu(temb)}


def modulation_stage(sd, cfg, silu_temb, dtype):
    """every AdaLN linear of silu(temb), laid out as `TB.mod_offsets` says: [rows, mod_width]."""
    s = silu_temb.to(dtype)
    return {"mod": torch.cat([_lin(sd, n, s) for n in adaln_names(cfg)], 1)}


def _qkv(w, p, x, names, norms, H):
    q = fo.rms_norm(fo._heads(fo._lin(w, p + names[0], x), H), w[p + norms[0] + ".weight"])
    k = fo.rms_norm(fo._heads(fo._lin(w, p + names[1], x), H), w[p + norms[1] + ".weight"])
    v = fo._heads(fo._lin(w, p + names[2], x), H)
    return q, k, v


def _attend(q, k, v, cos, sin):
    """`fo.joint_attention` after its projections: RoPE on q / k, attention, heads flattened."""
    q, k = fo.apply_rotary_emb(q, cos, sin), fo.apply_rotary_emb(k, cos, sin)
    o = _flat(fo.attention(q, k, v)).to(q.dtype)
    return o, torch.cat([_flat(q), _flat(k), _flat(v)], -1)


def double_stage(sd, cfg, blk, h_in, mod, cos, sin, S_txt, dtype):
    """`fo.double_block_mod` on the joint buffer h_in [B, S, d] (text rows first) with its intermediates."""
    d, H = cfg.inner_dim, cfg.num_attention_heads
    p = f"transformer_blocks.{blk}."
    w = _sub(sd, p, dtype)
    o = TB.mod_offsets(cfg)[0][blk]
    m = mod[:, o:o + 12 * d].to(dtype)
    shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp = m[:, :6 * d].chunk(6, dim=1)
    c_shift_msa, c_scale_msa, c_gate_msa, c_shift_mlp, c_scale_mlp, c_gate_mlp = m[:, 6 * d:].chunk(6, dim=1)
    h = h_in.to(dtype)
    c, x = h[:, :S_txt], h[:, S_txt:]

    xn = _modulate(x, shift_msa, scale_msa)
    cn = _modulate(c, c_shift_msa, c_scale_msa)
    a = p + "attn."
    q, k, v = _qkv(w, a, xn, ("to_q", "to_k", "to_v"), ("norm_q", "norm_k"), H)
    cq, ck, cv = _qkv(w, a, cn, ("add_q_proj", "add_k_proj", "add_v_proj"), ("norm_added_q", "norm_added_k"), H)
    attn, qkv = _attend(torch.cat([cq, q], 2), torch.cat([ck, k], 2), torch.cat([cv, v], 2), cos, sin)
    attn_x, attn_c = fo._lin(w, a + "to_out.0", attn[:, S_txt:]), fo._lin(w, a + "to_add_out", attn[:, :S_txt])

    x = x + gate_msa.unsqueeze(1) * attn_x
    xn2 = _modulate(x, shift_mlp, scale_mlp)
    act = F.gelu(fo._lin(w, p + "ff.net.0.proj", xn2), approximate="tanh")
    x = x + gate_mlp.unsqueeze(1) * fo._lin(w, p + "ff.net.2", act)

    c = c + c_gate_msa.unsqueeze(1) * attn_c
    cn2 = _modulate(c, c_shift_mlp, c_scale_mlp)
    cact = F.gelu(fo._lin(w, p + "ff_context.net.0.proj", cn2), approximate="tanh")
    c = c + c_gate_mlp.unsqueeze(1) * fo._lin(w, p + "ff_context.net.2", cact)
    return {"h": torch.cat([c, x], 1), "qkv": qkv, "attn": attn, "mlp": torch.cat([cact, act], 1),
            "xn": torch.cat([cn2, xn2], 1)}


def single_stage(sd, cfg, si, h_in, mod, cos, sin, dtype):
    """`fo.single_block_mod` with its intermediates."""
    d, H = cfg.inner_dim, cfg.num_attention_heads
    p = f"single_transformer_blocks.{si}."
    w = _sub(sd, p, dtype)
    o = TB.mod_offsets(cfg)[1][si]
    shift, scale, gate = mod[:, o:o + 3 * d].to(dtype).chunk(3, dim=1)
    h = h_in.to(dtype)
    hn = _modulate(h, shift, scale)
    mlp = F.gelu(fo._lin(w, p + "proj_mlp", hn), approximate="tanh")
    attn, qkv = _attend(*_qkv(w, p + "attn.", hn, ("to_q", "to_k", "to_v"), ("norm_q", "norm_k"), H), cos, sin)
    out = gate.unsqueeze(1) * fo._lin(w, p + "proj_out", torch.cat([attn, mlp], dim=2))
    return {"h": h + out, "qkv": qkv, "attn": attn, "mlp": mlp, "xn": hn}


def tail_stage(sd, cfg, h_fin, mod, S_txt, n_out, dtype):
    """norm_out (AdaLayerNormContinuous: scale first) and proj_out on the first n_out image rows."""
    d = cfg.inner_dim
    o = TB.mod_offsets(cfg)[2]
    scale, shift = mod[:, o:o + 2 * d].to(dtype).chunk(2, dim=1)
    x = h_fin[:, S_txt:S_txt + n_out].to(dtype)
    xn = fo.layer_norm(x) * (1 + scale)[:, None, :] + shift[:, None, :]
    return {"xn": xn, "out": _lin(sd, "proj_out", xn)}


# ------------------------------------------------------------------------------------------------ gates
def _by_head(t, head_dim=128):
    """[..., n * head_dim] -> [n, rest]: one row per head."""
    t = t.double()
    n = t.shape[-1] // head_dim
    return t.reshape(-1, n, head_dim).transpose(0, 1).reshape(n, -1)


def token_gates(stage, name, K, R, Y, S_txt, kinds=("rows", "cols"), heads=False, base=None):
    """gates of a [B, S, n] activation: token rows and channels of the text and the image rows apart; heads=True adds
    one slice per attention head (per q / k / v head when n = 3d).  With `base` (the block input) the same gates again
    on the block's own share K - base, which the residual identity would otherwise swamp."""
    B, S = K.shape[:2]
    out = []
    for part, sl, lab in (("text", slice(None, S_txt), TB.token_label(B, S_txt, S_txt)),
                          ("image", slice(S_txt, None), TB.token_label(B, S - S_txt, 0))):
        if not K[:, sl].numel():
            continue
        out += TB.gate(stage, f"{name} {part}", K[:, sl], R[:, sl], Y[:, sl], kinds, lab, beta=BETA)
        if base is not None:
            b = base[:, sl].double()
            out += TB.gate(stage, f"{name} - {name}_in {part}", K[:, sl].double() - b, R[:, sl].double() - b,
                           Y[:, sl].double() - b, kinds, lab, beta=BETA)
    if heads:
        n = K.shape[-1] // 128
        lab = TB.qkv_label(n // 3, 1) if n % 3 == 0 and name == "qkv" else (lambda kind, i: f"head {i}")
        out += [c for c in TB.gate(stage, f"{name} heads", _by_head(K), _by_head(R), _by_head(Y), ("rows",), lab, beta=BETA)
                if c.kind != "tensor"]
    return out


def row_gates(stage, name, K, R, Y):
    """gates of a [rows, n] tensor whose rows are (step, batch) rows of a schedule: rows and channels."""
    return TB.gate(stage, name, K, R, Y, ("rows", "cols"), beta=BETA)


def mod_gates(stage, K, R, Y, cfg):
    """gates of `mod` [rows, mod_width]: rows, columns and every d-wide chunk, labelled by block and chunk name."""
    d = cfg.inner_dim
    names = chunk_names(cfg)
    assert len(names) * d == K.shape[1]
    ch = lambda t: t.double().reshape(-1, len(names), d).transpose(0, 1)
    out = row_gates(stage, "mod", K, R, Y)
    out += [c for c in TB.gate(stage, "mod", ch(K), ch(R), ch(Y), ("chunks",), TB.chunk_label(names),
                               n_chunks=len(names), beta=BETA) if c.kind != "tensor"]
    return out


def block_gates(stage, K, R, Y, h_in, S_txt):
    """every gate of a block stage: K / R / Y are {h, qkv, attn, mlp, xn}."""
    out = token_gates(stage, "h", K["h"], R["h"], Y["h"], S_txt, base=h_in)
    out += token_gates(stage, "qkv", K["qkv"], R["qkv"], Y["qkv"], S_txt, heads=True)
    out += token_gates(stage, "attn", K["attn"], R["attn"], Y["attn"], S_txt, heads=True)
    out += token_gates(stage, "mlp", K["mlp"], R["mlp"], Y["mlp"], S_txt)
    out += token_gates(stage, "xn", K["xn"], R["xn"], Y["xn"], S_txt)
    return out
