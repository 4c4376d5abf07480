"""ORACLE — TEST INFRASTRUCTURE ONLY (see oracle/flux_oracle.py for the rules).

PyTorch restatement of the Qwen2.5-VL arithmetic the reference reaches through transformers 4.50
(`Qwen2_5_VisionTransformerPretrainedModel`, `Qwen2_5_VLModel`), written from the model's math: a ViT of pre-norm blocks
with 2-D RoPE over windowed and full bidirectional attention, a 2x2 patch merger, and a decoder of pre-norm layers with
M-RoPE and causal grouped-query attention.  It takes weights under the transformers-4.50 names at their true shapes
(vision head_dim 80, MLP 3420: no padding), so it knows nothing of the engine's kernel layout.

Every function runs in the dtype of its inputs: float64 gives the exact-math answer, bfloat16 what torch-eager does in
bf16.  Where transformers computes in float32 inside a bf16 model (RMSNorm's statistics, the vision RoPE, the rotary
angles) a bf16 run does the same, so the bf16 run is the yardstick the engine is held to.  Pinned against transformers'
`Qwen2_5_VLModel` in float64 by tests/test_qwen_stage_ref_cpu.py.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def _up(dtype):
    """the compute dtype of a step transformers runs in float32 (float64 stays float64)."""
    return torch.promote_types(dtype, torch.float32)


def rms_norm(x, w, eps=1e-6):
    xf = x.to(_up(x.dtype))
    return w * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)).to(x.dtype)


def _lin(sd, name, x):
    return F.linear(x, sd[name + ".weight"], sd.get(name + ".bias"))


def rotate_half(x):
    h = x.shape[-1] // 2
    return torch.cat((-x[..., h:], x[..., :h]), dim=-1)


def attention(q, k, v, mask=None, scale=None):
    """softmax(q k^T * scale + mask) v over [B, H, S, dh] (k / v may have fewer heads: grouped-query, head h reads KV head
    h // (H / Hkv)).  `mask` is boolean (True = attend).  bf16 on a GPU goes through F.scaled_dot_product_attention."""
    H, Hkv = q.shape[1], k.shape[1]
    if Hkv != H:
        k, v = k.repeat_interleave(H // Hkv, dim=1), v.repeat_interleave(H // Hkv, dim=1)
    scale = scale if scale is not None else q.shape[-1] ** -0.5
    if q.is_cuda and q.dtype != torch.float64:
        return F.scaled_dot_product_attention(q, k, v, attn_mask=mask, scale=scale)
    s = (q @ k.transpose(-1, -2)) * scale
    if mask is not None:
        s = s.masked_fill(~mask, float("-inf"))
    return torch.softmax(s, dim=-1) @ v


# ------------------------------------------------------------------------------------------------ vision tower
def patch_embed(sd, pix):
    """Conv3d with kernel = stride = (2, 14, 14) and no bias over [T, C*2*14*14] patches: a linear map."""
    w = sd["visual.patch_embed.proj.weight"]
    return pix @ w.reshape(w.shape[0], -1).transpose(0, 1)


def patch_positions(grid, merge=2):
    """(row, col) of every patch in the processor's order: per frame, merged 2x2 units row-major, patches row-major in a
    unit."""
    out = []
    for t, h, w in grid:
        r = torch.arange(h).view(h // merge, 1, merge, 1).expand(-1, w // merge, -1, merge)
        c = torch.arange(w).view(1, w // merge, 1, merge).expand(h // merge, -1, merge, -1)
        out.append(torch.stack([r.reshape(-1), c.reshape(-1)], -1).repeat(t, 1))
    return torch.cat(out)


def vision_rope(grid, head_dim, merge=2, theta=10000.0, dtype=torch.float64):
    """cos, sin [T, head_dim] in patch order: the first half of the rotary width turns with the patch row, the second
    with the column, each at the frequencies theta^(-2j / (head_dim / 2)); the angles are computed in `_up(dtype)`."""
    dim = head_dim // 2
    inv = 1.0 / theta ** (torch.arange(0, dim, 2, dtype=_up(dtype)) / dim)
    pos = patch_positions(grid, merge).to(_up(dtype))
    ang = torch.cat([pos[:, :1] * inv, pos[:, 1:] * inv], -1)
    emb = torch.cat([ang, ang], -1)
    return emb.cos(), emb.sin()


def window_index(grid, window_size=112, merge=2, patch=14):
    """(merged-token permutation into window order, cu_seqlens of the windows in patches).  A window covers
    window_size / patch / merge merged tokens a side; windows run row-major over the merged grid of every frame and
    tokens row-major inside a window; windows at the right and bottom edges are cut short."""
    vw = window_size // merge // patch
    idx, cu, off = [], [0], 0
    for t, h, w in grid:
        gh, gw = h // merge, w // merge
        for f in range(t):
            for r0 in range(0, gh, vw):
                for c0 in range(0, gw, vw):
                    rr = torch.arange(r0, min(r0 + vw, gh))
                    cc = torch.arange(c0, min(c0 + vw, gw))
                    tok = (off + f * gh * gw + rr[:, None] * gw + cc[None, :]).reshape(-1)
                    idx.append(tok)
                    cu.append(cu[-1] + tok.numel() * merge * merge)
        off += t * gh * gw
    return torch.cat(idx), cu


def full_cu_seqlens(grid):
    """cu_seqlens of full attention: one segment per frame."""
    cu = [0]
    for t, h, w in grid:
        cu += [cu[-1] + h * w * (f + 1) for f in range(t)]
    return cu


def segment_mask(cu, device=None):
    """[T, T] boolean: token i attends to token j when both lie in the same segment cu[s]:cu[s+1]."""
    seg = torch.repeat_interleave(torch.arange(len(cu) - 1), torch.tensor(cu[1:]) - torch.tensor(cu[:-1]))
    return (seg[:, None] == seg[None, :]).to(device)


def vision_block(sd, i, x, cos, sin, cu, vc):
    """ViT block i on x [T, hidden] with RoPE tables cos / sin [T, 80] in the same token order and attention
    restricted to the segments of `cu`.  -> {"h", "qkv" [T, 3, heads, 80] after RoPE, "attn" [T, heads*80],
    "a" [T, intermediate] (SwiGLU output)}."""
    p = f"visual.blocks.{i}."
    T, d = x.shape
    nh = vc.num_heads
    hd = d // nh
    xn = rms_norm(x, sd[p + "norm1.weight"])
    q, k, v = _lin(sd, p + "attn.qkv", xn).reshape(T, 3, nh, hd).unbind(1)
    up = _up(x.dtype)
    c, s = cos.to(up)[:, None], sin.to(up)[:, None]
    q = (q.to(up) * c + rotate_half(q.to(up)) * s).to(x.dtype)
    k = (k.to(up) * c + rotate_half(k.to(up)) * s).to(x.dtype)
    mask = segment_mask(cu, x.device)
    o = attention(q.transpose(0, 1)[None], k.transpose(0, 1)[None], v.transpose(0, 1)[None], mask, hd ** -0.5)
    attn = o[0].transpose(0, 1).reshape(T, d)
    h = x + _lin(sd, p + "attn.proj", attn)
    hn = rms_norm(h, sd[p + "norm2.weight"])
    a = F.silu(_lin(sd, p + "mlp.gate_proj", hn)) * _lin(sd, p + "mlp.up_proj", hn)
    h = h + _lin(sd, p + "mlp.down_proj", a)
    return {"h": h, "qkv": torch.stack([q, k, v], 1), "attn": attn, "a": a}


def merger(sd, x, merge=2):
    """ln_q (RMSNorm), every merge x merge consecutive tokens concatenated, Linear · erf-GELU · Linear."""
    xn = rms_norm(x, sd["visual.merger.ln_q.weight"]).reshape(x.shape[0] // merge ** 2, -1)
    return _lin(sd, "visual.merger.mlp.2", F.gelu(_lin(sd, "visual.merger.mlp.0", xn)))


def vision_forward(sd, vc, pix, grid):
    """The vision tower: merged image embeddings [T/4, out_hidden] in the processor's (un-windowed) token order."""
    m = vc.spatial_merge_size
    unit = m * m
    widx, cu_win = window_index(grid, vc.window_size, m, vc.patch_size)
    cu_full = full_cu_seqlens(grid)
    x = patch_embed(sd, pix)
    T = x.shape[0]
    perm = (widx[:, None] * unit + torch.arange(unit)).reshape(-1).to(x.device)      # patch order -> window order
    cos, sin = vision_rope(grid, vc.hidden_size // vc.num_heads, m, dtype=x.dtype)
    x, cos, sin = x[perm], cos.to(x.device)[perm], sin.to(x.device)[perm]
    for i in range(vc.depth):
        x = vision_block(sd, i, x, cos, sin, cu_full if i in vc.fullatt_block_indexes else cu_win, vc)["h"]
    merged = merger(sd, x, m)
    assert merged.shape[0] == T // unit
    return merged[torch.argsort(widx).to(x.device)]


# ------------------------------------------------------------------------------------------------ decoder
def mrope(pos, head_dim, theta, section, dtype=torch.float64):
    """cos, sin [B, L, head_dim] of M-RoPE position ids pos [3, B, L] (t, h, w): column pair j of the rotary half turns
    at theta^(-2j / head_dim) times the position on the axis whose section holds j (sections of `section` columns:
    t, then h, then w).  Angles in `_up(dtype)`, tables returned in `dtype`, as transformers casts them."""
    inv = 1.0 / theta ** (torch.arange(0, head_dim, 2, dtype=_up(dtype)) / head_dim)
    axis = torch.repeat_interleave(torch.arange(3), torch.tensor(list(section)))           # [head_dim / 2]
    p = pos.to(_up(dtype))                                                                   # [3, B, L]
    ang = p[axis].permute(1, 2, 0) * inv                                                     # [B, L, head_dim / 2]
    emb = torch.cat([ang, ang], -1)
    return emb.cos().to(dtype), emb.sin().to(dtype)


def causal_mask(L, spans=None, device=None):
    """[B or 1, 1, L, L] boolean: causal, and with spans [(lo, hi)] per sequence only within [lo, hi).  A padding row
    has no key: it is handled by the caller."""
    m = torch.ones(L, L, dtype=torch.bool).tril()
    if spans is None:
        return m[None, None].to(device)
    inside = torch.zeros(len(spans), L, dtype=torch.bool)
    for b, (lo, hi) in enumerate(spans):
        inside[b, lo:hi] = True
    return (m[None] & inside[:, None, :] & inside[:, :, None])[:, None].to(device)


def decoder_layer(sd, i, x, cos, sin, tc, spans=None, past_kv=None, past_lo=None):
    """Decoder layer i on x [B, L, hidden] with M-RoPE tables cos / sin [B, L, head_dim].

    Prefill (past_kv None): causal GQA; with spans [(lo, hi)] per sequence the tokens attend within their own span only
    and a token outside its span gets a zero attention output (flash-attention-2's unpad / pad).  Decode (past_kv =
    (K, V) [B, P, kv_heads, head_dim] after RoPE, L == 1): the new token attends to K/V rows past_lo[b]:P of its
    sequence and to itself.
    -> {"h", "q" [B, L, heads, hd], "k", "v" [B, L, kv_heads, hd] (after RoPE), "attn" [B, L, heads*hd], "a"}."""
    p = f"model.layers.{i}."
    B, L, d = x.shape
    nq, nkv = tc.num_attention_heads, tc.num_key_value_heads
    hd = d // nq
    xn = rms_norm(x, sd[p + "input_layernorm.weight"], tc.rms_norm_eps)
    q = _lin(sd, p + "self_attn.q_proj", xn).reshape(B, L, nq, hd)
    k = _lin(sd, p + "self_attn.k_proj", xn).reshape(B, L, nkv, hd)
    v = _lin(sd, p + "self_attn.v_proj", xn).reshape(B, L, nkv, hd)
    c, s = cos[:, :, None], sin[:, :, None]
    q, k = q * c + rotate_half(q) * s, k * c + rotate_half(k) * s
    if past_kv is None:
        o = attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), causal_mask(L, spans, x.device))
        o = o.transpose(1, 2).reshape(B, L, d)
        if spans is not None:
            keep = torch.zeros(B, L, 1, dtype=torch.bool)
            for b, (lo, hi) in enumerate(spans):
                keep[b, lo:hi] = True
            o = o.masked_fill(~keep.to(x.device), 0)
    else:
        assert L == 1
        rows = []
        for b in range(B):
            lo = 0 if past_lo is None else past_lo[b]
            kb = torch.cat([past_kv[0][b:b + 1, lo:], k[b:b + 1]], 1)
            vb = torch.cat([past_kv[1][b:b + 1, lo:], v[b:b + 1]], 1)
            rows.append(attention(q[b:b + 1].transpose(1, 2), kb.transpose(1, 2), vb.transpose(1, 2)))
        o = torch.cat(rows).transpose(1, 2).reshape(B, L, d)
    h = x + _lin(sd, p + "self_attn.o_proj", o)
    hn = rms_norm(h, sd[p + "post_attention_layernorm.weight"], tc.rms_norm_eps)
    a = F.silu(_lin(sd, p + "mlp.gate_proj", hn)) * _lin(sd, p + "mlp.up_proj", hn)
    h = h + _lin(sd, p + "mlp.down_proj", a)
    return {"h": h, "q": q, "k": k, "v": v, "attn": o, "a": a}


def final_norm(sd, x, tc):
    return rms_norm(x, sd["model.norm.weight"], tc.rms_norm_eps)


def lm_head(sd, x):
    return x @ sd["lm_head.weight"].transpose(0, 1)


def mlp2(pw, x):
    """MLP2 (`denoise_projector`): Linear · SiLU · Linear under the projector's names "0.weight", ..."""
    return _lin(pw, "2", F.silu(_lin(pw, "0", x)))


def embed_prompt(sd, ids, image_embeds=None, image_token_id=151655):
    """token embeddings [B, L, hidden] with the image embeddings put at the image-token positions, in order."""
    x = sd["model.embed_tokens.weight"][ids]
    if image_embeds is not None:
        x = x.clone()
        x[ids == image_token_id] = image_embeds.to(x.dtype)
    return x


def prefill(sd, tc, vc, ids, pos, pix=None, grid=None, spans=None):
    """The conditioning prefill: embed (with the vision tower's output scattered in), every decoder layer, final norm."""
    emb = vision_forward(sd, vc, pix, grid) if pix is not None else None
    x = embed_prompt(sd, ids, emb, tc.image_token_id)
    dt = x.dtype
    cos, sin = mrope(pos, tc.hidden_size // tc.num_attention_heads, tc.rope_theta, tc.mrope_section, dt)
    for i in range(tc.num_hidden_layers):
        x = decoder_layer(sd, i, x, cos.to(x.device), sin.to(x.device), tc, spans)["h"]
    return final_norm(sd, x, tc)


# ------------------------------------------------------------------------------------------------ weights
def state_dict_spec(tc, vc) -> dict[str, tuple]:
    s = {}
    H, I = vc.hidden_size, vc.intermediate_size
    s["visual.patch_embed.proj.weight"] = (H, vc.in_channels, vc.temporal_patch_size, vc.patch_size, vc.patch_size)
    for i in range(vc.depth):
        p = f"visual.blocks.{i}."
        s[p + "norm1.weight"] = s[p + "norm2.weight"] = (H,)
        s[p + "attn.qkv.weight"], s[p + "attn.qkv.bias"] = (3 * H, H), (3 * H,)
        s[p + "attn.proj.weight"], s[p + "attn.proj.bias"] = (H, H), (H,)
        for n in ("gate_proj", "up_proj"):
            s[p + f"mlp.{n}.weight"], s[p + f"mlp.{n}.bias"] = (I, H), (I,)
        s[p + "mlp.down_proj.weight"], s[p + "mlp.down_proj.bias"] = (H, I), (H,)
    mh = H * vc.spatial_merge_size ** 2
    s["visual.merger.ln_q.weight"] = (H,)
    s["visual.merger.mlp.0.weight"], s["visual.merger.mlp.0.bias"] = (mh, mh), (mh,)
    s["visual.merger.mlp.2.weight"], s["visual.merger.mlp.2.bias"] = (vc.out_hidden_size, mh), (vc.out_hidden_size,)
    d, It = tc.hidden_size, tc.intermediate_size
    hd = d // tc.num_attention_heads
    nkv = tc.num_key_value_heads * hd
    s["model.embed_tokens.weight"] = (tc.vocab_size, d)
    for i in range(tc.num_hidden_layers):
        p = f"model.layers.{i}."
        s[p + "input_layernorm.weight"] = s[p + "post_attention_layernorm.weight"] = (d,)
        for n, o in (("q_proj", d), ("k_proj", nkv), ("v_proj", nkv)):
            s[p + f"self_attn.{n}.weight"], s[p + f"self_attn.{n}.bias"] = (o, d), (o,)
        s[p + "self_attn.o_proj.weight"] = (d, d)
        s[p + "mlp.gate_proj.weight"] = s[p + "mlp.up_proj.weight"] = (It, d)
        s[p + "mlp.down_proj.weight"] = (d, It)
    s["model.norm.weight"] = (d,)
    s["lm_head.weight"] = (tc.vocab_size, d)
    return s


def make_synthetic_state_dict(text_cfg, vision_cfg, seed: int = 0, dtype=torch.float32, device="cpu"):
    """Random weights at fan_in^-1/2 (activations stay O(1) and every block's own share of the residual stream is a
    visible part of it), norm weights 1 + 0.1 N(0, 1), biases 0.1 N(0, 1), token embeddings N(0, 1).  Drawn on `device`
    in float32, one tensor at a time, then cast."""
    sd = {}
    g = torch.Generator(device=device).manual_seed(seed)
    for name, shape in state_dict_spec(text_cfg, vision_cfg).items():
        t = torch.randn(shape, generator=g, device=device)
        if name.endswith(".bias"):
            t.mul_(0.1)
        elif len(shape) == 1:
            t.mul_(0.1).add_(1.0)
        elif "embed_tokens" not in name:
            fan_in = 1
            for n in shape[1:]:
                fan_in *= n
            t.mul_(fan_in ** -0.5)
        sd[name] = t.to(dtype)
    return sd
