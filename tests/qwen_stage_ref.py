"""Float64 references of the Qwen2.5-VL conditioning path one stage at a time, and the gates that compare a stage's
tensors with them.

`B200Qwen2p5VL` (gpt_image_edit_b200/qwen2p5vl.py) runs in stages a test can drive one at a time: `_vision_embed`
(patch embed, RoPE tables, window gather), `_vision_block(i)`, `_vision_merge`, `_decoder_layer(i)` (prefill or one
decode step) and the final norm; MLP2 and `lm_head` follow.  Each function here is the oracle's composition of one stage
(oracle/qwen_oracle.py), run in the dtype it is given: float64 for the reference, bfloat16 for the yardstick (what torch
in bf16 makes of the same inputs, attention through F.scaled_dot_product_attention on a GPU).  The stage inputs are the
engine's bf16 tensors, so an error stays inside the stage that made it.  The oracle computes its own window order,
segment boundaries and RoPE tables from the image grids and position ids, so the engine's are checked, not reused.

The engine lays the ViT's heads out in 128-wide slots (80 real columns) and its MLP 3424 wide (3420 real): `vit_qkv`,
`vit_heads` and `vit_mlp` strip those slots before gating, and `vit_padding` returns them for an exact zero check.

The gates are train_block_ref's per-tensor rule and per-slice gate at `infer_block_ref.BETA`, over token rows (text,
image and padding rows apart in the decoder), channels, heads (the 80 real columns of a ViT head; each of the decoder's
q, k and v heads) and, in the ViT, attention windows (rows grouped by cu_seqlens, `segment_gate`).
"""
from __future__ import annotations

import torch

import infer_block_ref as IB
import train_block_ref as TB
from oracle import qwen_oracle as qo

HP = 128  # the engine's head slot


# ------------------------------------------------------------------------------------------------ engine layout
def vit_qkv(qkv, nh, hd=80):
    """engine ViT qkv [T, 3*nh*128] -> [T, 3*nh*hd] (real columns, q heads then k then v)"""
    return qkv.view(qkv.shape[0], 3 * nh, HP)[..., :hd].reshape(qkv.shape[0], -1)


def vit_heads(t, nh, hd=80):
    return t.view(t.shape[0], nh, HP)[..., :hd].reshape(t.shape[0], -1)


def vit_mlp(a, inter):
    return a[:, :inter]


def vit_padding(keep, nh, inter, hd=80):
    """the padding slots of a ViT block's buffers: {name: tensor} that must all be exactly zero"""
    T = keep["qkv"].shape[0]
    return {"qkv[:, 80:128]": keep["qkv"].view(T, 3 * nh, HP)[..., hd:], "attn_out[:, 80:128]":
            keep["attn_out"].view(T, nh, HP)[..., hd:], "a[:, 3420:]": keep["a"][:, inter:]}


# ------------------------------------------------------------------------------------------------ stages
def vit_context(vc, grid):
    """the oracle's window order and segments of an image batch: (window_index, cu_win, cu_full, patch permutation)"""
    m = vc.spatial_merge_size
    widx, cu_win = qo.window_index(grid, vc.window_size, m, vc.patch_size)
    perm = (widx[:, None] * m * m + torch.arange(m * m)).reshape(-1)
    return widx, cu_win, qo.full_cu_seqlens(grid), perm


def vit_embed_stage(sd, vc, pix, grid, dtype):
    """patch embed, rows gathered into window order: [T, hidden]"""
    x = qo.patch_embed(IB._sub(sd, "visual.patch_embed.", dtype), pix.to(dtype))
    return x[vit_context(vc, grid)[3].to(x.device)]


def vit_block_stage(sd, vc, i, x_in, grid, dtype):
    """ViT block i on the engine's block input (window order) -> {"h", "qkv" [T, 3*nh*80], "attn", "a"}"""
    _, cu_win, cu_full, perm = vit_context(vc, grid)
    cos, sin = qo.vision_rope(grid, vc.hidden_size // vc.num_heads, vc.spatial_merge_size, dtype=dtype)
    dev = x_in.device
    cu = cu_full if i in vc.fullatt_block_indexes else cu_win
    out = qo.vision_block(IB._sub(sd, f"visual.blocks.{i}.", dtype), i, x_in.to(dtype), cos[perm].to(dev),
                          sin[perm].to(dev), cu, vc)
    out["qkv"] = out["qkv"].reshape(x_in.shape[0], -1)
    return out


def vit_merge_stage(sd, vc, x_in, grid, dtype):
    """merger on the last block's output: {"merged" (window order), "out" (processor order)}"""
    widx = vit_context(vc, grid)[0]
    merged = qo.merger(IB._sub(sd, "visual.merger.", dtype), x_in.to(dtype), vc.spatial_merge_size)
    return {"merged": merged, "out": merged[torch.argsort(widx).to(merged.device)]}


def rope_tables(tc, pos, dtype, device):
    cos, sin = qo.mrope(pos.cpu(), tc.hidden_size // tc.num_attention_heads, tc.rope_theta, tc.mrope_section, dtype)
    return cos.to(device), sin.to(device)


def decoder_stage(sd, tc, i, x_in, pos, dtype, spans=None, past_kv=None, past_lo=None):
    """decoder layer i on the engine's layer input x_in [B, L, hidden], positions pos [3, B, L]
    -> {"h", "qkv" [B, L, (q + 2 kv heads) * hd] in the engine's column order, "attn", "a", "k", "v"}"""
    cos, sin = rope_tables(tc, pos, dtype, x_in.device)
    kv = None if past_kv is None else (past_kv[0].to(dtype), past_kv[1].to(dtype))
    out = qo.decoder_layer(IB._sub(sd, f"model.layers.{i}.", dtype), i, x_in.to(dtype), cos, sin, tc, spans, kv, past_lo)
    B, L = x_in.shape[:2]
    out["qkv"] = torch.cat([out["q"].reshape(B, L, -1), out["k"].reshape(B, L, -1), out["v"].reshape(B, L, -1)], -1)
    return out


def norm_stage(sd, tc, x_in, dtype):
    return qo.final_norm(IB._sub(sd, "model.norm.", dtype), x_in.to(dtype), tc)


def mlp2_stage(pw, x_in, dtype):
    return qo.mlp2({k: v.to(dtype) for k, v in pw.items()}, x_in.to(dtype))


def lm_head_stage(sd, x_in, dtype, chunk=16384):
    """logits [n, vocab], the vocab in chunks of `chunk` rows so a float64 copy of the whole lm_head is never made"""
    w = sd["lm_head.weight"]
    x = x_in.to(dtype)
    return torch.cat([x @ w[j:j + chunk].to(dtype).transpose(0, 1) for j in range(0, w.shape[0], chunk)], -1)


# ------------------------------------------------------------------------------------------------ gates
def segment_gate(stage, tensor, K, R, Y, cu, what="window"):
    """the per-slice gate over row segments cu[s]:cu[s+1] of unequal length: e_s = rms(K_s - R_s) / rms(R), which for
    equal segments is train_block_ref's |K_s - R_s| / rms_s |R_s|."""
    k, r, y = (t.double().reshape(t.shape[0], -1) for t in (K, R, Y))
    den = r.pow(2).mean().sqrt().clamp_min(1e-300)

    def errs(a):
        return torch.stack([(a[cu[s]:cu[s + 1]] - r[cu[s]:cu[s + 1]]).pow(2).mean().sqrt() for s in range(len(cu) - 1)]) / den

    e = torch.nan_to_num(errs(k), nan=float("inf"))
    i = int(e.argmax())
    em, ym = e.max().item(), errs(y).max().item()
    return TB.Check(stage, tensor, "segs", em, ym, em <= 2 * ym + IB.BETA, f"{what} {i} (rows {cu[i]}:{cu[i + 1]})")


def _by_head(t, hd):
    t = t.double()
    n = t.shape[-1] // hd
    return t.reshape(-1, n, hd).transpose(0, 1).reshape(n, -1)


def head_gates(stage, name, K, R, Y, hd, label):
    return [c for c in TB.gate(stage, f"{name} heads", _by_head(K, hd), _by_head(R, hd), _by_head(Y, hd), ("rows",), label,
                               beta=IB.BETA) if c.kind != "tensor"]


def _row_label(kind, i):
    return f"token {i}" if kind == "rows" else f"{kind[:-1]} {i}"


def vit_gates(stage, name, K, R, Y, cu, heads=None, base=None):
    """gates of a ViT activation [T, n] (window order): token rows, channels, one slice per window of `cu`, and with
    heads = (count, head_dim) one per head.  With `base` (the block input) again on the block's own share K - base."""
    out = []
    sets = [(name, K, R, Y)]
    if base is not None:
        b = base.double()
        sets.append((f"{name} - {name}_in", K.double() - b, R.double() - b, Y.double() - b))
    for tag, k, r, y in sets:
        out += TB.gate(stage, tag, k, r, y, ("rows", "cols"), _row_label, beta=IB.BETA)
        out.append(segment_gate(stage, tag, k, r, y, cu))
    if heads is not None:
        n, hd = heads
        lab = (lambda kind, i: f"{'qkv'[i // (n // 3)]} head {i % (n // 3)}") if name == "qkv" else (lambda kind, i: f"head {i}")
        out += head_gates(stage, name, K, R, Y, hd, lab)
    return out


def dec_gates(stage, name, K, R, Y, parts, heads=None, base=None):
    """gates of a decoder activation [B, L, n]: token rows and channels of each row set in `parts` ({name: boolean mask
    [B, L]}: text, image, padding) apart, and with heads = (labels, head_dim) one slice per head.  With `base` (the layer
    input) the same again on the layer's own share K - base."""
    L = K.shape[1]
    lab = lambda idx: (lambda kind, i: f"batch {int(idx[i]) // L} token {int(idx[i]) % L}" if kind == "rows"
                       else f"{kind[:-1]} {i}")
    flat = lambda t: t.double().reshape(-1, t.shape[-1])
    sets = [(name, flat(K), flat(R), flat(Y))]
    if base is not None:
        b = flat(base)
        sets.append((f"{name} - {name}_in", sets[0][1] - b, sets[0][2] - b, sets[0][3] - b))
    out = []
    for tag, k, r, y in sets:
        for part, m in parts.items():
            idx = m.reshape(-1).nonzero().squeeze(1)
            if idx.numel():
                dev = k.device
                out += TB.gate(stage, f"{tag} {part}", k[idx.to(dev)], r[idx.to(dev)], y[idx.to(dev)], ("rows", "cols"),
                               lab(idx), beta=IB.BETA)
    if heads is not None:
        labels, hd = heads
        out += head_gates(stage, name, flat(K), flat(R), flat(Y), hd, lambda kind, i: labels[i])
    return out


def qkv_head_labels(nq, nkv):
    return [f"q head {h}" for h in range(nq)] + [f"k head {h}" for h in range(nkv)] + [f"v head {h}" for h in range(nkv)]


def logits_gates(stage, K, R, Y, label):
    """gates of logits [rows, vocab]: one slice per row ((step, sequence) in decode) and per vocab column"""
    return TB.gate(stage, "logits", K, R, Y, ("rows", "cols"), label, beta=IB.BETA)
