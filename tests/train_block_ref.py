"""Float64 references of the FLUX training backward one stage at a time, and the per-slice gate that compares a stage's
gradients with them.

The engine's backward (`b2f_flux_train_backward`, csrc/flux_train.cu) runs in stages: the tail (norm_out + proj_out),
each transformer block from the last to the first, and the head (the gradient w.r.t. encoder_hidden_states); MLP2
follows in `FluxTrainGraph.backward`.  Each function here is the oracle's restatement of one stage, differentiated by
torch.autograd in the dtype it is given: float64 for the reference, bfloat16 for the yardstick (what torch-bf16
autograd of the same stage makes of the same inputs).  The stage inputs are leaves: the block input h, the incoming
residual-stream gradient, and the modulation rows `mod` exactly as the AdaLN GEMM produced them.  An error therefore
stays inside the stage that made it.

Gradients come back under diffusers names (`transformer_blocks.1.attn.to_q.weight`, ...), so
`test_train_flux_gpu._ref_for` maps them onto the engine's fused parameters.  The AdaLN linears get theirs from the
modulation gradient: weight = dmod^T . silu(temb), bias = sum_b dmod, rows in chunk order.

The gate (`gate`) measures, for slice s of a gradient, e_s = |K_s - R_s| / rms_s |R_s| (K the engine, R the reference)
and y_s the same for the yardstick, and requires max_s e_s <= 2 max_s y_s + beta.  Normalising by the rms over slices
keeps one slice's error visible at any tensor size, where one rel-L2 number over the tensor shrinks as 1/sqrt(slices).
"""
from __future__ import annotations

from dataclasses import dataclass

import torch
import torch.nn.functional as F

from oracle import flux_oracle as fo

BETA = 1e-2          # additive allowance of the per-slice gate
TENSOR_SLACK = 1e-2  # additive allowance of the per-tensor rule

CHUNKS = {
    "double": ("shift_msa", "scale_msa", "gate_msa", "shift_mlp", "scale_mlp", "gate_mlp"),
    "single": ("shift", "scale", "gate"),
    "norm_out": ("scale", "shift"),
}


def _leaf(t, dtype, grad=False):
    return t.detach().to(dtype).clone().requires_grad_(grad)


def mod_offsets(cfg: fo.FluxConfig):
    """column offset of each block's modulation rows in `mod` (b2f_flux_modulation): per double block 6d image then 6d
    text, per single block 3d, then norm_out's 2d."""
    d, nd = cfg.inner_dim, cfg.num_layers
    dbl = [i * 12 * d for i in range(nd)]
    sgl = [nd * 12 * d + i * 3 * d for i in range(cfg.num_single_layers)]
    return dbl, sgl, nd * 12 * d + cfg.num_single_layers * 3 * d


def adaln_grads(dmod, silu_temb):
    """(weight, bias) gradients of an AdaLN linear mod = silu_temb W^T + b from dmod [B, n*d]."""
    return dmod.transpose(0, 1) @ silu_temb.to(dmod.dtype), dmod.sum(0)


TRAINED_DOUBLE = ("attn.to_q", "attn.to_k", "attn.to_v", "attn.to_out.0")
TRAINED_SINGLE = ("attn.to_q", "attn.to_k", "attn.to_v")


def _weights(sd, prefix, dtype, trained):
    keys = {prefix + t + s for t in trained for s in (".weight", ".bias")}
    keys |= {prefix + "attn.norm_q.weight", prefix + "attn.norm_k.weight"}
    return {k: _leaf(v, dtype, k in keys) for k, v in sd.items() if k.startswith(prefix)}, sorted(keys)


def double_stage(sd, cfg, blk, h_in, dh_out, mod, silu_temb, cos, sin, S_txt, dtype):
    """One double block's backward: {"dh": d h_in, diffusers name: gradient, ..., "dmod": d e}."""
    d = cfg.inner_dim
    p = f"transformer_blocks.{blk}."
    w, keys = _weights(sd, p, dtype, TRAINED_DOUBLE)
    o = mod_offsets(cfg)[0][blk]
    h = _leaf(h_in, dtype, True)
    e = _leaf(mod[:, o:o + 6 * d], dtype, True)
    ec = _leaf(mod[:, o + 6 * d:o + 12 * d], dtype)
    c_out, x_out = fo.double_block_mod(w, blk, cfg, h[:, S_txt:], h[:, :S_txt], e, ec, cos, sin)
    out = torch.cat([c_out, x_out], 1)
    gs = torch.autograd.grad(out, [h, e] + [w[k] for k in keys], dh_out.to(dtype))
    res = {"dh": gs[0], "dmod": gs[1]}
    res.update(zip(keys, gs[2:]))
    res[p + "norm1.linear.weight"], res[p + "norm1.linear.bias"] = adaln_grads(gs[1], silu_temb)
    return res


def single_stage(sd, cfg, si, h_in, dh_out, mod, silu_temb, cos, sin, dtype):
    d = cfg.inner_dim
    p = f"single_transformer_blocks.{si}."
    w, keys = _weights(sd, p, dtype, TRAINED_SINGLE)
    o = mod_offsets(cfg)[1][si]
    h = _leaf(h_in, dtype, True)
    e = _leaf(mod[:, o:o + 3 * d], dtype, True)
    out = fo.single_block_mod(w, si, cfg, h, e, cos, sin)
    gs = torch.autograd.grad(out, [h, e] + [w[k] for k in keys], dh_out.to(dtype))
    res = {"dh": gs[0], "dmod": gs[1]}
    res.update(zip(keys, gs[2:]))
    res[p + "norm.linear.weight"], res[p + "norm.linear.bias"] = adaln_grads(gs[1], silu_temb)
    return res


def tail_stage(sd, cfg, h_fin, dout, mod, S_txt, n_out, dtype):
    """norm_out (scale first) + proj_out on the first n_out image rows: {"dh": [B, S, d], "dmod": d [scale | shift]}."""
    d = cfg.inner_dim
    o = mod_offsets(cfg)[2]
    x = _leaf(h_fin[:, S_txt:S_txt + n_out], dtype, True)
    e = _leaf(mod[:, o:o + 2 * d], dtype, True)
    scale, shift = e.chunk(2, dim=1)
    xn = fo.layer_norm(x) * (1 + scale)[:, None, :] + shift[:, None, :]
    out = F.linear(xn, sd["proj_out.weight"].to(dtype), sd["proj_out.bias"].to(dtype))
    gx, ge = torch.autograd.grad(out, [x, e], dout.to(dtype))
    dh = torch.zeros(h_fin.shape, dtype=dtype, device=h_fin.device)
    dh[:, S_txt:S_txt + n_out] = gx
    return {"dh": dh, "dmod": ge}


def head_stage(sd, dh, S_txt, dtype):
    """d encoder_hidden_states = dh[:, :S_txt] . context_embedder.weight"""
    return dh[:, :S_txt].to(dtype) @ sd["context_embedder.weight"].to(dtype)


def mlp2_stage(pw, x, d_vlm, dtype):
    """MLP2 enc = silu(x W0^T + b0) W2^T + b2: gradients under the projector's names ("0.weight", ...)."""
    w = {k: _leaf(v, dtype, True) for k, v in pw.items()}
    enc = F.linear(F.silu(F.linear(x.to(dtype), w["0.weight"], w["0.bias"])), w["2.weight"], w["2.bias"])
    return dict(zip(w, torch.autograd.grad(enc, list(w.values()), d_vlm.to(dtype))))


# ------------------------------------------------------------------------------------------------ gates
def rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def _view(t, kind, n_chunks=None):
    t = t.double()
    if kind == "rows":
        return t.reshape(-1, t.shape[-1])
    if kind == "cols":
        return t.reshape(-1, t.shape[-1]).transpose(0, 1)
    if kind == "chunks":
        return t.reshape(n_chunks, -1)
    if kind == "elems":
        return t.reshape(-1, 1)
    raise ValueError(kind)


def slice_errors(K, R, kind, n_chunks=None):
    """e_s = |K_s - R_s| / rms_s |R_s| over the slices of `kind`."""
    k, r = _view(K, kind, n_chunks), _view(R, kind, n_chunks)
    den = r.pow(2).sum(1).mean().sqrt().clamp_min(1e-300)
    return (k - r).norm(dim=1) / den


@dataclass
class Check:
    stage: str
    tensor: str
    kind: str          # "tensor" (rel-L2 rule) or the slice kind
    e: float           # engine: rel-L2, or max_s e_s
    y: float           # yardstick: rel-L2, or max_s y_s
    ok: bool
    where: str = ""    # the worst slice

    def __str__(self):
        ratio = self.e / self.y if self.y > 0 else (0.0 if self.e == 0 else float("inf"))
        return (f"{'ok  ' if self.ok else 'FAIL'} {self.stage:>8s} {self.tensor:44s} {self.kind:6s} e {self.e:.3e} "
                f"y {self.y:.3e} e/y {ratio:6.2f}  {self.where}")


def gate(stage, tensor, K, R, Y, kinds, label=None, n_chunks=None, beta=BETA):
    """The per-tensor rule and the per-slice gate of every kind in `kinds`.  label(kind, i) names slice i."""
    label = label or (lambda kind, i: f"{kind[:-1]} {i}")
    ek, et = rel(K, R), rel(Y, R)
    finite = bool(torch.isfinite(K).all())
    out = [Check(stage, tensor, "tensor", ek, et, finite and ek <= 2 * et + TENSOR_SLACK, "" if finite else "non-finite")]
    for kind in kinds:
        e, y = slice_errors(K, R, kind, n_chunks), slice_errors(Y, R, kind, n_chunks)
        e = torch.nan_to_num(e, nan=float("inf"))
        i = int(e.argmax())
        em, ym = e.max().item(), y.max().item()
        out.append(Check(stage, tensor, kind, em, ym, em <= 2 * ym + beta, label(kind, i)))
    return out


def token_label(B, S, S_txt):
    """labels of [B, S, d] rows (text rows first)."""
    def f(kind, i):
        if kind != "rows":
            return f"{kind[:-1]} {i}"
        b, s = divmod(i, S)
        return f"batch {b} text token {s}" if s < S_txt else f"batch {b} image token {s - S_txt}"
    return f


def dh_gates(stage, dh, R, Y, dh_out, B, S_txt):
    """gates of a stage's dh [B, S, d], text and image rows apart; with dh_out (the gradient the stage received) also
    of the stage's own share dh - dh_out, which the residual path's identity term would otherwise swamp."""
    S = dh.shape[1]
    out = []
    for part, sl, lab in (("text", slice(None, S_txt), token_label(B, S_txt, S_txt)),
                          ("image", slice(S_txt, None), token_label(B, S - S_txt, 0))):
        out += gate(stage, f"dh {part}", dh[:, sl], R[:, sl], Y[:, sl], ("rows",), lab)
        if dh_out is not None:
            o = dh_out[:, sl].double()
            out += gate(stage, f"dh - dh_out {part}", dh[:, sl].double() - o, R[:, sl].double() - o, Y[:, sl].double() - o,
                        ("rows",), lab)
    return out


def qkv_label(d, head_dim):
    def f(kind, i):
        if kind == "rows":
            return f"row {i} ({'qkv'[i // d]} head {(i % d) // head_dim})"
        return f"{kind[:-1]} {i}"
    return f


def chunk_label(names):
    return lambda kind, i: f"chunk {names[i]}" if kind == "chunks" else f"{kind[:-1]} {i}"
