"""Synthetic LoRAs for the FLUX denoiser in the three accepted layouts, and the references the LoRA tests compare with.

  make_lora(cfg, ...)        {diffusers module: (A [r, in], B [out, r], alpha | None)} on every nn.Linear (or a subset)
  to_diffusers / to_bfl / to_kohya   the same adapter as a state dict in each layout (BFL / kohya fuse q/k/v(/mlp) into
                             one module of the summed rank with a block-structured B, and swap norm_out's halves)
  merged(sd, lora, s)        oracle state dict with W + s * alpha/r * B A            (fp64 reference)
  peft_linear(lora, s)       context manager: the oracle's linears become x W^T + b + s * alpha/r * (x A^T) B^T in the
                             oracle's dtype, each product rounded as PEFT does it (the bf16 yardstick)
"""
from __future__ import annotations

import contextlib

import torch

from oracle import flux_oracle as fo


def _fused_groups(cfg):
    """BFL modules that fuse several diffusers linears: BFL name -> [diffusers names in row order]."""
    g = {}
    for i in range(cfg.num_layers):
        p = f"transformer_blocks.{i}.attn."
        g[f"double_blocks.{i}.img_attn.qkv"] = [p + "to_q", p + "to_k", p + "to_v"]
        g[f"double_blocks.{i}.txt_attn.qkv"] = [p + "add_q_proj", p + "add_k_proj", p + "add_v_proj"]
    for i in range(cfg.num_single_layers):
        p = f"single_transformer_blocks.{i}."
        g[f"single_blocks.{i}.linear1"] = [p + "attn.to_q", p + "attn.to_k", p + "attn.to_v", p + "proj_mlp"]
    return g


def _bfl_of(cfg):
    """diffusers module -> BFL module for the one-to-one linears."""
    from gpt_image_edit_b200 import lora as L
    out = {}
    for b, part in L.bfl_parts(cfg).items():
        if b in _fused_groups(cfg):
            continue
        out[part.target] = b
    return out


def linear_shapes(cfg):
    """diffusers module -> (out, in) for every nn.Linear of FluxTransformer2DModel."""
    from gpt_image_edit_b200 import lora as L
    return {n: (p.rows, p.in_features) for n, p in L.diffusers_parts(cfg).items()}


def make_lora(cfg, rank=4, seed=0, modules=None, alpha=8.0, a_std=0.05, b_std=0.05, device="cpu"):
    """{module: (A, B, alpha)} fp32; alpha None leaves the scaling at 1.0."""
    g = torch.Generator().manual_seed(seed)
    shapes = linear_shapes(cfg)
    out = {}
    for n in (modules if modules is not None else shapes):
        o, k = shapes[n]
        A = (torch.randn(rank, k, generator=g) * a_std).bfloat16().float()
        B = (torch.randn(o, rank, generator=g) * b_std).bfloat16().float()
        out[n] = (A.to(device), B.to(device), alpha)
    return out


def to_diffusers(lora, prefix="transformer."):
    sd = {}
    for n, (A, B, alpha) in lora.items():
        sd[f"{prefix}{n}.lora_A.weight"] = A.bfloat16()
        sd[f"{prefix}{n}.lora_B.weight"] = B.bfloat16()
        if alpha is not None:
            sd[f"{prefix}{n}.alpha"] = torch.tensor(float(alpha))
    return sd


def _bfl_modules(cfg, lora):
    """[(BFL module, A, B, alpha)]: the fused groups concatenated (every part must carry the same rank and alpha)."""
    shapes = linear_shapes(cfg)
    out, used = [], set()
    for b, parts in _fused_groups(cfg).items():
        have = [p for p in parts if p in lora]
        if not have:
            continue
        rs = {lora[p][0].shape[0] for p in have}
        als = {lora[p][2] for p in have}
        assert len(rs) == 1 and len(als) == 1, "a fused BFL module needs one rank and alpha across its parts"
        r = rs.pop()
        alpha = als.pop()
        R = r * len(have)
        rows = sum(shapes[p][0] for p in parts)
        A = torch.cat([lora[p][0] for p in have])
        B = torch.zeros(rows, R, dtype=A.dtype, device=A.device)
        row, c = 0, 0
        for p in parts:
            o = shapes[p][0]
            if p in lora:
                B[row:row + o, c:c + r] = lora[p][1]
                c += r
            row += o
        # alpha / R over the fused rank must equal alpha_part / r
        out.append((b, A, B, None if alpha is None else alpha * len(have)))
        used.update(have)
    one = _bfl_of(cfg)
    for n, (A, B, alpha) in lora.items():
        if n in used:
            continue
        if n == "norm_out.linear":   # BFL chunks (shift, scale)
            h = B.shape[0] // 2
            B = torch.cat([B[h:], B[:h]])
        out.append((one[n], A, B, alpha))
    return out


def to_bfl(cfg, lora):
    sd = {}
    for b, A, B, alpha in _bfl_modules(cfg, lora):
        sd[f"diffusion_model.{b}.lora_A.weight"] = A.bfloat16()
        sd[f"diffusion_model.{b}.lora_B.weight"] = B.bfloat16()
        if alpha is not None:
            sd[f"diffusion_model.{b}.alpha"] = torch.tensor(float(alpha))
    return sd


def to_kohya(cfg, lora):
    sd = {}
    for b, A, B, alpha in _bfl_modules(cfg, lora):
        k = "lora_unet_" + b.replace(".", "_")
        sd[f"{k}.lora_down.weight"] = A.bfloat16()
        sd[f"{k}.lora_up.weight"] = B.bfloat16()
        if alpha is not None:
            sd[f"{k}.alpha"] = torch.tensor(float(alpha))
    return sd


def _scaling(A, alpha):
    return 1.0 if alpha is None else float(alpha) / A.shape[0]


def merged(sd, loras, dtype=torch.float64):
    """Oracle state dict (diffusers names) in `dtype` with every adapter merged: W + s * alpha/r * B A.
    loras: [(lora, s)]."""
    out = {k: v.to(dtype) for k, v in sd.items()}
    for lora, s in loras:
        for n, (A, B, alpha) in lora.items():
            w = out[n + ".weight"]
            out[n + ".weight"] = w + (s * _scaling(A, alpha)) * (B.to(w.device, dtype) @ A.to(w.device, dtype))
    return out


@contextlib.contextmanager
def peft_linear(loras):
    """The oracle's linears with unfused adapters as PEFT runs them: base = F.linear(x, W, b), then
    result + lora_B(lora_A(x)) * scaling for each adapter, in the activation dtype.  loras: [(lora, s)]."""
    orig = fo._lin

    def lin(sd, name, x):
        y = orig(sd, name, x)
        for lora, s in loras:
            if name in lora:
                A, B, alpha = lora[name]
                t = torch.nn.functional.linear(x, A.to(x.device, x.dtype))
                y = y + torch.nn.functional.linear(t, B.to(x.device, x.dtype)) * (s * _scaling(A, alpha))
        return y
    fo._lin = lin
    try:
        yield
    finally:
        fo._lin = orig
