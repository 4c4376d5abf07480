"""ORACLE — TEST INFRASTRUCTURE ONLY.  Never imported by the product (gpt_image_edit_b200/, univa/).

CPU/GPU PyTorch restatement of the arithmetic the reference reaches through diffusers==0.32.2
(`FluxTransformer2DModel`, requirements.txt:21), which is NOT vendored under /root/reference and
not installable here.  Every function names the reference call site it serves and the diffusers
symbol it restates (SURVEY.md Appendix A).  The op ORDER and the dtype of every intermediate follow
torch-eager execution of the diffusers modules, so running this file on bf16 tensors reproduces the
reference's bf16 rounding chain, and running it on fp32/fp64 tensors gives the exact-math answer.

PARITY UNPINNED by the reference: /root/reference holds no tests, golden vectors or fixtures for
this path (SURVEY.md §4, §8c).  The pins this repo adds instead:
  * oracle ≡ torchtitan.experiments.flux (an independent BFL-layout FLUX in site-packages) to
    fp32 round-off, with weights mapped by SURVEY.md A.7 — tests/test_oracle_cpu.py
    (test_oracle_matches_torchtitan_golden, test_live_crosscheck_against_torchtitan_if_available,
    test_oracle_guidance_embedder_matches_torchtitan_plus_guidance) over the fixtures tests/golden/make_golden.py writes
    (flux_toy_titan.pt, flux_toy_titan_guidance.pt);
  * the sampling loop built on it is bit-identical to the reference's own FluxKontextPipeline.__call__ executed from its
    file (oracle/pipeline_oracle.py, tests/golden/pipeline_ref_loop.pt);
  * scheduler/packing invariants quoted in SURVEY.md §8c.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this package.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import torch
import torch.nn.functional as F


@dataclass
class FluxConfig:
    """diffusers FluxTransformer2DModel config for FLUX.1-Kontext-dev (SURVEY.md Appendix A)."""

    in_channels: int = 64
    out_channels: int = 64
    num_layers: int = 19
    num_single_layers: int = 38
    attention_head_dim: int = 128
    num_attention_heads: int = 24
    joint_attention_dim: int = 4096
    pooled_projection_dim: int = 768
    guidance_embeds: bool = True
    axes_dims_rope: tuple = (16, 56, 56)
    theta: float = 10000.0
    mlp_ratio: int = 4

    @property
    def inner_dim(self) -> int:
        return self.attention_head_dim * self.num_attention_heads

    @staticmethod
    def toy(**kw) -> "FluxConfig":
        base = dict(num_layers=2, num_single_layers=2, attention_head_dim=128, num_attention_heads=2,
                    joint_attention_dim=256, pooled_projection_dim=64)
        base.update(kw)
        return FluxConfig(**base)


# ----------------------------------------------------------------------------- synthetic weights
def state_dict_spec(cfg: FluxConfig) -> dict[str, tuple]:
    """name -> shape, in diffusers state-dict naming (SURVEY.md A.6; reference train_denoiser.py:77-108)."""
    d, dh = cfg.inner_dim, cfg.attention_head_dim
    s: dict[str, tuple] = {}

    def lin(name, out_f, in_f):
        s[name + ".weight"] = (out_f, in_f)
        s[name + ".bias"] = (out_f,)

    lin("x_embedder", d, cfg.in_channels)
    lin("context_embedder", d, cfg.joint_attention_dim)
    for emb, in_f in (("timestep_embedder", 256), ("guidance_embedder", 256), ("text_embedder", cfg.pooled_projection_dim)):
        if emb == "guidance_embedder" and not cfg.guidance_embeds:
            continue
        lin(f"time_text_embed.{emb}.linear_1", d, in_f)
        lin(f"time_text_embed.{emb}.linear_2", d, d)
    for i in range(cfg.num_layers):
        p = f"transformer_blocks.{i}."
        lin(p + "norm1.linear", 6 * d, d)
        lin(p + "norm1_context.linear", 6 * d, d)
        for n in ("to_q", "to_k", "to_v", "add_q_proj", "add_k_proj", "add_v_proj", "to_out.0", "to_add_out"):
            lin(p + "attn." + n, d, d)
        for n in ("norm_q", "norm_k", "norm_added_q", "norm_added_k"):
            s[p + f"attn.{n}.weight"] = (dh,)
        lin(p + "ff.net.0.proj", cfg.mlp_ratio * d, d)
        lin(p + "ff.net.2", d, cfg.mlp_ratio * d)
        lin(p + "ff_context.net.0.proj", cfg.mlp_ratio * d, d)
        lin(p + "ff_context.net.2", d, cfg.mlp_ratio * d)
    for i in range(cfg.num_single_layers):
        p = f"single_transformer_blocks.{i}."
        lin(p + "norm.linear", 3 * d, d)
        for n in ("to_q", "to_k", "to_v"):
            lin(p + "attn." + n, d, d)
        for n in ("norm_q", "norm_k"):
            s[p + f"attn.{n}.weight"] = (dh,)
        lin(p + "proj_mlp", cfg.mlp_ratio * d, d)
        lin(p + "proj_out", d, d + cfg.mlp_ratio * d)
    lin("norm_out.linear", 2 * d, d)
    lin("proj_out", cfg.out_channels, d)
    return s


def make_synthetic_state_dict(cfg: FluxConfig, seed: int = 0, dtype=torch.float32, device="cpu",
                              std: float = 0.02, bias_std: float = 0.02, norm_jitter: float = 0.1):
    """Seeded random weights with the real architecture's shapes (no checkpoints exist offline).

    SURVEY.md §8d fixes N(0, 0.02^2) for weights; biases/norm weights are also randomised here so
    that a kernel which drops a bias or a norm weight cannot pass parity.
    Each tensor is drawn from its own generator seeded by (seed, index) so shapes can be generated
    independently of each other and on any device.
    """
    sd = {}
    for idx, (name, shape) in enumerate(state_dict_spec(cfg).items()):
        g = torch.Generator(device="cpu").manual_seed(seed * 1_000_003 + idx)
        if name.endswith("norm_q.weight") or name.endswith("norm_k.weight") or "norm_added" in name:
            t = 1.0 + norm_jitter * torch.randn(shape, generator=g)
        elif name.endswith(".bias"):
            t = bias_std * torch.randn(shape, generator=g)
        else:
            t = std * torch.randn(shape, generator=g)
        sd[name] = t.to(dtype=dtype, device=device)
    return sd


# ----------------------------------------------------------------------------- building blocks
def timestep_sinusoid(t: torch.Tensor, dim: int = 256, max_period: float = 10000.0) -> torch.Tensor:
    """diffusers `Timesteps(256, flip_sin_to_cos=True, downscale_freq_shift=0)` (A.3): [cos | sin]."""
    half = dim // 2
    exponent = -math.log(max_period) * torch.arange(0, half, dtype=torch.float32, device=t.device) / half
    emb = t[:, None].float() * torch.exp(exponent)[None, :]
    return torch.cat([torch.cos(emb), torch.sin(emb)], dim=-1)


def _lin(sd, name, x):
    return F.linear(x, sd[name + ".weight"], sd.get(name + ".bias"))


def time_text_embed(sd, cfg, timestep, guidance, pooled):
    """`CombinedTimestepGuidanceTextProjEmbeddings.forward` (A.3)."""
    p = "time_text_embed."
    t_proj = timestep_sinusoid(timestep).to(pooled.dtype)
    t_emb = _lin(sd, p + "timestep_embedder.linear_2", F.silu(_lin(sd, p + "timestep_embedder.linear_1", t_proj)))
    if cfg.guidance_embeds:
        g_proj = timestep_sinusoid(guidance).to(pooled.dtype)
        g_emb = _lin(sd, p + "guidance_embedder.linear_2", F.silu(_lin(sd, p + "guidance_embedder.linear_1", g_proj)))
        t_emb = t_emb + g_emb
    txt = _lin(sd, p + "text_embedder.linear_2", F.silu(_lin(sd, p + "text_embedder.linear_1", pooled)))
    return t_emb + txt


def rope_tables(ids: torch.Tensor, axes_dim=(16, 56, 56), theta: float = 10000.0):
    """`FluxPosEmbed.forward` (A.2): float64 angles, repeat_interleave(2), cast to fp32. -> cos, sin [S, sum(axes)]."""
    pos = ids.float()
    cos_out, sin_out = [], []
    for i, d in enumerate(axes_dim):
        freqs = 1.0 / (theta ** (torch.arange(0, d, 2, dtype=torch.float64, device=ids.device)[: d // 2] / d))
        ang = torch.outer(pos[:, i].to(torch.float64), freqs)
        cos_out.append(ang.cos().repeat_interleave(2, dim=1).float())
        sin_out.append(ang.sin().repeat_interleave(2, dim=1).float())
    return torch.cat(cos_out, dim=-1), torch.cat(sin_out, dim=-1)


def apply_rotary_emb(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor) -> torch.Tensor:
    """diffusers `apply_rotary_emb(use_real=True, use_real_unbind_dim=-1)`: interleaved pairs, fp32 math."""
    cos, sin = cos[None, None], sin[None, None]
    xr, xi = x.reshape(*x.shape[:-1], -1, 2).unbind(-1)
    x_rot = torch.stack([-xi, xr], dim=-1).flatten(3)
    ct = torch.promote_types(x.dtype, torch.float32)          # fp32 for 16-bit inputs, fp64 stays fp64
    return (x.to(ct) * cos + x_rot.to(ct) * sin).to(x.dtype)


def rms_norm(x: torch.Tensor, weight: torch.Tensor, eps: float = 1e-6) -> torch.Tensor:
    """diffusers `RMSNorm.forward`: fp32 variance, x*rsqrt in fp32, cast to weight dtype when that is 16-bit, * weight."""
    var = x.to(torch.float32 if x.dtype != torch.float64 else torch.float64).pow(2).mean(-1, keepdim=True)
    x = x * torch.rsqrt(var + eps)
    if weight.dtype in (torch.float16, torch.bfloat16):
        x = x.to(weight.dtype)
    return x * weight


def layer_norm(x: torch.Tensor, eps: float = 1e-6) -> torch.Tensor:
    return F.layer_norm(x, (x.shape[-1],), None, None, eps)


def attention(q, k, v, attn_mask=None):
    """`F.scaled_dot_product_attention(q, k, v, attn_mask, dropout_p=0, is_causal=False)`; q,k,v [B,H,S,dh]."""
    if q.dtype == torch.float64 or not q.is_cuda:
        # explicit math keeps the CPU oracle independent of SDPA backend selection
        if q.shape[1] > 1 and q.shape[1] * q.shape[2] * k.shape[2] * 4 > (2 << 30):
            # bound the score matrix to one head at a time (full-size CPU baseline runs)
            return torch.cat([attention(q[:, h:h + 1], k[:, h:h + 1], v[:, h:h + 1], attn_mask)
                              for h in range(q.shape[1])], dim=1)
        scale = 1.0 / math.sqrt(q.shape[-1])
        s = torch.matmul(q, k.transpose(-1, -2)) * scale
        if attn_mask is not None:
            s = s.masked_fill(~attn_mask, float("-inf")) if attn_mask.dtype == torch.bool else s + attn_mask
        return torch.matmul(torch.softmax(s.float() if s.dtype != torch.float64 else s, dim=-1).to(v.dtype), v)
    return F.scaled_dot_product_attention(q, k, v, attn_mask=attn_mask, dropout_p=0.0, is_causal=False)


def _heads(x, H):
    B, S, D = x.shape
    return x.view(B, S, H, D // H).transpose(1, 2)


def joint_attention(sd, prefix, cfg, x, c, cos, sin, attn_mask=None):
    """`FluxAttnProcessor2_0.__call__` (A.2). c=None for single-stream blocks."""
    H = cfg.num_attention_heads
    q = rms_norm(_heads(_lin(sd, prefix + "to_q", x), H), sd[prefix + "norm_q.weight"])
    k = rms_norm(_heads(_lin(sd, prefix + "to_k", x), H), sd[prefix + "norm_k.weight"])
    v = _heads(_lin(sd, prefix + "to_v", x), H)
    if c is not None:
        cq = rms_norm(_heads(_lin(sd, prefix + "add_q_proj", c), H), sd[prefix + "norm_added_q.weight"])
        ck = rms_norm(_heads(_lin(sd, prefix + "add_k_proj", c), H), sd[prefix + "norm_added_k.weight"])
        cv = _heads(_lin(sd, prefix + "add_v_proj", c), H)
        q, k, v = torch.cat([cq, q], 2), torch.cat([ck, k], 2), torch.cat([cv, v], 2)  # TEXT FIRST
    q, k = apply_rotary_emb(q, cos, sin), apply_rotary_emb(k, cos, sin)
    o = attention(q, k, v, attn_mask)
    B, _, S, dh = o.shape
    o = o.transpose(1, 2).reshape(B, S, H * dh).to(q.dtype)
    if c is None:
        return o, None
    Sc = c.shape[1]
    return _lin(sd, prefix + "to_out.0", o[:, Sc:]), _lin(sd, prefix + "to_add_out", o[:, :Sc])


def double_block(sd, i, cfg, x, c, temb, cos, sin, attn_mask=None):
    """`FluxTransformerBlock.forward` (A.1)."""
    p = f"transformer_blocks.{i}."
    e = _lin(sd, p + "norm1.linear", F.silu(temb))
    ec = _lin(sd, p + "norm1_context.linear", F.silu(temb))
    return double_block_mod(sd, i, cfg, x, c, e, ec, cos, sin, attn_mask)


def double_block_mod(sd, i, cfg, x, c, e, ec, cos, sin, attn_mask=None):
    """`double_block` after its two AdaLN linears: e / ec [B, 6d] are the image / text modulation rows
    (shift, scale, gate of the attention, then of the MLP)."""
    p = f"transformer_blocks.{i}."
    shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp = e.chunk(6, dim=1)
    xn = layer_norm(x) * (1 + scale_msa[:, None]) + shift_msa[:, None]
    c_shift_msa, c_scale_msa, c_gate_msa, c_shift_mlp, c_scale_mlp, c_gate_mlp = ec.chunk(6, dim=1)
    cn = layer_norm(c) * (1 + c_scale_msa[:, None]) + c_shift_msa[:, None]

    attn_x, attn_c = joint_attention(sd, p + "attn.", cfg, xn, cn, cos, sin, attn_mask)

    x = x + gate_msa.unsqueeze(1) * attn_x
    xn2 = layer_norm(x) * (1 + scale_mlp[:, None]) + shift_mlp[:, None]
    ff = _lin(sd, p + "ff.net.2", F.gelu(_lin(sd, p + "ff.net.0.proj", xn2), approximate="tanh"))
    x = x + gate_mlp.unsqueeze(1) * ff

    c = c + c_gate_msa.unsqueeze(1) * attn_c
    cn2 = layer_norm(c) * (1 + c_scale_mlp[:, None]) + c_shift_mlp[:, None]
    ffc = _lin(sd, p + "ff_context.net.2", F.gelu(_lin(sd, p + "ff_context.net.0.proj", cn2), approximate="tanh"))
    c = c + c_gate_mlp.unsqueeze(1) * ffc
    return c, x


def single_block(sd, i, cfg, h, temb, cos, sin, attn_mask=None):
    """`FluxSingleTransformerBlock.forward` (A.1)."""
    e = _lin(sd, f"single_transformer_blocks.{i}.norm.linear", F.silu(temb))
    return single_block_mod(sd, i, cfg, h, e, cos, sin, attn_mask)


def single_block_mod(sd, i, cfg, h, e, cos, sin, attn_mask=None):
    """`single_block` after its AdaLN linear: e [B, 3d] is the modulation row (shift, scale, gate)."""
    p = f"single_transformer_blocks.{i}."
    shift, scale, gate = e.chunk(3, dim=1)
    hn = layer_norm(h) * (1 + scale[:, None]) + shift[:, None]
    m = F.gelu(_lin(sd, p + "proj_mlp", hn), approximate="tanh")
    a, _ = joint_attention(sd, p + "attn.", cfg, hn, None, cos, sin, attn_mask)
    out = gate.unsqueeze(1) * _lin(sd, p + "proj_out", torch.cat([a, m], dim=2))
    return h + out


@dataclass
class Trace:
    """Optional per-stage capture for block-level parity tests."""
    enabled: bool = False
    t: dict = field(default_factory=dict)

    def put(self, k, v):
        if self.enabled:
            self.t[k] = v.detach().clone()


def flux_forward(sd, cfg: FluxConfig, hidden_states, encoder_hidden_states, pooled_projections, timestep,
                 img_ids, txt_ids, guidance=None, attention_mask=None, trace: Trace | None = None):
    """`FluxTransformer2DModel.forward(...)[0]` (A.1).  Call sites in the reference:
    univa/utils/flux_pipeline.py:1067-1077, univa/models/modeling_univa_denoise_tower.py:103-110.
    `timestep`/`guidance` arrive already divided by 1000 (pipeline :1069) / raw (guidance), as in the reference.
    """
    tr = trace or Trace()
    x = _lin(sd, "x_embedder", hidden_states)
    t = timestep.to(x.dtype) * 1000
    g = guidance.to(x.dtype) * 1000 if guidance is not None else None
    temb = time_text_embed(sd, cfg, t, g, pooled_projections)
    tr.put("temb", temb)
    c = _lin(sd, "context_embedder", encoder_hidden_states)
    if txt_ids.ndim == 3:
        txt_ids = txt_ids[0]
    if img_ids.ndim == 3:
        img_ids = img_ids[0]
    ids = torch.cat((txt_ids, img_ids), dim=0)
    cos, sin = rope_tables(ids, cfg.axes_dims_rope, cfg.theta)
    tr.put("x0", x)
    tr.put("c0", c)
    for i in range(cfg.num_layers):
        c, x = double_block(sd, i, cfg, x, c, temb, cos, sin, attention_mask)
        tr.put(f"double{i}.x", x)
        tr.put(f"double{i}.c", c)
    h = torch.cat([c, x], dim=1)
    for i in range(cfg.num_single_layers):
        h = single_block(sd, i, cfg, h, temb, cos, sin, attention_mask)
        tr.put(f"single{i}.h", h)
    x = h[:, c.shape[1]:]
    e = _lin(sd, "norm_out.linear", F.silu(temb).to(x.dtype))
    scale, shift = torch.chunk(e, 2, dim=1)  # SCALE FIRST (AdaLayerNormContinuous)
    x = layer_norm(x) * (1 + scale)[:, None, :] + shift[:, None, :]
    return _lin(sd, "proj_out", x)
