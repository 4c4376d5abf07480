"""Drop-in for the object the reference passes as `transformer=` to FluxKontextPipeline
(`model.denoise_tower.denoiser`, a diffusers `FluxTransformer2DModel`; reference
univa/serve/cli.py:64-68, univa/models/modeling_univa_denoise_tower.py:21) — same call signature,
config attributes and state-dict key names, but the forward is a single C-ABI call into libb2f
(`b2f_flux_forward`, hand-written sm_90a kernels).  Nothing here computes the model in torch.

Storage: projections that the engine runs as one GEMM (q/k/v, the single block's q/k/v/proj_mlp,
every AdaLN linear) are STORED row-concatenated; `state_dict()` / `load_state_dict()` expose and
accept the diffusers names (SURVEY.md A.6) as views, so checkpoints interchange.
"""
from __future__ import annotations

import ctypes as C
import math
from collections import OrderedDict
from dataclasses import dataclass
from types import SimpleNamespace

import torch

from . import _lib, flux_layout
from ._lib import check, ptr, stream_ptr
from .lora import FluxLoraMixin


class FluxTransformerConfig(SimpleNamespace):
    """Attribute names follow diffusers FluxTransformer2DModel.config (the pipeline reads
    `.in_channels` and `.guidance_embeds`: reference flux_pipeline.py:975, :1011)."""

    def __init__(self, **kw):
        base = dict(patch_size=1, in_channels=64, out_channels=64, num_layers=19, num_single_layers=38,
                    attention_head_dim=128, num_attention_heads=24, joint_attention_dim=4096,
                    pooled_projection_dim=768, guidance_embeds=True, axes_dims_rope=(16, 56, 56))
        base.update(kw)
        super().__init__(**base)

    def get(self, k, default=None):
        return getattr(self, k, default)


class Transformer2DModelOutput(SimpleNamespace):
    pass


@dataclass(frozen=True)
class FirstBlockCacheConfig:
    """First-block cache (`B200FluxTransformer2DModel.enable_cache`; the shape of diffusers' later
    `FirstBlockCacheConfig`): a forward whose block-0 residual moved by less than `threshold` (relative L1 distance to the
    last step that ran in full, pooled over the batch) skips the other blocks and reuses their residual from that step.
    0 never skips; +inf skips every step after the first of a run."""
    threshold: float

    def __post_init__(self):
        t = float(self.threshold)
        if math.isnan(t) or t < 0:
            raise ValueError(f"FirstBlockCacheConfig: threshold must be >= 0 (got {self.threshold})")


class _CacheState:
    """One branch's b2f_flux_cache over device memory owned here."""

    def __init__(self):
        self.mem = None
        self.h = None
        self.key = None
        self.calls = 0

    def ensure(self, nbytes: int, device):
        if self.mem is not None and self.mem.numel() >= nbytes:
            return
        self.close()
        self.mem = torch.empty(nbytes, dtype=torch.uint8, device=device)
        h = C.c_void_p()
        check(_lib.lib.b2f_flux_cache_create(C.byref(h), ptr(self.mem), nbytes), "b2f_flux_cache_create")
        self.h = h

    def reset(self):
        if self.h:
            check(_lib.lib.b2f_flux_cache_reset(self.h), "b2f_flux_cache_reset")
        self.key = None
        self.calls = 0

    def close(self):
        if self.h and _lib is not None and getattr(_lib, "lib", None) is not None:
            _lib.lib.b2f_flux_cache_destroy(self.h)
        self.h = None
        self.mem = None


def _storage(cfg: FluxTransformerConfig):
    """Every stored linear as (bound name, out, in, views) in allocation order, which is the order randomize_ draws
    them in; views: (diffusers name, row0, rows).  The fused block linears, the fused AdaLN weight, the embedders and
    proj_out, the other block linears."""
    lay = flux_layout.layout(cfg)
    adaln = [t for t in lay if t.kind == "adaln"]
    row0 = [sum(t.out for t in adaln[:j]) for j in range(len(adaln))]
    # the embedders are allocated with guidance before text, proj_out last
    emb = sorted((t for t in lay if t.kind == "embedder"),
                 key=lambda t: (".text_embedder." in t.name) + 2 * (t.name == "proj_out"))
    return ([(t.name, t.out, t.inp, t.parts) for t in lay if len(t.parts) > 1]
            + [("adaln", sum(t.out for t in adaln), adaln[0].inp, tuple((t.name, r, t.out) for t, r in zip(adaln, row0)))]
            + [(t.name, t.out, t.inp, t.parts) for t in emb]
            + [(t.name, t.out, t.inp, t.parts) for t in lay if t.kind == "block" and len(t.parts) == 1])


def text_windows(mask: torch.Tensor, B: int, S_txt: int) -> torch.Tensor:
    """The per-item text windows of an encoder attention mask: [B, S_txt], each row one contiguous run of nonzeros
    covering at least one token (left padding, as the Qwen processor pads, or right padding) -> int32 [B, 2] (lo, hi)
    on the host.  Rows with holes, empty rows and shapes other than [B, S_txt] are refused."""
    from .qwen2p5vl import padding_spans

    if mask.dim() != 2 or tuple(mask.shape) != (B, S_txt):
        raise _lib.B2FError(f"encoder_attention_mask: expected [{B}, {S_txt}], got {tuple(mask.shape)}")
    return torch.tensor(padding_spans(mask), dtype=torch.int32)


class B200FluxTransformer2DModel(FluxLoraMixin, torch.nn.Module):
    def __init__(self, config: FluxTransformerConfig | None = None, device="cuda", **kw):
        super().__init__()
        self.config = config or FluxTransformerConfig(**kw)
        cfg = self.config
        dev = torch.device(device)
        if dev.type != "cuda":
            raise _lib.B2FError("B200FluxTransformer2DModel lives on a CUDA device; there is no CPU path")
        self.inner_dim = cfg.num_attention_heads * cfg.attention_head_dim
        self._store: "OrderedDict[str, torch.Tensor]" = OrderedDict()   # bound name -> storage tensor
        self._views: "OrderedDict[str, torch.Tensor]" = OrderedDict()   # diffusers name -> view
        mk = lambda *shape: torch.zeros(shape, device=dev, dtype=torch.bfloat16)
        for name, o, i, views in _storage(cfg):
            w, b = mk(o, i), mk(o)
            self._store[name + ".weight"], self._store[name + ".bias"] = w, b
            for v, r, n in views:
                self._views[v + ".weight"], self._views[v + ".bias"] = (w, b) if len(views) == 1 else (w[r:r + n],
                                                                                                    b[r:r + n])
        for name in flux_layout.norm_weights(cfg):
            w = torch.ones(cfg.attention_head_dim, device=dev, dtype=torch.bfloat16)
            self._store[name] = w
            self._views[name] = w
        for k, t in self._store.items():   # registered so .parameters()/.to() bookkeeping sees them
            self.register_buffer("w__" + k.replace(".", "__"), t, persistent=False)

        ccfg = _lib.FluxCfg(cfg.num_attention_heads, cfg.attention_head_dim, cfg.num_layers, cfg.num_single_layers,
                            cfg.in_channels, cfg.out_channels, cfg.joint_attention_dim, cfg.pooled_projection_dim,
                            int(bool(cfg.guidance_embeds)), 4)
        h = C.c_void_p()
        check(_lib.lib.b2f_flux_create(C.byref(h), C.byref(ccfg)), "b2f_flux_create")
        self._h = h
        for k, t in self._store.items():
            check(_lib.lib.b2f_flux_bind_weight(self._h, k.encode(), ptr(t), t.numel()), f"bind {k}")
        check(_lib.lib.b2f_flux_finalize(self._h), "b2f_flux_finalize")
        self.mod_width = int(_lib.lib.b2f_flux_mod_width(self._h))
        self._ws = {}
        self._rope = None
        self._schedule = None
        self.gradient_checkpointing = False
        self._fp8 = None   # bound name -> (e4m3 weight, fp32 scales) while FP8 is enabled
        self._fp8_unfused = False   # FP8 linears accept unfused LoRA adapters (b2f_flux_set_fp8 mode 2)
        self._fp8_attn = False
        self._cache_cfg = None      # FirstBlockCacheConfig while the first-block cache is on
        self._cache_states = {}     # branch name -> _CacheState
        self._cache_epoch = 0       # bumped by every change of the weights or FP8 switches
        self._text_wins = {}        # (mask identity) -> (mask, int32 [B, 2] device windows): validated once per mask
        self.cache_log = []         # one dict(branch, step, dist, hit) per cached forward since cache_reset()
        self._lora_init()

    def __del__(self):
        for st in getattr(self, "_cache_states", {}).values():
            st.close()
        h = getattr(self, "_h", None)
        if h and _lib is not None and getattr(_lib, "lib", None) is not None:  # not during interpreter teardown
            _lib.lib.b2f_flux_destroy(h)
            self._h = None

    # ------------------------------------------------------------------ nn.Module surface
    @property
    def dtype(self):
        return torch.bfloat16

    @property
    def device(self):
        return next(iter(self._store.values())).device

    def state_dict(self, *a, **k):
        return OrderedDict((n, t) for n, t in self._views.items())

    def load_state_dict(self, sd, strict: bool = True, assign: bool = False):
        missing = [k for k in self._views if k not in sd]
        unexpected = [k for k in sd if k not in self._views]
        if strict and (missing or unexpected):
            raise RuntimeError(f"load_state_dict: missing {missing[:5]}... unexpected {unexpected[:5]}...")
        with torch.no_grad():
            for k, v in self._views.items():
                if k in sd:
                    if tuple(sd[k].shape) != tuple(v.shape):
                        raise RuntimeError(f"{k}: shape {tuple(sd[k].shape)} != {tuple(v.shape)}")
                    v.copy_(sd[k])
        self._fp8_requantize()
        self._cache_epoch += 1
        return SimpleNamespace(missing_keys=missing, unexpected_keys=unexpected)

    @torch.no_grad()
    def randomize_(self, seed: int = 0, std: float = 0.02, bias_std: float = 0.02):
        """Seeded synthetic weights drawn on the device (no checkpoints exist offline; SURVEY.md §8d):
        weights ~ N(0, std^2), biases ~ N(0, bias_std^2), RMSNorm weights = 1."""
        g = torch.Generator(device=self.device).manual_seed(seed)
        for k, t in self._store.items():
            if k.endswith("norm_q.weight") or k.endswith("norm_k.weight") or "norm_added" in k:
                t.fill_(1.0)
            else:
                s_ = bias_std if k.endswith(".bias") else std
                # draw in fp32 chunks to bound temporary memory for the multi-GB fused tensors
                flat = t.view(-1)
                step = 1 << 26
                for o in range(0, flat.numel(), step):
                    n = min(step, flat.numel() - o)
                    flat[o:o + n] = (torch.randn(n, device=self.device, generator=g) * s_).to(torch.bfloat16)
        self._fp8_requantize()
        self._cache_epoch += 1
        return self

    def named_parameters_diffusers(self):
        yield from self._views.items()

    def enable_gradient_checkpointing(self):  # reference train_denoiser.py:486
        self.gradient_checkpointing = True

    def to(self, *args, **kwargs):  # the pipeline calls pipe.to(device) (reference cli.py:69)
        for a in list(args) + list(kwargs.values()):
            if isinstance(a, (str, torch.device)) and torch.device(a).type != "cuda":
                raise _lib.B2FError("B200FluxTransformer2DModel cannot leave the GPU: there is no CPU path")
            if isinstance(a, torch.dtype) and a != torch.bfloat16:
                raise _lib.B2FError("B200FluxTransformer2DModel computes in bfloat16 only")
        return self

    # ------------------------------------------------------------------ FP8
    @property
    def fp8_enabled(self) -> bool:
        """The block linears run in FP8."""
        return self._fp8 is not None

    @property
    def fp8_unfused_lora(self) -> bool:
        """The FP8 block linears run unfused LoRA adapters (enable_fp8(unfused_lora=True))."""
        return self._fp8 is not None and self._fp8_unfused

    @property
    def fp8_attention_enabled(self) -> bool:
        """The blocks' joint attention runs in FP8."""
        return self._fp8_attn

    @torch.no_grad()
    def enable_fp8(self, linears: bool = True, attention: bool = False, unfused_lora: bool = False):
        """Run parts of every transformer block in FP8 (e4m3 operands on the FP8 tensor cores; include/b2f.h).  Each
        switch turns its part on and leaves the others as they are.

        linears    the ten block linears: per-token activation scales, per-output-channel weight scales.  Adds an e4m3
                   copy of those weights (912 d^2 bytes: 8.6 GB at FLUX size) and quantizes it on the device.  The
                   bf16 weights stay the master copy: state_dict(), fuse_lora and training keep seeing them, and
                   load_state_dict / randomize_ / fuse_lora / unfuse_lora re-quantize.  Unfused LoRA adapters must be
                   fused first, unless `unfused_lora` is on.
        unfused_lora  the FP8 block linears (turned on if they are off) also run unfused LoRA adapters: each adapted
                   linear runs its bf16 down projection T on the linear's bf16 input and adds T Bcat^T as bf16 k-blocks
                   after the e4m3 ones of the same GEMM (b2f_gemm_fp8_lora), so the update carries no e4m3 rounding.
                   set_adapters, delete_adapters, disable_lora / enable_lora and the per-call scale then act without
                   touching the e4m3 weights; a LayerNorm whose output feeds an adapted linear runs one extra bf16
                   pass.  Adapters loaded before or after this call act alike.  Off by default: then an unfused
                   adapter is refused while the linears are in FP8.
        attention  the joint attention: Q / K quantized per head, V per channel, P in e4m3 (b2f_attention_fp8).  Adds
                   about 3 bytes per token and channel of workspace.  Touches no weight, so unfused LoRA adapters keep
                   working.  Accuracy cost: e4m3 keeps 3 mantissa bits, so every score carries an error of a few percent
                   of sum |q_i k_i|.  Flat attention rows barely notice; peaked ones do (13 % rel-L2 to exact attention
                   on synthetic heads with a median row max p of 0.6, against 0.17 % for bf16; README), which can be
                   visible in images from checkpoints with such heads."""
        if unfused_lora and not self.fp8_unfused_lora:
            if self._fp8 is None:
                self._enable_fp8_linears(mode=2)
            else:
                check(_lib.lib.b2f_flux_set_fp8(self._h, 2), "b2f_flux_set_fp8")
                self._fp8_unfused = True
                self._lora_rebind()   # adapters loaded while FP8 refused them act now
        elif linears and self._fp8 is None:
            self._enable_fp8_linears()
        if attention and not self._fp8_attn:
            check(_lib.lib.b2f_flux_set_fp8_attention(self._h, 1), "b2f_flux_set_fp8_attention")
            self._fp8_attn = True
        self._cache_epoch += 1
        return self

    def _enable_fp8_linears(self, mode: int = 1):
        if self._lora_bound and mode != 2:
            raise _lib.B2FError("enable_fp8: unfused LoRA adapters are active; fuse_lora() them first")
        fp8 = OrderedDict()
        for name in (t.name for t in flux_layout.layout(self.config) if t.kind == "block"):
            w = self._store[name + ".weight"]
            fp8[name] = (torch.empty(w.shape, device=w.device, dtype=torch.float8_e4m3fn),
                         torch.empty(w.shape[0], device=w.device, dtype=torch.float32))
        self._fp8 = fp8
        self._fp8_requantize()
        for name, (w8, ws) in fp8.items():
            check(_lib.lib.b2f_flux_bind_fp8(self._h, name.encode(), ptr(w8), ptr(ws), w8.numel()),
                  f"b2f_flux_bind_fp8 {name}")
        check(_lib.lib.b2f_flux_set_fp8(self._h, mode), "b2f_flux_set_fp8")
        self._fp8_unfused = mode == 2
        if mode == 2:
            self._lora_rebind()

    def disable_fp8(self):
        """Back to bf16 block linears and attention; the FP8 weight copies are released."""
        self._cache_epoch += 1
        if self._fp8_attn:
            check(_lib.lib.b2f_flux_set_fp8_attention(self._h, 0), "b2f_flux_set_fp8_attention")
            self._fp8_attn = False
        if self._fp8 is None:
            return self
        check(_lib.lib.b2f_flux_set_fp8(self._h, 0), "b2f_flux_set_fp8")
        self._fp8_unfused = False
        for name in self._fp8:
            check(_lib.lib.b2f_flux_bind_fp8(self._h, name.encode(), None, None, 0), f"b2f_flux_bind_fp8 {name}")
        self._fp8 = None
        self._lora_rebind()   # adapters loaded while FP8 was on act unfused again
        return self

    @torch.no_grad()
    def _fp8_requantize(self):
        """FP8 copies <- the row rule (b2f_quant_fp8_rows) of the current bf16 weights, in place."""
        if getattr(self, "_fp8", None) is None:
            return
        for name, (w8, ws) in self._fp8.items():
            w = self._store[name + ".weight"]
            check(_lib.lib.b2f_quant_fp8_rows(ptr(w), w.stride(0), 0, ptr(w8), w8.stride(0), 0, ptr(ws), 0, 1,
                                              w.shape[0], w.shape[1], stream_ptr()), f"b2f_quant_fp8_rows {name}")

    # ------------------------------------------------------------------ first-block cache
    @property
    def cache_enabled(self) -> bool:
        return self._cache_cfg is not None

    def enable_cache(self, config: FirstBlockCacheConfig):
        """Turn on the first-block cache (include/b2f.h, b2f_flux_forward_cached): every full forward runs the
        embedders and block 0, and skips blocks 1.. when block 0's residual moved by less than `config.threshold` since
        the last step of the same branch that ran in full.  An approximation whose hit rate and image quality depend on
        the checkpoint.  The decision is taken for the whole batch, so an item's result can depend on its batch-mates.
        Each branch (joint_attention_kwargs["_b2f_cache_branch"]; FluxKontextPipeline routes the positive forward as
        "cond", the true-CFG negative one as "uncond") keeps its own state of about 10 d bytes per image token plus 4 d
        per output token (302 MB at 1024^2, B = 1).  A cached forward waits on the device once (it reads the decision
        back), so it cannot be captured into a CUDA graph."""
        if not isinstance(config, FirstBlockCacheConfig):
            raise TypeError("enable_cache takes a FirstBlockCacheConfig")
        self._cache_cfg = config
        self.cache_reset()
        return self

    def disable_cache(self):
        """Back to uncached forwards; the states' memory is released."""
        self._cache_cfg = None
        for st in self._cache_states.values():
            st.close()
        self._cache_states = {}
        self.cache_log = []
        return self

    def cache_reset(self):
        """Invalidate every branch's state and clear `cache_log` (FluxKontextPipeline calls this at the start of each
        call, so every image starts with a full step)."""
        for st in self._cache_states.values():
            st.reset()
        self.cache_log = []

    def _cache_forward(self, jak, lora_scale, hs, enc, mod, out, B, S_img, S_txt, n_out, ws, nws):
        branch = str(jak.get("_b2f_cache_branch", "default"))
        st = self._cache_states.get(branch)
        if st is None:
            st = self._cache_states[branch] = _CacheState()
        st.ensure(int(_lib.lib.b2f_flux_cache_bytes(self._h, B, S_img, S_txt, n_out)), self.device)
        key = (self._cache_epoch, self._lora_version, lora_scale)
        if st.key != key:   # weights, adapters, LoRA scale or FP8 switches changed what the blocks compute
            check(_lib.lib.b2f_flux_cache_reset(st.h), "b2f_flux_cache_reset")
            st.key = key
        hit, dist = C.c_int(), C.c_float()
        check(_lib.lib.b2f_flux_forward_cached(self._h, st.h, float(self._cache_cfg.threshold), ptr(hs), ptr(enc),
                                               ptr(mod), mod.stride(0), ptr(out), B, S_img, S_txt, n_out, ptr(ws), nws,
                                               C.byref(hit), C.byref(dist), stream_ptr()), "b2f_flux_forward_cached")
        self.cache_log.append(dict(branch=branch, step=st.calls, dist=float(dist.value), hit=bool(hit.value)))
        st.calls += 1

    def debug_cache(self, branch: str, B: int, S_img: int, n_out: int) -> SimpleNamespace:
        """Views of one branch's cache state in include/b2f.h's layout: r (the slot holding r_prev) and r_other [B,
        S_img, d] fp32, R [B, n_out, d] fp32, y0 [B, S_img, d] bf16 (block 0's output rows of the last call), and
        `valid`.  For tests; only for reading."""
        st = self._cache_states[branch]
        valid, slot = C.c_int(), C.c_int()
        check(_lib.lib.b2f_flux_cache_state(st.h, C.byref(valid), C.byref(slot)), "b2f_flux_cache_state")
        a = lambda n: (n + 255) // 256 * 256
        d = self.inner_dim
        N = B * S_img * d
        off = (-st.mem.data_ptr()) % 256
        o_r1 = a(4 * N)
        o_R = o_r1 + a(4 * N)
        o_p = o_R + a(4 * B * n_out * d)
        o_xy = o_p + a(16 * ((B * S_img + 7) // 8)) + 256
        m = st.mem[off:]
        r = [m[0:4 * N].view(torch.float32).view(B, S_img, d), m[o_r1:o_r1 + 4 * N].view(torch.float32).view(B, S_img, d)]
        return SimpleNamespace(valid=bool(valid.value), r=r[slot.value], r_other=r[1 - slot.value],
                               R=m[o_R:o_R + 4 * B * n_out * d].view(torch.float32).view(B, n_out, d),
                               y0=m[o_xy:o_xy + 2 * N].view(torch.bfloat16).view(B, S_img, d))

    # ------------------------------------------------------------------ helpers
    def _workspace(self, nbytes: int, tag) -> torch.Tensor:
        buf = self._ws.get(tag)
        if buf is None or buf.numel() < nbytes:
            buf = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
            self._ws[tag] = buf
        return buf

    def _temb_mod(self, t1000: torch.Tensor, g1000: torch.Tensor | None, pooled: torch.Tensor, want_silu: bool = False):
        """rows of (timestep*1000, guidance*1000) fp32 + pooled bf16 -> (temb, mod) via the C ABI
        (want_silu: also silu(temb), the input of every AdaLN linear — the training step needs it)."""
        rows = t1000.numel()
        d = self.inner_dim
        temb = torch.empty((rows, d), device=self.device, dtype=torch.bfloat16)
        stemb = torch.empty_like(temb)
        mod = torch.empty((rows, self.mod_width), device=self.device, dtype=torch.bfloat16)
        nws = int(_lib.lib.b2f_flux_temb_workspace_bytes(self._h, rows))
        ws = self._workspace(nws, "temb")
        check(_lib.lib.b2f_flux_temb(self._h, ptr(t1000), ptr(g1000), ptr(pooled), pooled.stride(0), rows,
                                     ptr(temb), ptr(stemb), ptr(ws), nws, stream_ptr()), "b2f_flux_temb")
        if self._lora_bound:   # AdaLN adapters run as their own K-extended launches over their rows of adaln
            nws = int(_lib.lib.b2f_flux_modulation_workspace_bytes(self._h, rows))
            ws = self._workspace(nws, "mod")
            check(_lib.lib.b2f_flux_modulation_ws(self._h, ptr(stemb), rows, ptr(mod), ptr(ws), nws, stream_ptr()),
                  "b2f_flux_modulation_ws")
        else:
            check(_lib.lib.b2f_flux_modulation(self._h, ptr(stemb), rows, ptr(mod), stream_ptr()),
                  "b2f_flux_modulation")
        if want_silu:
            return temb, mod, stemb
        return temb, mod

    @staticmethod
    def _times1000(x: torch.Tensor) -> torch.Tensor:
        # diffusers: `timestep.to(hidden_states.dtype) * 1000` in bf16 (SURVEY.md A.1/A.3), then the
        # sinusoid uses `.float()` of that value.  Scalar bookkeeping, kept in torch on purpose.
        return (x.to(torch.bfloat16) * 1000).float().contiguous()

    def prepare_schedule(self, timesteps_over_1000: torch.Tensor, guidance: torch.Tensor | None,
                         pooled_projections: torch.Tensor, lora_scale: float = 1.0):
        """Hoist the AdaLN modulation of a whole sampling schedule (one weight-streaming GEMM
        with M = steps*B instead of `steps` GEMMs with M = B).  timesteps_over_1000: [n_steps]
        values exactly as the loop will pass them (bf16, already divided by 1000).  lora_scale: the
        joint_attention_kwargs["scale"] the loop will pass (unfused AdaLN adapters act at that scale); a
        forward whose scale or adapters differ from the schedule's computes its own modulation."""
        n = timesteps_over_1000.numel()
        self._set_lora_scale(lora_scale)
        B = pooled_projections.shape[0]
        t = self._times1000(timesteps_over_1000.reshape(n, 1).expand(n, B).reshape(-1))
        g = None
        if self.config.guidance_embeds:
            g = self._times1000(guidance.reshape(1, B).expand(n, B).reshape(-1))
        pooled = pooled_projections.to(torch.bfloat16).repeat(n, 1).contiguous()
        _, mod = self._temb_mod(t, g, pooled)
        self._schedule = SimpleNamespace(n=n, B=B, mod=mod.view(n, B, self.mod_width),
                                         lora_key=(self._lora_version, float(lora_scale)))
        return self._schedule

    def _set_lora_scale(self, s: float):
        check(_lib.lib.b2f_flux_set_lora_scale(self._h, float(s)), "b2f_flux_set_lora_scale")

    def _set_rope(self, txt_ids, img_ids, S_txt: int, S_img: int):
        """FluxPosEmbed tables for [txt; img] ids, handed to the engine (rebuilt only when the ids change)."""
        if txt_ids.dim() == 3:
            txt_ids = txt_ids[0]
        if img_ids.dim() == 3:
            img_ids = img_ids[0]
        key = (txt_ids.data_ptr(), img_ids.data_ptr(), S_txt, S_img, txt_ids._version, img_ids._version)
        if self._rope is None or self._rope[0] != key:
            from . import ops
            ids = torch.cat((txt_ids.float(), img_ids.float()), dim=0).contiguous()
            cos, sin = ops.rope_tables(ids, tuple(self.config.axes_dims_rope))
            self._rope = (key, cos, sin, (txt_ids, img_ids))
        _, cos, sin, _keep = self._rope
        check(_lib.lib.b2f_flux_set_rope(self._h, ptr(cos), ptr(sin), S_txt + S_img), "b2f_flux_set_rope")

    def _text_window(self, mask: torch.Tensor, B: int, S_txt: int) -> torch.Tensor:
        """Device windows of `mask` (text_windows), validated and uploaded once per mask tensor: a sampling loop that
        passes the same mask every step pays one host round trip per call.  The entry keeps the mask alive, so its
        address cannot be reused by another tensor while the entry exists, and an in-place write bumps _version."""
        key = (mask.data_ptr(), mask._version, tuple(mask.shape), str(mask.device), B, S_txt)
        hit = self._text_wins.get(key)
        if hit is None:
            win = text_windows(mask, B, S_txt).to(self.device)
            if len(self._text_wins) >= 8:
                self._text_wins.clear()
            hit = self._text_wins[key] = (mask, win)
        return hit[1]

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(self, hidden_states, encoder_hidden_states=None, pooled_projections=None, timestep=None,
                img_ids=None, txt_ids=None, guidance=None, joint_attention_kwargs=None, return_dict=True,
                encoder_attention_mask=None, **unused):
        """encoder_attention_mask: optional [B, S_txt] mask of the text tokens (1 = token, 0 = padding), each row one
        contiguous run of ones (text_windows).  Batch item b then computes what it computes alone on its unpadded text:
        masked text tokens are never keys for any query, and their content, NaN included, cannot reach an unmasked
        output.  Image tokens are always valid."""
        cfg = self.config
        if self._fp8 is not None and self._lora_bound and not self._fp8_unfused:
            raise _lib.B2FError("FP8 is enabled and LoRA adapters are active unfused: fuse_lora() them first "
                                "(or disable_fp8())")
        jak = dict(joint_attention_kwargs or {})
        if jak.get("attention_mask") is not None:
            raise _lib.B2FError("attention_mask (mixed-size training batches) is not implemented in libb2f")
        B, S_img, _ = hidden_states.shape
        S_txt = encoder_hidden_states.shape[1]
        S = S_txt + S_img
        win = None if encoder_attention_mask is None else self._text_window(encoder_attention_mask, B, S_txt)
        hs = hidden_states.to(torch.bfloat16).contiguous()
        enc = encoder_hidden_states.to(torch.bfloat16).contiguous()
        self._set_rope(txt_ids, img_ids, S_txt, S_img)

        lora_scale = float(jak.pop("scale", 1.0))   # diffusers pops `scale` the same way (PEFT per-call scale)
        self._set_lora_scale(lora_scale)
        step = jak.get("_b2f_schedule_step")
        if (step is not None and self._schedule is not None and self._schedule.B == B
                and self._schedule.lora_key == (self._lora_version, lora_scale)):
            mod = self._schedule.mod[int(step)]
        else:
            t = self._times1000(timestep.reshape(-1).expand(B))
            g = self._times1000(guidance.reshape(-1).expand(B)) if cfg.guidance_embeds else None
            pooled = pooled_projections.to(torch.bfloat16).contiguous()
            _, mod = self._temb_mod(t, g, pooled)
        n_out = int(jak.get("_b2f_out_rows", S_img))
        out = torch.empty((B, n_out, cfg.out_channels), device=self.device, dtype=torch.bfloat16)
        nws = int(_lib.lib.b2f_flux_workspace_bytes(self._h, B, S_img, S_txt))
        ws = self._workspace(nws, "fwd")
        if self._cache_cfg is not None and "_b2f_block_range" in jak:
            raise _lib.B2FError("_b2f_block_range with the first-block cache on: the cache runs whole forwards only "
                                "(disable_cache() first)")
        if win is not None:
            check(_lib.lib.b2f_flux_set_text_window(self._h, ptr(win), B), "b2f_flux_set_text_window")
        try:
            if self._cache_cfg is not None:
                self._cache_forward(jak, lora_scale, hs, enc, mod, out, B, S_img, S_txt, n_out, ws, nws)
                return (out,) if not return_dict else Transformer2DModelOutput(sample=out)
            first, last = jak.get("_b2f_block_range", (0, -1))
            check(_lib.lib.b2f_flux_forward(self._h, ptr(hs), ptr(enc), ptr(mod), mod.stride(0), ptr(out), B, S_img,
                                            S_txt, n_out, ptr(ws), nws, int(first), int(last), stream_ptr()),
                  "b2f_flux_forward")
        finally:
            if win is not None:
                check(_lib.lib.b2f_flux_set_text_window(self._h, None, 0), "b2f_flux_set_text_window")
        if not return_dict:
            return (out,)
        return Transformer2DModelOutput(sample=out)

    def debug_hidden(self, B: int, S_img: int, S_txt: int) -> torch.Tensor:
        """View of the joint activation buffer h[B, S_txt+S_img, d] inside the workspace (block-level
        parity tests read it after a partial-range forward)."""
        return self.debug_buffers(B, S_img, S_txt).h

    def debug_buffers(self, B: int, S_img: int, S_txt: int) -> SimpleNamespace:
        """Views of the whole forward workspace in b2f_flux_forward's layout (text rows first): h and xn [B, S, d],
        qkv [B, S, 3d], cat [B, S, 5d].  After a partial-range forward they hold what the last block left (stage-level
        parity tests read them); the views are only for reading.  With FP8 enabled the blocks quantize their
        LayerNorm outputs straight to e4m3 and do not write xn, except for a LayerNorm feeding an unfused adapter
        (enable_fp8(unfused_lora=True))."""
        ws = self._ws["fwd"]
        off = (-ws.data_ptr()) % 256
        S, d = S_img + S_txt, self.inner_dim
        n = B * S * d
        h, xn, qkv, cat = ws[off:off + 20 * n].view(torch.bfloat16).split([n, n, 3 * n, 5 * n])
        return SimpleNamespace(h=h.view(B, S, d), xn=xn.view(B, S, d), qkv=qkv.view(B, S, 3 * d),
                               cat=cat.view(B, S, 5 * d))
