"""LoRA adapters for the FLUX denoiser: state-dict parsing (host only) and the model-side adapter bookkeeping.

Replaces diffusers' `FluxLoraLoaderMixin` / PEFT as the reference's `FluxKontextPipeline` inherits them (reference
univa/utils/flux_pipeline.py:30, 193-195; per-call scale `joint_attention_kwargs["scale"]`, :922-924).

Accepted layouts (a dict of tensors or a .safetensors file):

  diffusers / PEFT   transformer.<diffusers module>.lora_A.weight / .lora_B.weight   (also without `transformer.`)
  BFL / FLUX code    diffusion_model.<BFL module>.lora_A.weight / .lora_B.weight
  kohya sd-scripts   lora_unet_<BFL module, dots as underscores>.lora_down.weight / .lora_up.weight

A is [r, in] (lora_A / lora_down), B is [out, r] (lora_B / lora_up); an optional `<module>.alpha` makes the scaling
alpha / r, otherwise it is 1.0 (how network alphas become PEFT's lora_alpha).

Every adapter becomes, per engine linear ("target"), one (A [R, in], B [out, R], scale [R]) triple.  The engine stores
several diffusers linears as one fused weight (attn.qkv = [to_q; to_k; to_v], attn.add_qkv, single qkv_mlp =
[to_q; to_k; to_v; proj_mlp]); adapters on such parts become one target on the fused weight: A is the row
concatenation of the parts' A, B is block structured (each part's B in its own output rows and rank columns, zero
elsewhere).  The AdaLN linears (norm1.linear, norm1_context.linear, norm.linear, norm_out.linear) are targets of their
own (rows of the fused adaln weight).  BFL's final_layer.adaLN_modulation.1 chunks (shift, scale) where diffusers'
norm_out.linear chunks (scale, shift): its B rows are swapped.

Anything that is not a LoRA of a linear of the denoiser is refused with a B2FError naming the first offending keys —
text-encoder adapters, DoRA magnitudes, full-weight .diff / .diff_b patches, adapters on norm weights, unknown
modules, A/B ranks that disagree and shapes that do not match the model.  Nothing is skipped silently.
"""
from __future__ import annotations

import os
import re
from collections import OrderedDict
from dataclasses import dataclass

import torch

from ._lib import B2FError


# ------------------------------------------------------------------------------------------------ targets
@dataclass(frozen=True)
class Part:
    """A diffusers linear inside an engine target: rows [row0, row0 + rows) of the target's weight."""
    target: str
    row0: int
    rows: int
    in_features: int
    swap_halves: bool = False     # BFL final_layer.adaLN_modulation.1: (shift, scale) -> (scale, shift)


def targets(cfg) -> "OrderedDict[str, tuple[int, int]]":
    """engine target name -> (out_features, in_features), in the engine's order."""
    d = cfg.num_attention_heads * cfg.attention_head_dim
    t: "OrderedDict[str, tuple[int, int]]" = OrderedDict()
    t["x_embedder"] = (d, cfg.in_channels)
    t["context_embedder"] = (d, cfg.joint_attention_dim)
    embs = ["timestep_embedder", "text_embedder"] + (["guidance_embedder"] if cfg.guidance_embeds else [])
    for e in embs:
        t[f"time_text_embed.{e}.linear_1"] = (d, cfg.pooled_projection_dim if e == "text_embedder" else 256)
        t[f"time_text_embed.{e}.linear_2"] = (d, d)
    for i in range(cfg.num_layers):
        p = f"transformer_blocks.{i}."
        for n, o, k in (("attn.qkv", 3 * d, d), ("attn.add_qkv", 3 * d, d), ("attn.to_out.0", d, d),
                        ("attn.to_add_out", d, d), ("ff.net.0.proj", 4 * d, d), ("ff.net.2", d, 4 * d),
                        ("ff_context.net.0.proj", 4 * d, d), ("ff_context.net.2", d, 4 * d),
                        ("norm1.linear", 6 * d, d), ("norm1_context.linear", 6 * d, d)):
            t[p + n] = (o, k)
    for i in range(cfg.num_single_layers):
        p = f"single_transformer_blocks.{i}."
        t[p + "qkv_mlp"] = (7 * d, d)
        t[p + "proj_out"] = (d, 5 * d)
        t[p + "norm.linear"] = (3 * d, d)
    t["norm_out.linear"] = (2 * d, d)
    t["proj_out"] = (cfg.out_channels, d)
    return t


def adaln_targets(cfg) -> set:
    return {n for n in targets(cfg) if n.endswith("norm1.linear") or n.endswith("norm1_context.linear")
            or n.endswith(".norm.linear") or n == "norm_out.linear"}


def diffusers_parts(cfg) -> "dict[str, Part]":
    """diffusers module name -> Part (every nn.Linear of FluxTransformer2DModel)."""
    d = cfg.num_attention_heads * cfg.attention_head_dim
    out = {}
    for name, (o, k) in targets(cfg).items():
        if not name.endswith(("attn.qkv", "attn.add_qkv", "qkv_mlp")):
            out[name] = Part(name, 0, o, k)
    for i in range(cfg.num_layers):
        p = f"transformer_blocks.{i}."
        for j, n in enumerate(("to_q", "to_k", "to_v")):
            out[p + "attn." + n] = Part(p + "attn.qkv", j * d, d, d)
        for j, n in enumerate(("add_q_proj", "add_k_proj", "add_v_proj")):
            out[p + "attn." + n] = Part(p + "attn.add_qkv", j * d, d, d)
    for i in range(cfg.num_single_layers):
        p = f"single_transformer_blocks.{i}."
        for j, n in enumerate(("to_q", "to_k", "to_v")):
            out[p + "attn." + n] = Part(p + "qkv_mlp", j * d, d, d)
        out[p + "proj_mlp"] = Part(p + "qkv_mlp", 3 * d, 4 * d, d)
    return out


def bfl_parts(cfg) -> "dict[str, Part]":
    """BFL / original FLUX module name -> Part (SURVEY.md A.7)."""
    tg = targets(cfg)

    def whole(name, swap=False):
        o, k = tg[name]
        return Part(name, 0, o, k, swap)
    out = {"img_in": whole("x_embedder"), "txt_in": whole("context_embedder"),
           "time_in.in_layer": whole("time_text_embed.timestep_embedder.linear_1"),
           "time_in.out_layer": whole("time_text_embed.timestep_embedder.linear_2"),
           "vector_in.in_layer": whole("time_text_embed.text_embedder.linear_1"),
           "vector_in.out_layer": whole("time_text_embed.text_embedder.linear_2"),
           "final_layer.linear": whole("proj_out"),
           "final_layer.adaLN_modulation.1": whole("norm_out.linear", swap=True)}
    if cfg.guidance_embeds:
        out["guidance_in.in_layer"] = whole("time_text_embed.guidance_embedder.linear_1")
        out["guidance_in.out_layer"] = whole("time_text_embed.guidance_embedder.linear_2")
    for i in range(cfg.num_layers):
        p, q = f"double_blocks.{i}.", f"transformer_blocks.{i}."
        for b, dn in (("img_mod.lin", "norm1.linear"), ("txt_mod.lin", "norm1_context.linear"),
                      ("img_attn.qkv", "attn.qkv"), ("txt_attn.qkv", "attn.add_qkv"),
                      ("img_attn.proj", "attn.to_out.0"), ("txt_attn.proj", "attn.to_add_out"),
                      ("img_mlp.0", "ff.net.0.proj"), ("img_mlp.2", "ff.net.2"),
                      ("txt_mlp.0", "ff_context.net.0.proj"), ("txt_mlp.2", "ff_context.net.2")):
            out[p + b] = whole(q + dn)
    for i in range(cfg.num_single_layers):
        p, q = f"single_blocks.{i}.", f"single_transformer_blocks.{i}."
        for b, dn in (("linear1", "qkv_mlp"), ("linear2", "proj_out"), ("modulation.lin", "norm.linear")):
            out[p + b] = whole(q + dn)
    return out


# ------------------------------------------------------------------------------------------------ parsing
_NORM_RE = re.compile(r"(norm_q|norm_k|norm_added_q|norm_added_k|query_norm|key_norm)(\.|$)")
_TE_PREFIXES = ("text_encoder.", "text_encoder_2.", "lora_te_", "lora_te1_", "lora_te2_", "te_", "te1_", "te2_")


def _refuse(what: str, keys) -> None:
    keys = sorted(keys)
    more = f" (and {len(keys) - 5} more)" if len(keys) > 5 else ""
    raise B2FError(f"LoRA state dict: {what}: {keys[:5]}{more}")


def read_state_dict(src, weight_name: str | None = None) -> dict:
    """A dict of tensors as is; a .safetensors file, or a directory holding `weight_name`
    (default pytorch_lora_weights.safetensors), read on the host."""
    if isinstance(src, dict):
        return src
    path = os.fspath(src)
    if os.path.isdir(path):
        path = os.path.join(path, weight_name or "pytorch_lora_weights.safetensors")
    if not path.endswith(".safetensors") or not os.path.isfile(path):
        raise B2FError(f"LoRA weights: {path} is not a .safetensors file (no hub access: pass a local file or a dict)")
    from safetensors.torch import load_file
    return load_file(path)


@dataclass
class TargetLora:
    """One adapter on one engine target: A [R, in], B [out, R], per-rank-column scale (alpha_i / r_i) [R]."""
    A: torch.Tensor
    B: torch.Tensor
    scale: torch.Tensor

    @property
    def rank(self) -> int:
        return int(self.A.shape[0])


def parse(sd: dict, cfg) -> "OrderedDict[str, TargetLora]":
    """LoRA state dict (any of the three layouts) -> {engine target: TargetLora}, targets in the engine's order.
    Tensors come back in fp32 on the device they were given on."""
    te = [k for k in sd if k.startswith(_TE_PREFIXES)]
    if te:
        _refuse("text-encoder (CLIP / T5) adapters are not supported", te)
    dora = [k for k in sd if "lora_magnitude_vector" in k or k.endswith(".dora_scale")]
    if dora:
        _refuse("DoRA magnitude vectors are not supported", dora)
    diff = [k for k in sd if k.endswith((".diff", ".diff_b"))]
    if diff:
        _refuse("full-weight .diff / .diff_b patches are not supported", diff)

    dparts, bparts = diffusers_parts(cfg), bfl_parts(cfg)
    kohya = {k.replace(".", "_"): k for k in bparts}
    # (Part, module key as written) -> {"A", "B", "alpha"}
    mods: "dict[str, dict]" = {}
    unknown, norms = [], []
    for key, t in sd.items():
        m = re.fullmatch(r"(.+?)\.(lora_A\.weight|lora_B\.weight|lora_down\.weight|lora_up\.weight|alpha)", key)
        if not m:
            (norms if _NORM_RE.search(key) else unknown).append(key)
            continue
        mod, what = m.group(1), m.group(2)
        if mod.startswith("lora_unet_"):
            b = kohya.get(mod[len("lora_unet_"):])
            part = bparts.get(b) if b else None
        elif mod.startswith("diffusion_model."):
            part = bparts.get(mod[len("diffusion_model."):])
        else:
            name = mod[len("transformer."):] if mod.startswith("transformer.") else mod
            part = dparts.get(name)
        if part is None:
            (norms if _NORM_RE.search(mod) else unknown).append(key)
            continue
        slot = {"lora_A.weight": "A", "lora_down.weight": "A", "lora_B.weight": "B", "lora_up.weight": "B",
                "alpha": "alpha"}[what]
        ent = mods.setdefault(mod, {"part": part})
        ent[slot] = t
    if norms:
        _refuse("adapters on norm weights are not supported", norms)
    if unknown:
        _refuse("keys that are not a LoRA of a linear of the FLUX transformer", unknown)

    # validate every module, then group by target
    per_target: "dict[str, list]" = {}
    seen_parts: dict = {}
    for mod, ent in mods.items():
        part: Part = ent["part"]
        if "A" not in ent or "B" not in ent:
            _refuse("modules without both lora_A/lora_down and lora_B/lora_up", [mod])
        A, B = ent["A"], ent["B"]
        if A.dim() != 2 or B.dim() != 2 or A.shape[0] != B.shape[1]:
            _refuse(f"A {tuple(A.shape)} and B {tuple(B.shape)} ranks disagree", [mod])
        if A.shape[1] != part.in_features or B.shape[0] != part.rows:
            _refuse(f"shapes A {tuple(A.shape)}, B {tuple(B.shape)} do not match the model's "
                    f"[{part.rows}, {part.in_features}] linear", [mod])
        key = (part.target, part.row0)
        if key in seen_parts:
            _refuse("two adapters for the same linear", [seen_parts[key], mod])
        seen_parts[key] = mod
        r = int(A.shape[0])
        alpha = ent.get("alpha")
        s = float(alpha.reshape(-1)[0]) / r if alpha is not None else 1.0
        B = B.float()
        if part.swap_halves:
            h = B.shape[0] // 2
            B = torch.cat([B[h:], B[:h]])
        per_target.setdefault(part.target, []).append((part.row0, part.rows, A.float(), B, s))

    out: "OrderedDict[str, TargetLora]" = OrderedDict()
    tg = targets(cfg)
    for name, (o, k) in tg.items():
        subs = per_target.get(name)
        if not subs:
            continue
        subs.sort(key=lambda e: e[0])
        R = sum(int(e[2].shape[0]) for e in subs)
        dev = subs[0][2].device
        A = torch.cat([e[2] for e in subs])
        B = torch.zeros(o, R, device=dev)
        scale = torch.empty(R, device=dev)
        c = 0
        for row0, rows, a, b, s in subs:
            r = int(a.shape[0])
            B[row0:row0 + rows, c:c + r] = b
            scale[c:c + r] = s
            c += r
        out[name] = TargetLora(A, B, scale)
    return out


# ------------------------------------------------------------------------------------------------ model side
def _pad64(r: int) -> int:
    return -(-r // 64) * 64


class FluxLoraMixin:
    """diffusers' PEFT adapter surface on B200FluxTransformer2DModel (load_lora_adapter, set_adapters, fuse_lora, ...).

    Adapters are kept per target in fp32 on the device.  The active, unfused ones are bound to the engine as one
    concatenated (Acat, Bcat, colscale) per target — colscale = alpha_i / r_i x adapter weight_i on adapter i's rank
    columns — and run as the down projection + K-extended GEMM of b2f_gemm_bf16_lora; the per-call
    joint_attention_kwargs["scale"] multiplies every colscale (b2f_flux_set_lora_scale).

    Active set: `set_adapters` always replaces it.  Loading an adapter adds it to the active set with weight 1.0 and
    leaves the adapters already active as they were (so two loads without set_adapters run both).
    """

    def _lora_init(self):
        self._lora: "OrderedDict[str, OrderedDict[str, TargetLora]]" = OrderedDict()   # adapter -> target -> lora
        self._lora_active: "OrderedDict[str, float]" = OrderedDict()                     # adapter -> weight
        self._lora_enabled = True
        self._lora_fused: set = set()            # adapters merged into the weights
        self._lora_saved: dict = {}              # target -> copy of its weight rows before the first fuse
        self._lora_bound: dict = {}              # target -> (Acat, Bcat, colscale) the engine borrows
        self._lora_version = 0                   # bumped on every change the forward / hoisted schedule depends on

    # ---------------------------------------------------------------- helpers
    def _lora_weight(self, target: str) -> torch.Tensor:
        w = self._store.get(target + ".weight")
        return w if w is not None else self._views[target + ".weight"]

    def _lora_unfused_set(self) -> "OrderedDict[str, float]":
        if not self._lora_enabled:
            return OrderedDict()
        return OrderedDict((n, w) for n, w in self._lora_active.items() if n not in self._lora_fused)

    def _lora_concat(self, names: "OrderedDict[str, float]", pad: bool):
        """target -> (Acat bf16 [R, in], Bcat bf16 [out, R], colscale fp32 [R]) over the adapters `names`, in order;
        R padded to a multiple of 64 with zeros when `pad`."""
        per: "dict[str, list]" = {}
        for n, wgt in names.items():
            for t, tl in self._lora[n].items():
                per.setdefault(t, []).append((tl, wgt))
        out = {}
        for t, lst in per.items():
            R = sum(tl.rank for tl, _ in lst)
            Rp = _pad64(R) if pad else R
            o, k = int(lst[0][0].B.shape[0]), int(lst[0][0].A.shape[1])
            A = torch.zeros(Rp, k, device=self.device, dtype=torch.bfloat16)
            B = torch.zeros(o, Rp, device=self.device, dtype=torch.bfloat16)
            cs = torch.zeros(Rp, device=self.device, dtype=torch.float32)
            c = 0
            for tl, wgt in lst:
                r = tl.rank
                A[c:c + r] = tl.A
                B[:, c:c + r] = tl.B
                cs[c:c + r] = tl.scale * wgt
                c += r
            out[t] = (A, B, cs)
        return out

    def _lora_rebind(self):
        from . import _lib
        _lib.check(_lib.lib.b2f_flux_clear_lora(self._h), "b2f_flux_clear_lora")
        self._lora_bound = self._lora_concat(self._lora_unfused_set(), pad=True)
        # with FP8 linears enabled the engine takes unfused adapters only with enable_fp8(unfused_lora=True); otherwise
        # the forward refuses until they are fused or FP8 is off
        refused = getattr(self, "_fp8", None) is not None and not getattr(self, "_fp8_unfused", False)
        for t, (A, B, cs) in ({} if refused else self._lora_bound).items():
            _lib.check(_lib.lib.b2f_flux_bind_lora(self._h, t.encode(), A.data_ptr(), B.data_ptr(), cs.data_ptr(),
                                                   int(A.shape[0])), f"b2f_flux_bind_lora {t}")
        self._lora_version += 1
        self._schedule = None

    def lora_unfused_active(self) -> bool:
        """True while an adapter acts on the forward without being merged into the weights."""
        return bool(self._lora_bound)

    # ---------------------------------------------------------------- diffusers surface
    def load_lora_adapter(self, pretrained_model_name_or_path_or_dict, adapter_name: str | None = None,
                          weight_name: str | None = None, prefix: str | None = "transformer", **kw):
        sd = read_state_dict(pretrained_model_name_or_path_or_dict, weight_name)
        if adapter_name is None:
            i = 0
            while f"default_{i}" in self._lora:
                i += 1
            adapter_name = f"default_{i}"
        if adapter_name in self._lora:
            raise ValueError(f"adapter name {adapter_name!r} is already in use")
        parsed = parse(sd, self.config)
        if not parsed:
            raise B2FError("LoRA state dict: no adapter weights for the transformer")
        self._lora[adapter_name] = OrderedDict(
            (t, TargetLora(tl.A.to(self.device, torch.float32), tl.B.to(self.device, torch.float32),
                           tl.scale.to(self.device, torch.float32))) for t, tl in parsed.items())
        self._lora_active[adapter_name] = 1.0
        self._lora_rebind()
        return adapter_name

    def set_adapters(self, adapter_names, weights=None):
        names = [adapter_names] if isinstance(adapter_names, str) else list(adapter_names)
        missing = [n for n in names if n not in self._lora]
        if missing:
            raise ValueError(f"unknown adapters {missing}; loaded: {list(self._lora)}")
        if weights is None:
            weights = [1.0] * len(names)
        elif isinstance(weights, (int, float)):
            weights = [float(weights)] * len(names)
        weights = list(weights)
        if len(weights) != len(names):
            raise ValueError(f"{len(names)} adapters but {len(weights)} weights")
        self._lora_active = OrderedDict((n, 1.0 if w is None else float(w)) for n, w in zip(names, weights))
        self._lora_rebind()

    def get_active_adapters(self) -> list:
        return list(self._lora_active) if self._lora_enabled else []

    def get_list_adapters(self) -> dict:
        return {"transformer": list(self._lora)}

    def delete_adapters(self, adapter_names):
        names = [adapter_names] if isinstance(adapter_names, str) else list(adapter_names)
        for n in names:
            if n not in self._lora:
                raise ValueError(f"unknown adapter {n!r}")
            del self._lora[n]
            self._lora_active.pop(n, None)
            self._lora_fused.discard(n)        # merged weights stay merged; unfuse_lora still restores them
        self._lora_rebind()

    def disable_lora(self):
        self._lora_enabled = False
        self._lora_rebind()

    def enable_lora(self):
        self._lora_enabled = True
        self._lora_rebind()

    def unload_lora(self):
        """Drop every adapter.  Weights merged by fuse_lora stay merged (they are just weights now)."""
        self._lora.clear()
        self._lora_active.clear()
        self._lora_fused.clear()
        self._lora_saved.clear()
        self._lora_rebind()

    @torch.no_grad()
    def fuse_lora(self, lora_scale: float = 1.0, adapter_names=None, **kw):
        """Merge adapters into the weights: W <- bf16(W + lora_scale * sum_i w_i alpha_i / r_i B_i A_i), one fp32
        accumulation and one rounding per element (b2f_lora_fuse).  Defaults to the active, unfused adapters.  The
        weight rows are saved first, so unfuse_lora restores them exactly (diffusers subtracts the delta again,
        which is inexact in bf16)."""
        from . import _lib
        if adapter_names is None:
            names = OrderedDict((n, w) for n, w in self._lora_active.items() if n not in self._lora_fused)
        else:
            names = [adapter_names] if isinstance(adapter_names, str) else list(adapter_names)
            missing = [n for n in names if n not in self._lora]
            if missing:
                raise ValueError(f"unknown adapters {missing}")
            names = OrderedDict((n, self._lora_active.get(n, 1.0)) for n in names if n not in self._lora_fused)
        for t, (A, B, cs) in self._lora_concat(names, pad=False).items():
            w = self._lora_weight(t)
            if t not in self._lora_saved:
                self._lora_saved[t] = w.clone()
            _lib.check(_lib.lib.b2f_lora_fuse(w.data_ptr(), w.stride(0), w.shape[0], w.shape[1], B.data_ptr(),
                                              B.stride(0), A.data_ptr(), A.stride(0), cs.data_ptr(), float(lora_scale),
                                              int(A.shape[0]), _lib.stream_ptr()), f"b2f_lora_fuse {t}")
        self._lora_fused.update(names)
        self._fp8_requantize()
        self._lora_rebind()

    @torch.no_grad()
    def unfuse_lora(self, **kw):
        """Restore the weight rows saved by the first fuse_lora, bit for bit; the adapters act unfused again."""
        for t, saved in self._lora_saved.items():
            self._lora_weight(t).copy_(saved)
        self._lora_saved.clear()
        self._lora_fused.clear()
        self._fp8_requantize()
        self._lora_rebind()
