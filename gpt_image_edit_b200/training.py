"""Stage-2 training engine over libb2f (reference train_denoiser.py:829-1181, scripts/accelerate_configs/zero2.json).

What the reference assembles from accelerate + DeepSpeed ZeRO-2 + torch.autograd, written out for this engine:

  FluxTrainGraph       forward with per-block checkpoints / backward with per-block recompute of the FLUX denoiser
                       (`b2f_flux_train_forward` / `b2f_flux_train_backward`) plus MLP2's forward / backward
                       (two wgmma GEMMs each way), gradients in fp32
  trainable_params()   the reference's trainable set (train_denoiser.py:71-119, 519-548) mapped onto this repo's
                       fused weight storage
  ShardedAdamW         ZeRO-2: gradients live in per-block buckets; each bucket is reduce-scattered (NCCL, fp32)
                       as soon as its block's backward has been enqueued — on a side stream, overlapping the
                       backward of the next block —, every rank keeps fp32 master weights and Adam moments for
                       its 1/world slice only, clips by the global norm, updates its slice and all-gathers the new
                       bf16 weights (zero2.json: stage 2, reduce_scatter true, overlap_comm true)

All arithmetic is libb2f (`train_ops`); torch provides storage, streams and the process group.  The `math`
argument exists so that the CPU `gloo` tests can substitute the oracle's torch implementations for the CUDA
kernels when they check the sharding logic; the product never passes it.
"""
from __future__ import annotations

from dataclasses import dataclass

import torch
import torch.distributed as dist

from . import _lib
from ._lib import check, ptr, stream_ptr


# ------------------------------------------------------------------------------------------------ trainable set
def get_trainable_params(layers_to_train=None, num_transformer_blocks: int = 19, only_img_branch: bool = True):
    """Component-name list of the reference (train_denoiser.py:71-112), same strings in the same order."""
    layers_to_train = list(range(57)) if layers_to_train is None else layers_to_train
    components = []
    transformer_components = ["attn.norm_q", "attn.norm_k", "attn.to_q", "attn.to_k", "attn.to_v", "attn.to_out", "norm1.linear"]
    single_transformer_components = ["attn.norm_q", "attn.norm_k", "attn.to_q", "attn.to_k", "attn.to_v", "norm.linear"]
    if not only_img_branch:
        transformer_components.extend(["norm1_context.linear", "attn.norm_added_q", "attn.norm_added_k", "ff.net", "ff_context.net"])
        single_transformer_components.extend(["proj_mlp", "proj_out"])
    for layer in layers_to_train:
        if layer < num_transformer_blocks:
            prefix = f"denoise_tower.denoiser.transformer_blocks.{layer}"
            base = transformer_components
        else:
            prefix = f"denoise_tower.denoiser.single_transformer_blocks.{layer - num_transformer_blocks}"
            base = single_transformer_components
        components.extend([f"{prefix}.{comp}" for comp in base])
    return components


def check_param_is_in_components(name: str, components) -> bool:      # train_denoiser.py:118-119
    return any(component in name for component in components)


def trained_flux_layers(mc) -> list:
    """Block indices whose components train under a ModelConfig (train_denoiser.py:527-543): none with `only_tune_mlp2`,
    none when `flux_train_layer_idx` is left at its default None, else the listed ones (0-18 double, 19-56 single)."""
    if mc.only_tune_mlp2 or mc.flux_train_layer_idx is None:
        return []
    return list(mc.flux_train_layer_idx)


@dataclass
class Param:
    name: str            # diffusers-style name(s) this tensor answers to (for the log / checkpoint)
    storage: torch.Tensor  # contiguous bf16 view into the model's weight storage
    bind_key: str | None   # b2f_flux_bind_grad key (None: MLP2, handled in Python)
    bucket: int
    grad: torch.Tensor | None = None    # fp32 view into the bucket's flat gradient
    offset: int = 0


def trainable_params(model, layers_to_train=None, only_img_branch: bool = True, with_tune_mlp2: bool = True):
    """[Param] for a UnivaQwen2p5VLForConditionalGeneration: bucket i = FLUX block i, last bucket = MLP2."""
    if not only_img_branch:
        raise _lib.B2FError("only_tune_image_branch=False (FF / text-stream weights) is not built: every stage yaml of the "
                            "reference trains the image branch only")
    den = model.denoise_tower.denoiser
    cfg = den.config
    d = den.inner_dim
    nd, ns = cfg.num_layers, cfg.num_single_layers
    layers = list(range(nd + ns)) if layers_to_train is None else [l for l in layers_to_train if l < nd + ns]
    st = den._store
    adaln_w, adaln_b = st["adaln.weight"], st["adaln.bias"]
    out = []
    for l in layers:
        if l < nd:
            p = f"transformer_blocks.{l}."
            r0 = l * 12 * d
            out += [Param(p + "attn.to_q|to_k|to_v.weight", st[p + "attn.qkv.weight"], p + "attn.qkv.weight", l),
                    Param(p + "attn.to_q|to_k|to_v.bias", st[p + "attn.qkv.bias"], p + "attn.qkv.bias", l),
                    Param(p + "attn.to_out.0.weight", st[p + "attn.to_out.0.weight"], p + "attn.to_out.0.weight", l),
                    Param(p + "attn.to_out.0.bias", st[p + "attn.to_out.0.bias"], p + "attn.to_out.0.bias", l),
                    Param(p + "attn.norm_q.weight", st[p + "attn.norm_q.weight"], p + "attn.norm_q.weight", l),
                    Param(p + "attn.norm_k.weight", st[p + "attn.norm_k.weight"], p + "attn.norm_k.weight", l),
                    Param(p + "norm1.linear.weight", adaln_w[r0:r0 + 6 * d], p + "norm1.linear.weight", l),
                    Param(p + "norm1.linear.bias", adaln_b[r0:r0 + 6 * d], p + "norm1.linear.bias", l)]
        else:
            j = l - nd
            p = f"single_transformer_blocks.{j}."
            r0 = nd * 12 * d + j * 3 * d
            out += [Param(p + "attn.to_q|to_k|to_v.weight", st[p + "qkv_mlp.weight"][:3 * d], p + "attn.qkv.weight", l),
                    Param(p + "attn.to_q|to_k|to_v.bias", st[p + "qkv_mlp.bias"][:3 * d], p + "attn.qkv.bias", l),
                    Param(p + "attn.norm_q.weight", st[p + "attn.norm_q.weight"], p + "attn.norm_q.weight", l),
                    Param(p + "attn.norm_k.weight", st[p + "attn.norm_k.weight"], p + "attn.norm_k.weight", l),
                    Param(p + "norm.linear.weight", adaln_w[r0:r0 + 3 * d], p + "norm.linear.weight", l),
                    Param(p + "norm.linear.bias", adaln_b[r0:r0 + 3 * d], p + "norm.linear.bias", l)]
    if with_tune_mlp2:
        proj = model.denoise_tower.denoise_projector
        b = nd + ns
        out += [Param("denoise_projector.0.weight", proj.w0, None, b), Param("denoise_projector.0.bias", proj.b0, None, b),
                Param("denoise_projector.2.weight", proj.w2, None, b), Param("denoise_projector.2.bias", proj.b2, None, b)]
    for q in out:
        if not q.storage.is_contiguous():
            raise _lib.B2FError(f"{q.name}: trainable storage must be contiguous")
    return out


# ------------------------------------------------------------------------------------------------ ZeRO-2 AdamW
class _B2FMath:
    """The CUDA kernels (train_ops).  CPU tests substitute oracle.train_oracle.TorchMath."""

    @staticmethod
    def cast_to_f32(src):
        from . import train_ops as T
        return T.cast(src.contiguous(), torch.float32)

    @staticmethod
    def cast_to_bf16(src):
        from . import train_ops as T
        return T.cast(src.contiguous(), torch.bfloat16)

    @staticmethod
    def sumsq(g, out, accumulate):
        from . import train_ops as T
        T.grad_sumsq(g, out=out, accumulate=accumulate)

    @staticmethod
    def clip_coef(sumsq, max_norm, pre_scale):
        from . import train_ops as T
        return T.clip_coef(sumsq, max_norm, pre_scale)

    @staticmethod
    def adamw(p32, m, v, g, p16, **kw):
        from . import train_ops as T
        T.adamw_step_(p32, m, v, g, p16=p16, **kw)


@dataclass
class _Bucket:
    params: list
    size: int            # padded to a multiple of world * 64 elements
    flat_grad: torch.Tensor = None     # fp32 [size]: this rank's (local) gradients of the bucket
    shard_grad: torch.Tensor = None    # fp32 [size / world]: the reduced slice this rank owns
    p32: torch.Tensor = None
    m: torch.Tensor = None
    v: torch.Tensor = None
    flat_p16: torch.Tensor = None      # bf16 [size]: updated weights, all-gathered
    reduced: torch.cuda.Event | None = None


class ShardedAdamW:
    """AdamW with ZeRO-2 partitioning over `group` (world 1: plain AdamW with fp32 master weights)."""

    def __init__(self, params, lr=1e-5, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01, max_grad_norm=1.0,
                 group=None, math=None, comm_stream=None):
        self.math = math or _B2FMath
        self.group = group
        self.world = dist.get_world_size(group) if (dist.is_available() and dist.is_initialized()) else 1
        self.rank = dist.get_rank(group) if self.world > 1 else 0
        self.lr, self.betas, self.eps, self.wd, self.max_grad_norm = lr, betas, eps, weight_decay, max_grad_norm
        self.step_count = 0
        self.comm_stream = comm_stream
        nb = max(p.bucket for p in params) + 1
        self.buckets: list[_Bucket] = []
        for b in range(nb):
            ps = [p for p in params if p.bucket == b]
            if not ps:
                self.buckets.append(None)
                continue
            dev = ps[0].storage.device
            off = 0
            for p in ps:
                p.offset = off
                off += (p.storage.numel() + 63) // 64 * 64      # 256-byte aligned fp32 views for the TMA-free kernels
            quantum = self.world * 64
            size = (off + quantum - 1) // quantum * quantum
            bk = _Bucket(ps, size)
            bk.flat_grad = torch.zeros(size, device=dev, dtype=torch.float32)
            for p in ps:
                p.grad = bk.flat_grad[p.offset:p.offset + p.storage.numel()].view(p.storage.shape)
            n = size // self.world
            bk.shard_grad = bk.flat_grad if self.world == 1 else torch.zeros(n, device=dev, dtype=torch.float32)
            # fp32 master copy of this rank's slice (DeepSpeed bf16 optimizer: fp32 partitions of the bf16 weights)
            flat16 = torch.zeros(size, device=dev, dtype=torch.bfloat16)
            for p in ps:
                flat16[p.offset:p.offset + p.storage.numel()].copy_(p.storage.reshape(-1))
            bk.flat_p16 = flat16
            lo = self.rank * n
            bk.p32 = self.math.cast_to_f32(flat16[lo:lo + n])
            bk.m = torch.zeros_like(bk.p32)
            bk.v = torch.zeros_like(bk.p32)
            self.buckets.append(bk)
        dev = params[0].storage.device
        self._sumsq = torch.zeros(1, device=dev, dtype=torch.float32)
        self.last_grad_norm = None

    # -- gradient reduction -------------------------------------------------------------------
    def reduce_bucket(self, b: int):
        """reduce-scatter bucket b's local gradients (sum over ranks) into this rank's slice.  Enqueued on the comm
        stream after everything already enqueued on the current stream (the block's backward)."""
        bk = self.buckets[b]
        if bk is None or self.world == 1:
            return
        if self.comm_stream is not None:
            self.comm_stream.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(self.comm_stream):
                dist.reduce_scatter_tensor(bk.shard_grad, bk.flat_grad, op=dist.ReduceOp.SUM, group=self.group)
                bk.reduced = torch.cuda.Event()
                bk.reduced.record(self.comm_stream)
        else:
            dist.reduce_scatter_tensor(bk.shard_grad, bk.flat_grad, op=dist.ReduceOp.SUM, group=self.group)

    def reduce_all(self):
        for b in range(len(self.buckets)):
            self.reduce_bucket(b)

    # -- the update ---------------------------------------------------------------------------
    def step(self, lr: float | None = None):
        """clip_grad_norm_(max_grad_norm) + AdamW on this rank's slices + all-gather of the new bf16 weights.
        Gradients are averaged over ranks (DDP / ZeRO semantics): the 1/world factor is folded into the clip scale."""
        lr = self.lr if lr is None else lr
        self.step_count += 1
        live = [bk for bk in self.buckets if bk is not None]
        if self.comm_stream is not None and self.world > 1:
            torch.cuda.current_stream().wait_stream(self.comm_stream)
        for i, bk in enumerate(live):
            self.math.sumsq(bk.shard_grad, self._sumsq, accumulate=i > 0)
        if self.world > 1:
            dist.all_reduce(self._sumsq, op=dist.ReduceOp.SUM, group=self.group)
        coef, norm = self.math.clip_coef(self._sumsq, self.max_grad_norm, 1.0 / self.world)
        self.last_grad_norm = norm
        for bk in live:
            n = bk.size // self.world
            lo = self.rank * n
            self.math.adamw(bk.p32, bk.m, bk.v, bk.shard_grad, bk.flat_p16[lo:lo + n], lr=lr, betas=self.betas, eps=self.eps,
                            weight_decay=self.wd, step=self.step_count, gscale=coef)
            if self.world > 1:
                dist.all_gather_into_tensor(bk.flat_p16, bk.flat_p16[lo:lo + n].clone(), group=self.group)
            for p in bk.params:        # scatter the flat bucket back into the model's (fused) weight storage
                p.storage.copy_(bk.flat_p16[p.offset:p.offset + p.storage.numel()].view(p.storage.shape))
        return norm

    def zero_grad(self):
        for bk in self.buckets:
            if bk is not None:
                bk.flat_grad.zero_()

    def state_dict(self):
        return {"step": self.step_count, "rank": self.rank, "world": self.world,
                "buckets": [None if bk is None else {"p32": bk.p32, "m": bk.m, "v": bk.v} for bk in self.buckets]}

    def load_state_dict(self, sd):
        """Restore a `state_dict()` of the same partitioning: step count, fp32 master slices and moments — and the bf16
        weights the model computes with, which are the rounded masters of ALL ranks (each rank rounds its slice, the
        slices are all-gathered and scattered into the model's storage, exactly as at the end of `step`).  What
        `accelerator.load_state` does for the reference (train_denoiser.py:769: DeepSpeed reloads module + optimizer)."""
        if sd["world"] != self.world or sd.get("rank", self.rank) != self.rank:
            raise _lib.B2FError(f"optimizer state is rank {sd.get('rank')} of {sd['world']} ranks, this process is rank "
                                f"{self.rank} of {self.world}")
        if len(sd["buckets"]) != len(self.buckets):
            raise _lib.B2FError(f"optimizer state has {len(sd['buckets'])} buckets, this run has {len(self.buckets)}")
        for bk, s in zip(self.buckets, sd["buckets"]):
            if (bk is None) != (s is None) or (bk is not None and s["p32"].numel() != bk.p32.numel()):
                raise _lib.B2FError("optimizer state does not match this run's trainable set (bucket sizes differ)")
        self.step_count = sd["step"]
        for bk, s in zip(self.buckets, sd["buckets"]):
            if bk is None:
                continue
            bk.p32.copy_(s["p32"]); bk.m.copy_(s["m"]); bk.v.copy_(s["v"])
            n = bk.size // self.world
            lo = self.rank * n
            bk.flat_p16[lo:lo + n].copy_(self.math.cast_to_bf16(bk.p32))
            if self.world > 1:
                dist.all_gather_into_tensor(bk.flat_p16, bk.flat_p16[lo:lo + n].clone(), group=self.group)
            for p in bk.params:
                p.storage.copy_(bk.flat_p16[p.offset:p.offset + p.storage.numel()].view(p.storage.shape))


# ------------------------------------------------------------------------------------------------ forward / backward
class FluxTrainGraph:
    """One training forward/backward of MLP2 -> FLUX denoiser with the gradients of `params` accumulated into their
    fp32 buffers.  Reference: lvlm_model(..., output_type="denoise_model_pred") + accelerator.backward(loss),
    train_denoiser.py:1073-1093, 1172."""

    def __init__(self, model, params, on_block_done=None):
        self.model = model
        self.den = model.denoise_tower.denoiser
        if getattr(self.den, "lora_unfused_active", lambda: False)():
            raise _lib.B2FError("the denoiser has unfused LoRA adapters active and the training backward does not see them: "
                           "fuse_lora() or disable / unload them first")
        self.proj = getattr(model.denoise_tower, "denoise_projector", None)
        self.params = params
        self.on_block_done = on_block_done          # callback(bucket) after a block's gradients are complete
        self._bound = False
        self._mlp2 = {p.name: p for p in params if p.bind_key is None}
        self.n_blocks = self.den.config.num_layers + self.den.config.num_single_layers
        self._trained_blocks = sorted({p.bucket for p in params if p.bind_key is not None})

    def _bind(self):
        for p in self.params:
            if p.bind_key is not None:
                check(_lib.lib.b2f_flux_bind_grad(self.den._h, p.bind_key.encode(), ptr(p.grad), p.grad.numel()),
                      f"bind grad {p.bind_key}")
        self._bound = True

    def forward(self, vlm_hidden, hidden_states, timestep, guidance, pooled, img_ids, n_out_rows, prefix_embeds=None):
        """vlm_hidden [B, L, 3584] (Qwen2.5-VL prefill output, frozen) -> MLP2 -> [vlm ‖ prefix] -> denoiser.
        Returns model_pred [B, n_out_rows, 64] bf16 (the target tokens)."""
        from . import ops
        den = self.den
        if not self._bound:
            self._bind()
        x = vlm_hidden.to(torch.bfloat16).contiguous()
        self._x = x
        self._pre = ops.linear(x, self.proj.w0, self.proj.b0)                     # kept for silu'
        self._act = torch.empty_like(self._pre)
        check(_lib.lib.b2f_silu(ptr(self._pre), ptr(self._act), self._pre.numel(), stream_ptr()), "b2f_silu")
        enc_vlm = ops.linear(self._act, self.proj.w2, self.proj.b2)
        self._L = enc_vlm.shape[1]
        enc = enc_vlm if prefix_embeds is None else torch.cat([enc_vlm, prefix_embeds.to(torch.bfloat16)], dim=1)
        enc = enc.contiguous()
        B, S_img, _ = hidden_states.shape
        S_txt = enc.shape[1]
        txt_ids = torch.zeros(S_txt, 3, device=enc.device, dtype=torch.bfloat16)
        den._set_rope(txt_ids, img_ids, S_txt, S_img)
        t = den._times1000(timestep.reshape(-1).expand(B))
        g = den._times1000(guidance.reshape(-1).expand(B)) if den.config.guidance_embeds else None
        _, mod, stemb = den._temb_mod(t, g, pooled.to(torch.bfloat16).contiguous(), want_silu=True)
        hs = hidden_states.to(torch.bfloat16).contiguous()
        out = torch.empty((B, n_out_rows, den.config.out_channels), device=enc.device, dtype=torch.bfloat16)
        nws = int(_lib.lib.b2f_flux_train_workspace_bytes(den._h, B, S_img, S_txt))
        ws = den._workspace(nws, "train")
        check(_lib.lib.b2f_flux_train_forward(den._h, ptr(hs), ptr(enc), ptr(mod), mod.stride(0), ptr(out), B, S_img, S_txt,
                                              n_out_rows, ptr(ws), nws, stream_ptr()), "b2f_flux_train_forward")
        self._ctx = dict(B=B, S_img=S_img, S_txt=S_txt, n_out=n_out_rows, mod=mod, stemb=stemb, ws=ws, nws=nws, hs=hs, enc=enc)
        return out

    def backward(self, dpred, accumulate: bool = False):
        from . import train_ops as T
        den, c = self.den, self._ctx
        d_enc = torch.empty_like(c["enc"])
        dpred = dpred.contiguous()

        def run(first, last):
            check(_lib.lib.b2f_flux_train_backward(den._h, ptr(dpred), ptr(c["mod"]), c["mod"].stride(0), ptr(c["stemb"]),
                                                   c["stemb"].stride(0), ptr(d_enc), c["B"], c["S_img"], c["S_txt"],
                                                   c["n_out"], int(accumulate), ptr(c["ws"]), c["nws"], first, last,
                                                   stream_ptr()), "b2f_flux_train_backward")

        if self.on_block_done is None:
            run(0, -1)
        else:
            # block by block: each block's gradient bucket is reduced while the next block's backward runs
            for blk in range(self.n_blocks - 1, -1, -1):
                run(blk, blk + 1)
                self.on_block_done(blk)
        # MLP2: enc_vlm = silu(x W0^T + b0) W2^T + b2
        if self._mlp2:
            d_vlm = d_enc[:, :self._L]
            m = self._mlp2
            T.linear_wgrad(d_vlm, self._act, out=m["denoise_projector.2.weight"].grad, accumulate=accumulate)
            self._bias_grad(d_vlm, m["denoise_projector.2.bias"].grad, accumulate)
            dpre = T.linear_dgrad(d_vlm, self.proj.w2, epilogue=T.EPI_DSILU, aux=self._pre)
            T.linear_wgrad(dpre, self._x, out=m["denoise_projector.0.weight"].grad, accumulate=accumulate)
            self._bias_grad(dpre, m["denoise_projector.0.bias"].grad, accumulate)
            if self.on_block_done is not None:
                self.on_block_done(self.n_blocks)
        return d_enc

    @staticmethod
    def _bias_grad(dy, dst, accumulate):
        from . import train_ops as T
        _, col = T.gate_bwd(dy, want_dy=False)                    # [B, D] per-batch column sums
        _lib.check(_lib.lib.b2f_col_reduce(ptr(col), col.shape[0], col.shape[1], ptr(dst), col.shape[1], 1, int(accumulate),
                                           stream_ptr()), "b2f_col_reduce")


def flow_matching_loss(pred, target, weight=None, grad_scale: float = 1.0):
    """(loss, dpred): mean(weight * (pred - target)^2) and its gradient (train_denoiser.py:1105-1167)."""
    from . import train_ops as T
    return T.mse_loss(pred.contiguous(), target.contiguous(), weight=weight, grad_scale=grad_scale)


def pad_x_and_mask(xs, masks=None, max_h=None, max_w=None):
    """Mixed-size batches (train_denoiser.py:158-183): zero-pad a list of [1, C, h_i, w_i] tensors on the right / bottom to
    a common size and concatenate; `masks` (same shapes) are cut to one channel and padded the same way.
    Returns (x [B, C, H, W], mask [B, 1, H, W] | None)."""
    F = torch.nn.functional
    max_h = max(t.shape[2] for t in xs) if max_h is None else max_h
    max_w = max(t.shape[3] for t in xs) if max_w is None else max_w
    pad = lambda t: F.pad(t, (0, max_w - t.shape[3], 0, max_h - t.shape[2]), mode="constant", value=0)
    x = torch.cat([pad(t) for t in xs], dim=0)
    if masks is None or masks[0] is None:
        return x, None
    return x, torch.cat([pad(m[:, :1]) for m in masks], dim=0)


def pack_training_latents(pipe, noisy, cond, device, dtype):
    """The transformer's token inputs for one training micro-batch (train_denoiser.py:996-1056): the noised target latents
    [B, C, h, w] packed into 2x2 patches, followed — when a context image is given — by the packed VAE latents of the
    context (`prepare_latents` encodes it and returns it PACKED, the target comes back unpacked and is packed here), and
    the position ids of both (context ids carry 1 in their first coordinate).  Returns (tokens [B, S, 4C], ids [S, 3])."""
    B, C, h, w = noisy.shape
    vsf = pipe.vae_scale_factor
    if cond is not None:
        latents, image_latents, ids_t, ids_c = pipe.prepare_latents(cond, B, C, h * vsf, w * vsf, dtype, device, None, noisy)
        packed_t = pipe._pack_latents(latents, B, C, h, w)
        if image_latents is None:
            return packed_t, ids_t
        return torch.cat([packed_t, image_latents], dim=1), torch.cat([ids_t, ids_c], dim=0)
    return pipe._pack_latents(noisy.to(dtype), B, C, h, w), pipe._prepare_latent_image_ids(B, h // 2, w // 2, device, dtype)


def loss_weights(weighting, B, C, h, w, area_weights=None, weight_mask=None, unpad_sizes=None):
    """The element weights of the flow-matching loss and the factor that turns their weighted MEAN over [B, C, h, w] into
    the reference's loss (train_denoiser.py:1117-1165):
      weighting [B,1,1,1] (SD3 scheme or sigmas) x area-mask weights (tensor, nearest-resized to the latent; or, for mixed-size
      batches, a list resized to each sample's own latent size and zero-padded) x weight_mask (1 inside each sample's latent);
      loss = mean(w * err^2) without a weight_mask, sum(w * err^2) / weight_mask.sum() / C with one.
    Returns (weights [B,1,h,w] or [B,1,1,1] fp32, scale)."""
    F = torch.nn.functional
    wt = weighting.float()
    if area_weights is not None:
        if isinstance(area_weights, (list, tuple)):
            sizes = unpad_sizes if unpad_sizes is not None else [(h, w)] * len(area_weights)
            aw = [F.interpolate(a.float(), size=tuple(sz), mode="nearest") for a, sz in zip(area_weights, sizes)]
            aw, _ = pad_x_and_mask(aw, max_h=h, max_w=w)
        else:
            aw = area_weights.float()
            if aw.shape[-2:] != (h, w):
                aw = F.interpolate(aw, size=(h, w), mode="nearest")
        wt = wt * aw
    scale = 1.0
    if weight_mask is not None:
        wt = wt * weight_mask.float()
        scale = float(B * C * h * w) / (float(weight_mask.float().sum()) * C)
    return wt, scale


# ------------------------------------------------------------------------------------------------ one optimisation step
def compute_density_for_timestep_sampling(weighting_scheme, batch_size, logit_mean=0.0, logit_std=1.0, mode_scale=1.29,
                                          generator=None, device="cpu"):
    """diffusers.training_utils.compute_density_for_timestep_sampling (SD3 paper, section 3.1): u in (0, 1)."""
    import math
    if weighting_scheme == "logit_normal":
        u = torch.normal(mean=logit_mean, std=logit_std, size=(batch_size,), generator=generator, device=device)
        return torch.sigmoid(u)
    u = torch.rand(size=(batch_size,), generator=generator, device=device)
    if weighting_scheme == "mode":
        u = 1 - u - mode_scale * (torch.cos(math.pi * u / 2) ** 2 - 1 + u)
    return u


def compute_loss_weighting_for_sd3(weighting_scheme, sigmas):
    """diffusers.training_utils.compute_loss_weighting_for_sd3."""
    import math
    if weighting_scheme == "sigma_sqrt":
        return (sigmas ** -2.0).float()
    if weighting_scheme == "cosmap":
        return 2 / (math.pi * (1 - 2 * sigmas + 2 * sigmas ** 2))
    return torch.ones_like(sigmas)


def optimizer_state_bytes(n_params: int, world: int) -> int:
    """Device bytes ShardedAdamW allocates per rank for `n_params` trainable parameters: the full fp32 gradient buffer and
    bf16 flat copy, plus this rank's 1/world slice of the reduced fp32 gradient (world > 1), fp32 master weights and the
    two Adam moments."""
    n = int(n_params)
    return 4 * n + 2 * n + (4 * n // world if world > 1 else 0) + 12 * n // world


def check_optimizer_fits(n_params: int, world: int, device: torch.device) -> None:
    """Refuses, before allocating, a ZeRO-2 optimizer whose per-rank state exceeds the device memory still free (the model
    weights are resident by then), and names the smallest world size whose state would fit."""
    if device.type != "cuda":
        return
    free, _ = torch.cuda.mem_get_info(device)
    need = optimizer_state_bytes(n_params, world)
    if need <= free:
        return
    fits = [w for w in (2, 4, 8, 16, 32, 64) if w > world and optimizer_state_bytes(n_params, w) <= free]
    hint = f"at least {fits[0]} ranks" if fits else "more ranks or fewer trainable parameters"
    raise _lib.B2FError(f"ZeRO-2 state for {n_params / 1e9:.2f} B trainable parameters needs {need / 2**30:.1f} GiB per rank "
                        f"at world size {world}, {free / 2**30:.1f} GiB of device memory is free: use {hint} "
                        "(activation memory comes on top)")


class Stage2Trainer:
    """`train_denoiser.py`'s loop body (:829-1181) on this engine: VAE-encode target and context, flow-matching noising,
    Qwen2.5-VL prefill (frozen) -> MLP2 -> FLUX with block checkpoints, loss, backward, ZeRO-2 AdamW step.

    `tc` / `mc` are the reference's TrainingConfig / ModelConfig (univa/training/configuration_denoise.py)."""

    def __init__(self, model, vae, pipe, tc, mc, empty_pooled, group=None, overlap_comm: bool = True):
        from .scheduler import FlowMatchEulerDiscreteScheduler
        self.model, self.vae, self.pipe, self.tc, self.mc = model, vae, pipe, tc, mc
        self.empty_pooled = empty_pooled                      # [1, 768] CLIP pooled embedding of "" (:795-805)
        den = model.denoise_tower.denoiser
        # which tensors train (train_denoiser.py:513-548): everything is frozen first; `only_tune_mlp2` un-freezes MLP2 alone;
        # otherwise the FLUX components of `flux_train_layer_idx` — None (the schema's default) un-freezes NO FLUX layer, the
        # stage-2 yaml lists all 57 — and, with `with_tune_mlp2`, MLP2
        params = trainable_params(model, layers_to_train=trained_flux_layers(mc), only_img_branch=mc.only_tune_image_branch,
                                  with_tune_mlp2=bool(mc.only_tune_mlp2 or mc.with_tune_mlp2))
        if not params:
            raise _lib.B2FError("nothing to train: set model_config.flux_train_layer_idx, with_tune_mlp2 or only_tune_mlp2 "
                                "(the reference's optimizer would be built over an empty parameter list)")
        if tc.optimizer.lower() != "adamw":
            raise _lib.B2FError(f"optimizer={tc.optimizer!r}: only AdamW is built (the stage yamls of the reference use adamw)")
        if tc.gradient_checkpointing:
            den.enable_gradient_checkpointing()               # always on in this engine: the backward recomputes each block
        world = dist.get_world_size(group) if (dist.is_available() and dist.is_initialized()) else 1
        check_optimizer_fits(sum(p.storage.numel() for p in params), world, params[0].storage.device)
        comm = torch.cuda.Stream() if (overlap_comm and world > 1) else None
        self.opt = ShardedAdamW(params, lr=tc.learning_rate, betas=(tc.adam_beta1, tc.adam_beta2), eps=tc.adam_epsilon,
                                weight_decay=tc.adam_weight_decay, max_grad_norm=tc.max_grad_norm, group=group, comm_stream=comm)
        self.params = params
        self._micro = 0
        self.graph = FluxTrainGraph(model, params, on_block_done=self._block_done if world > 1 else None)
        self.sched = FlowMatchEulerDiscreteScheduler()         # noise_scheduler_copy (:437-440)
        self.global_step = 0
        self.gen = None

    def _block_done(self, bucket):
        # reduce a block's gradients as soon as they are complete, but only on the last micro-batch of an accumulation window
        if (self._micro + 1) % self.tc.gradient_accumulation_steps == 0:
            self.opt.reduce_bucket(bucket)

    def lr_at(self, step: int) -> float:
        """The learning rate of optimizer step `step` (0-based) under diffusers' get_scheduler("constant" |
        "constant_with_warmup" | "linear" | "cosine" | "cosine_with_restarts" | "polynomial") as the reference builds it (:707-716): warm-up and total steps are both
        multiplied by the process count there because accelerate steps the scheduler once per process, so in optimizer steps
        the multiplier is step / warmup during the warm-up (0 for the very first update, as LambdaLR gives) and the named
        decay over max_train_steps after it."""
        import math
        tc = self.tc
        base, warm, total = tc.learning_rate, int(tc.lr_warmup_steps or 0), max(tc.max_train_steps or 1, 1)
        name = tc.lr_scheduler
        if name == "constant":
            return base
        if step < warm:
            return base * step / max(1, warm)
        if name == "constant_with_warmup":
            return base
        prog = (step - warm) / max(1, total - warm)
        if name == "linear":
            return base * max(0.0, 1.0 - prog)
        if name == "cosine":
            return base * max(0.0, 0.5 * (1.0 + math.cos(math.pi * float(tc.lr_num_cycles) * 2.0 * prog)))
        if name == "cosine_with_restarts":
            if prog >= 1.0:
                return 0.0
            return base * max(0.0, 0.5 * (1.0 + math.cos(math.pi * ((float(tc.lr_num_cycles) * prog) % 1.0))))
        if name == "polynomial":                                  # lr_end = 1e-7, power = lr_power (:715)
            lr_end = 1e-7
            if step > total:
                return lr_end
            return (base - lr_end) * (1.0 - prog) ** float(getattr(tc, "lr_power", 1.0)) + lr_end
        raise _lib.B2FError(f"lr_scheduler={name!r} is not built (constant, constant_with_warmup, linear, cosine, "
                            "cosine_with_restarts, polynomial are)")

    @torch.no_grad()
    def _vae_latents(self, image, generator=None):
        # :887-898 — latent_dist.sample(), then (z - shift) * scale
        z = self.vae.encode(image.to(self.vae.dtype)).latent_dist.sample(generator=generator)
        return (z.float() - self.vae.config.shift_factor) * self.vae.config.scaling_factor

    def sample_sigmas(self, bsz, latent_hw, device):
        """(sigmas [B], timesteps [B]) as :939-993."""
        import math
        tc = self.tc
        if tc.discrete_timestep:
            u = compute_density_for_timestep_sampling(tc.weighting_scheme, bsz, tc.logit_mean, tc.logit_std, tc.mode_scale,
                                                      generator=self.gen, device=device)
            n = self.sched.config["num_train_timesteps"]
            idx = (u * n).long().clamp_(max=n - 1)
            sig = torch.linspace(1, n, n, device=device).flip(0) / n   # FlowMatchEulerDiscreteScheduler's table: (N..1) / N
            if not self.sched.config.get("use_dynamic_shifting", True):   # FLUX: dynamic shifting, table left unshifted
                shift = self.sched.config.get("shift", 1.0)
                sig = shift * sig / (1 + (shift - 1) * sig)
            sigmas = sig[idx]
            return sigmas, sigmas * n
        sigmas = torch.sigmoid(torch.randn((bsz,), device=device, dtype=torch.float32, generator=self.gen))
        from .pipeline import calculate_shift
        c = self.sched.config
        mu = calculate_shift((latent_hw[0] * latent_hw[1]) // 4, c["base_image_seq_len"], c["max_image_seq_len"], c["base_shift"],
                             c["max_shift"])
        s = math.exp(mu)
        sigmas = (sigmas * s) / (1 + (s - 1) * sigmas)
        return sigmas, sigmas * 1000.0

    def step(self, batch) -> dict:
        """One micro-batch (and, at the end of an accumulation window, one optimizer step).  batch keys as the reference's
        dataloader: generated_image [B,3,H,W], ref_pixel_values [B,(n,)3,H,W] | None, input_ids, attention_mask,
        pixel_values, image_grid_thw, weights [B,1,h,w] | None."""
        tc, mc = self.tc, self.mc
        dev = self.model.device
        pipe = self.pipe
        gen_img = batch["generated_image"]
        cond = batch.get("ref_pixel_values")
        if cond is not None:
            if cond.ndim == 5:
                cond = cond.view(-1, *cond.shape[2:])
            cond = cond.to(dev, dtype=torch.float32)
        weight_mask = unpad_sizes = None
        if isinstance(gen_img, (list, tuple)):
            # mixed-size batch (:907-916): every target encoded at its own size, latents zero-padded to the largest; the
            # padding is excluded from the loss through weight_mask.  (The reference also builds a token mask and passes it
            # as joint_attention_kwargs, which UnivaDenoiseTower.forward pops and drops (:77): attention sees the padding.)
            if len(gen_img) == 1:
                raise ValueError("a list of target images needs batch_size != 1 (train_denoiser.py:909)")
            unpad = [self._vae_latents(x.to(dev), self.gen) for x in gen_img]
            unpad_sizes = [tuple(x.shape[-2:]) for x in unpad]
            model_input, weight_mask = pad_x_and_mask(unpad, [torch.ones_like(x) for x in unpad])
        else:
            model_input = self._vae_latents(gen_img.to(dev), self.gen)                       # [B,16,h,w] fp32
        B, C, h, w = model_input.shape
        noise = torch.randn(model_input.shape, device=dev, dtype=model_input.dtype, generator=self.gen)
        sigmas, timesteps = self.sample_sigmas(B, (h, w), dev)
        s4 = sigmas.view(B, 1, 1, 1)
        noisy = (1.0 - s4) * model_input + s4 * noise                                       # :995
        packed, img_ids = pack_training_latents(pipe, noisy, cond, dev, torch.bfloat16)
        S_tgt = (h // 2) * (w // 2)
        guidance = torch.full((B,), float(mc.guidance_scale), device=dev)
        if mc.vlm_residual_image_factor:
            raise _lib.B2FError("vlm_residual_image_factor > 0 is not built (0.0 in every stage yaml)")
        with torch.no_grad():
            hidden = self.model.prefill_hidden(batch["input_ids"].to(dev), pixel_values=None if batch.get("pixel_values") is None
                                               else batch["pixel_values"].to(dev), attention_mask=batch["attention_mask"].to(dev),
                                               image_grid_thw=batch.get("image_grid_thw"))
        prefix = batch.get("t5_prompt_embeds")                                              # None when drop_t5_rate = 1
        n_out = S_tgt if (mc.joint_ref_feature and cond is not None) or cond is None else packed.shape[1]
        pred = self.graph.forward(hidden, packed, (timesteps / 1000).to(torch.bfloat16), guidance,
                                  self.empty_pooled.expand(B, -1), img_ids, n_out, prefix_embeds=prefix)
        if pred.shape[1] != S_tgt:
            raise _lib.B2FError("joint_ref_feature=false with a context image compares context tokens with the target "
                                "(the reference would fail in _unpack_latents); set joint_ref_feature: true")
        target = pipe._pack_latents(noise - model_input, B, C, h, w).float().contiguous()   # packing is a permutation
        weighting = sigmas.view(B, 1, 1, 1) if tc.sigmas_as_weight else \
            compute_loss_weighting_for_sd3(tc.weighting_scheme, sigmas).view(B, 1, 1, 1)
        am = batch.get("weights") if tc.mask_weight_type is not None else None
        if am is not None:
            am = [a.to(dev) for a in am] if isinstance(am, (list, tuple)) else am.to(dev)
        wt, wscale = loss_weights(weighting, B, C, h, w, area_weights=am, weight_mask=weight_mask, unpad_sizes=unpad_sizes)
        wts = None
        if wscale != 1.0 or (wt.numel() > 1 and not bool((wt == 1).all())):
            wts = pipe._pack_latents((wt * wscale).expand(B, C, h, w).contiguous(), B, C, h, w).float().contiguous()
        ga = tc.gradient_accumulation_steps
        loss, dpred = flow_matching_loss(pred, target, weight=wts, grad_scale=1.0 / ga)
        if getattr(self, "trace", None) is not None:          # test / debug hook: checksums of the step's intermediates
            cs = lambda t: float(t.double().sum())
            self.trace.append(dict(sigmas=sigmas.tolist(), model_input=cs(model_input), noise=cs(noise), packed=cs(packed),
                                   hidden=cs(hidden), pred=cs(pred), target=cs(target), loss=float(loss),
                                   wts=None if wts is None else cs(wts)))
        self.graph.backward(dpred, accumulate=(self._micro % ga) != 0)
        self._micro += 1
        out = {"loss": loss, "sigmas": sigmas, "stepped": False}
        if self._micro % ga == 0:
            if self.graph.on_block_done is None:
                self.opt.reduce_all()
            lr = self.lr_at(self.global_step)
            out["grad_norm"] = self.opt.step(lr)
            out["lr"] = lr
            out["stepped"] = True
            self.global_step += 1
        return out
