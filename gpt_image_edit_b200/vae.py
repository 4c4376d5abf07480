"""Drop-in for the object the reference uses as `pipe.vae` / `vae` (diffusers `AutoencoderKL` with
the FLUX config; reference univa/utils/flux_pipeline.py:255-258, 609-611, 1128-1129;
train_denoiser.py:428, 887-898).  encode/decode are single C-ABI calls into libb2f
(`b2f_vae_encode` / `b2f_vae_decode`: wgmma implicit-GEMM convs, fused GroupNorm+SiLU passes).

Weights are stored in the layout the kernels consume (OHWI conv weights, fused mid-attention qkv,
padded biases); `state_dict()` / `load_state_dict()` speak the diffusers layout and key names.
"""
from __future__ import annotations

import ctypes as C
from collections import OrderedDict
from types import SimpleNamespace

import torch

from . import _lib
from ._lib import check, ptr, stream_ptr


class VaeConfig(SimpleNamespace):
    def __init__(self, **kw):
        base = dict(in_channels=3, out_channels=3, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
                    latent_channels=16, norm_num_groups=32, scaling_factor=0.3611, shift_factor=0.1159,
                    use_quant_conv=False, use_post_quant_conv=False, mid_block_add_attention=True)
        base.update(kw)
        super().__init__(**base)

    def get(self, k, default=None):
        return getattr(self, k, default)


def _spec(cfg):
    """diffusers name -> ('conv3', O, I) | ('conv1', O, I) | ('lin', O, I) | ('vec', n)."""
    s = OrderedDict()

    def conv3(n, o, i):
        s[n + ".weight"], s[n + ".bias"] = ("conv3", o, i), ("vec", o)

    def norm(n, c):
        s[n + ".weight"], s[n + ".bias"] = ("vec", c), ("vec", c)

    def resnet(n, i, o):
        norm(n + ".norm1", i)
        conv3(n + ".conv1", o, i)
        norm(n + ".norm2", o)
        conv3(n + ".conv2", o, o)
        if i != o:
            s[n + ".conv_shortcut.weight"], s[n + ".conv_shortcut.bias"] = ("conv1", o, i), ("vec", o)

    def mid(n, c):
        resnet(n + ".resnets.0", c, c)
        norm(n + ".attentions.0.group_norm", c)
        for t in ("to_q", "to_k", "to_v", "to_out.0"):
            s[f"{n}.attentions.0.{t}.weight"], s[f"{n}.attentions.0.{t}.bias"] = ("lin", c, c), ("vec", c)
        resnet(n + ".resnets.1", c, c)

    boc = cfg.block_out_channels
    conv3("encoder.conv_in", boc[0], cfg.in_channels)
    ch = boc[0]
    for i, o in enumerate(boc):
        for j in range(cfg.layers_per_block):
            resnet(f"encoder.down_blocks.{i}.resnets.{j}", ch, o)
            ch = o
        if i != len(boc) - 1:
            conv3(f"encoder.down_blocks.{i}.downsamplers.0.conv", o, o)
    mid("encoder.mid_block", boc[-1])
    norm("encoder.conv_norm_out", boc[-1])
    conv3("encoder.conv_out", 2 * cfg.latent_channels, boc[-1])
    rev = list(reversed(boc))
    conv3("decoder.conv_in", rev[0], cfg.latent_channels)
    mid("decoder.mid_block", rev[0])
    ch = rev[0]
    for i, o in enumerate(rev):
        for j in range(cfg.layers_per_block + 1):
            resnet(f"decoder.up_blocks.{i}.resnets.{j}", ch, o)
            ch = o
        if i != len(rev) - 1:
            conv3(f"decoder.up_blocks.{i}.upsamplers.0.conv", o, o)
    norm("decoder.conv_norm_out", rev[-1])
    conv3("decoder.conv_out", cfg.out_channels, rev[-1])
    return s


def stage_shapes(cfg, side: str, h: int, w: int) -> list:
    """(name, C, h, w) of every stage's output in the engine's numbering (b2f_vae_set_stop_stage, include/b2f.h);
    h, w: the image size for the encoder, the latent size for the decoder."""
    boc, L = cfg.block_out_channels, cfg.layers_per_block
    mid = lambda p, c, h, w: [(f"{p}.mid_block.{n}", c, h, w) for n in ("resnets.0", "attentions.0", "resnets.1")]
    if side == "encoder":
        out = [("encoder.conv_in", boc[0], h, w)]
        for i, c in enumerate(boc):
            out += [(f"encoder.down_blocks.{i}.resnets.{j}", c, h, w) for j in range(L)]
            if i != len(boc) - 1:
                h, w = h // 2, w // 2
                out.append((f"encoder.down_blocks.{i}.downsamplers.0", c, h, w))
        return out + mid("encoder", boc[-1], h, w) + [("encoder.conv_out", 2 * cfg.latent_channels, h, w)]
    if side != "decoder":
        raise ValueError(f"side must be 'encoder' or 'decoder', not {side!r}")
    out = [("decoder.conv_in", boc[-1], h, w)] + mid("decoder", boc[-1], h, w)
    for i, c in enumerate(reversed(boc)):
        out += [(f"decoder.up_blocks.{i}.resnets.{j}", c, h, w) for j in range(L + 1)]
        if i != len(boc) - 1:
            h, w = 2 * h, 2 * w
            out.append((f"decoder.up_blocks.{i}.upsamplers.0", c, h, w))
    return out + [("decoder.conv_out", cfg.out_channels, h, w)]


class DiagonalGaussianDistribution:
    """diffusers' latent_dist over the moments the encoder produced (mean | logvar on dim 1)."""

    def __init__(self, moments: torch.Tensor):
        self.parameters = moments
        self.mean, logvar = torch.chunk(moments, 2, dim=1)
        self.logvar = torch.clamp(logvar, -30.0, 20.0)
        self.std = torch.exp(0.5 * self.logvar)

    def mode(self):
        return self.mean

    def sample(self, generator=None):
        from .pipeline import randn_tensor      # diffusers samples through randn_tensor (CPU generators allowed)
        noise = randn_tensor(self.mean.shape, generator=generator, device=self.mean.device, dtype=self.mean.dtype)
        return self.mean + self.std * noise


class B200AutoencoderKL(torch.nn.Module):
    def __init__(self, config: VaeConfig | None = None, device="cuda", **kw):
        super().__init__()
        self.config = config or VaeConfig(**kw)
        cfg = self.config
        dev = torch.device(device)
        if dev.type != "cuda":
            raise _lib.B2FError("B200AutoencoderKL lives on a CUDA device; there is no CPU path")
        self._dev = dev
        self._spec = _spec(cfg)
        self._store: "OrderedDict[str, torch.Tensor]" = OrderedDict()
        z = lambda *shape: torch.zeros(shape, device=dev, dtype=torch.bfloat16)
        for name, sp in self._spec.items():
            if ".attentions.0.to_" in name and ".to_out." not in name:
                continue  # fused below
            if sp[0] == "conv3":
                ipad = 64 if sp[2] < 64 else sp[2]
                self._store[name] = z(sp[1], 3, 3, ipad)
            elif sp[0] in ("conv1", "lin"):
                self._store[name] = z(sp[1], sp[2])
            else:
                self._store[name] = z((sp[1] + 7) // 8 * 8)
        for side in ("encoder", "decoder"):
            c = cfg.block_out_channels[-1]
            self._store[f"{side}.mid_block.attentions.0.qkv.weight"] = z(3 * c, c)
            self._store[f"{side}.mid_block.attentions.0.qkv.bias"] = z(3 * c)
        for k, t in self._store.items():
            self.register_buffer("w__" + k.replace(".", "__"), t, persistent=False)
        boc = cfg.block_out_channels
        ccfg = _lib.VaeCfg((C.c_int * 4)(*boc), cfg.layers_per_block, cfg.latent_channels, cfg.in_channels, cfg.out_channels)
        h = C.c_void_p()
        check(_lib.lib.b2f_vae_create(C.byref(h), C.byref(ccfg)), "b2f_vae_create")
        self._h = h
        for k, t in self._store.items():
            check(_lib.lib.b2f_vae_bind_weight(self._h, k.encode(), ptr(t), t.numel()), f"bind {k}")
        self._ws = None
        self.use_slicing = False

    # diffusers' AutoencoderKL memory options, reached through FluxKontextPipeline.enable_vae_slicing / _tiling
    # (reference flux_pipeline.py:615-646).  Slicing runs one batch item per kernel sequence (same results: every
    # normalisation of the VAE is per item) and bounds the workspace to one image.  Tiling changes the output (overlapping
    # tiles are blended) to fit small memories; with 180 GB of HBM per GPU it is refused rather than approximated.
    def enable_slicing(self):
        self.use_slicing = True

    def disable_slicing(self):
        self.use_slicing = False

    def enable_tiling(self, *a, **k):
        raise _lib.B2FError("tiled VAE encode / decode is not built: a 1024x1024 decode needs < 4 GB of workspace here")

    def disable_tiling(self):
        pass

    def _sliced(self, fn, x):
        """fn over single-item views of x, results concatenated (use_slicing with a batch)."""
        self.use_slicing = False
        try:
            return [fn(x[i:i + 1]) for i in range(x.shape[0])]
        finally:
            self.use_slicing = True

    def __del__(self):
        h = getattr(self, "_h", None)
        if h and _lib is not None and getattr(_lib, "lib", None) is not None:  # not during interpreter teardown
            _lib.lib.b2f_vae_destroy(h)
            self._h = None

    @property
    def dtype(self):
        return torch.bfloat16

    @property
    def device(self):
        return self._dev

    def to(self, *args, **kwargs):
        for a in list(args) + list(kwargs.values()):
            if isinstance(a, (str, torch.device)) and torch.device(a).type != "cuda":
                raise _lib.B2FError("B200AutoencoderKL cannot leave the GPU: there is no CPU path")
        return self

    def storage(self):
        return list(self._store.values())

    # ------------------------------------------------------------------ weights
    def _fused_slot(self, name):
        for i, t in enumerate(("to_q", "to_k", "to_v")):
            tag = f".attentions.0.{t}."
            if tag in name:
                return name.replace(tag, ".attentions.0.qkv."), i
        return None, None

    @torch.no_grad()
    def load_state_dict(self, sd, strict: bool = True, assign: bool = False):
        missing = [k for k in self._spec if k not in sd]
        if strict and missing:
            raise RuntimeError(f"load_state_dict: missing {missing[:5]}...")
        for name, sp in self._spec.items():
            if name not in sd:
                continue
            src = sd[name].to(self._dev, torch.bfloat16)
            fused, slot = self._fused_slot(name)
            if fused is not None:
                c = sp[1]
                self._store[fused][slot * c:(slot + 1) * c].copy_(src)
            elif sp[0] == "conv3":
                dst = self._store[name]
                dst.zero_()
                dst[:, :, :, : sp[2]].copy_(src.permute(0, 2, 3, 1))
            elif sp[0] == "conv1":
                self._store[name].copy_(src.reshape(sp[1], sp[2]))
            elif sp[0] == "lin":
                self._store[name].copy_(src)
            else:
                dst = self._store[name]
                dst.zero_()
                dst[: sp[1]].copy_(src)
        return SimpleNamespace(missing_keys=missing, unexpected_keys=[k for k in sd if k not in self._spec])

    def state_dict(self, *a, **k):
        out = OrderedDict()
        for name, sp in self._spec.items():
            fused, slot = self._fused_slot(name)
            if fused is not None:
                c = sp[1]
                out[name] = self._store[fused][slot * c:(slot + 1) * c]
            elif sp[0] == "conv3":
                out[name] = self._store[name][:, :, :, : sp[2]].permute(0, 3, 1, 2)
            elif sp[0] == "conv1":
                out[name] = self._store[name].view(sp[1], sp[2], 1, 1)
            elif sp[0] == "lin":
                out[name] = self._store[name]
            else:
                out[name] = self._store[name][: sp[1]]
        return out

    @torch.no_grad()
    def randomize_(self, seed: int = 0):
        """Seeded synthetic weights (fan-in scaled so activations stay O(1) through the conv stacks)."""
        g = torch.Generator(device=self._dev).manual_seed(seed)
        sd = {}
        for name, sp in self._spec.items():
            if sp[0] == "conv3":
                t = torch.randn(sp[1], sp[2], 3, 3, device=self._dev, generator=g) * (1.0 / (9 * sp[2])) ** 0.5
            elif sp[0] == "conv1":
                t = torch.randn(sp[1], sp[2], 1, 1, device=self._dev, generator=g) * (1.0 / sp[2]) ** 0.5
            elif sp[0] == "lin":
                t = torch.randn(sp[1], sp[2], device=self._dev, generator=g) * (1.0 / sp[2]) ** 0.5
            elif name.endswith(".weight"):
                t = 1.0 + 0.1 * torch.randn(sp[1], device=self._dev, generator=g)
            else:
                t = 0.05 * torch.randn(sp[1], device=self._dev, generator=g)
            sd[name] = t
        self.load_state_dict(sd)
        return self

    # ------------------------------------------------------------------ compute
    def _workspace(self, N, H, W):
        n = int(_lib.lib.b2f_vae_workspace_bytes(self._h, N, H, W))
        if self._ws is None or self._ws.numel() < n:
            self._ws = torch.empty(n, dtype=torch.uint8, device=self._dev)
        return self._ws, n

    @torch.no_grad()
    def encode(self, x: torch.Tensor, return_dict: bool = True):
        """x: [N,3,H,W] bf16 / fp32 in [-1, 1], or uint8 pixels [N,H,W,3] (PIL / numpy layout): then the reference's
        `(u/255 - 0.5)/0.5` normalisation (cli.py:99-116) runs inside the kernel that feeds encoder.conv_in."""
        if not x.is_cuda or x.dim() != 4 or x.dtype not in (torch.bfloat16, torch.float32, torch.uint8):
            raise _lib.B2FError("vae.encode: CUDA [N,3,H,W] bf16/fp32 tensor or uint8 [N,H,W,3] pixels required")
        x = x.contiguous()
        if self.use_slicing and x.shape[0] > 1:
            mom = torch.cat([d.latent_dist.parameters for d in self._sliced(self.encode, x)], dim=0)
            dist = DiagonalGaussianDistribution(mom)
            return SimpleNamespace(latent_dist=dist) if return_dict else (dist,)
        if x.dtype == torch.uint8:
            N, H, W, C = x.shape
            if C != self.config.in_channels:
                raise _lib.B2FError(f"vae.encode: uint8 input must be [N,H,W,{self.config.in_channels}], got {tuple(x.shape)}")
            kind = 2
        else:
            N, _, H, W = x.shape
            kind = int(x.dtype == torch.float32)
        ws, n = self._workspace(N, H, W)
        mom = torch.empty((N, 2 * self.config.latent_channels, H // 8, W // 8), device=self._dev, dtype=torch.bfloat16)
        check(_lib.lib.b2f_vae_encode(self._h, ptr(x), kind, N, H, W, ptr(mom), ptr(ws), n, stream_ptr()), "b2f_vae_encode")
        dist = DiagonalGaussianDistribution(mom)
        return SimpleNamespace(latent_dist=dist) if return_dict else (dist,)

    @torch.no_grad()
    def decode(self, z: torch.Tensor, return_dict: bool = True, generator=None):
        if not z.is_cuda or z.dim() != 4:
            raise _lib.B2FError("vae.decode: CUDA [N,C,h,w] tensor required")
        z = z.to(torch.bfloat16).contiguous()
        if self.use_slicing and z.shape[0] > 1:
            img = torch.cat([d.sample for d in self._sliced(self.decode, z)], dim=0)
            return SimpleNamespace(sample=img) if return_dict else (img,)
        N, _, h, w = z.shape
        ws, n = self._workspace(N, 8 * h, 8 * w)
        img = torch.empty((N, self.config.out_channels, 8 * h, 8 * w), device=self._dev, dtype=torch.bfloat16)
        check(_lib.lib.b2f_vae_decode(self._h, ptr(z), N, h, w, ptr(img), ptr(ws), n, stream_ptr()), "b2f_vae_decode")
        return SimpleNamespace(sample=img) if return_dict else (img,)

    # ------------------------------------------------------------------ stages (tests)
    @torch.no_grad()
    def stage_output(self, x: torch.Tensor, side: str, stage: int) -> torch.Tensor:
        """The NCHW bf16 activation after stage `stage` (1-based, `stage_shapes` order) of encode(x) or decode(x), run
        through the engine's own code path up to that stage; the last stage is the moments / the image."""
        shapes = stage_shapes(self.config, side, *x.shape[-2:])
        if not 1 <= stage <= len(shapes):
            raise ValueError(f"{side} stage {stage} outside 1..{len(shapes)}")
        if stage == len(shapes):
            return self.encode(x).latent_dist.parameters if side == "encoder" else self.decode(x, return_dict=False)[0]
        check(_lib.lib.b2f_vae_set_stop_stage(self._h, stage), "b2f_vae_set_stop_stage")
        sliced, self.use_slicing = self.use_slicing, False      # one run over the whole batch fills the workspace
        try:
            self.encode(x) if side == "encoder" else self.decode(x)
        finally:
            self.use_slicing = sliced
            check(_lib.lib.b2f_vae_set_stop_stage(self._h, 0), "b2f_vae_set_stop_stage")
        _, c, h, w = shapes[stage - 1]
        n = x.shape[0] * h * w * c
        off = -self._ws.data_ptr() % 256
        act = self._ws[off:off + 2 * n].view(torch.bfloat16).view(x.shape[0], h, w, c)
        return act.permute(0, 3, 1, 2).contiguous()

    @torch.no_grad()
    def decode_u8(self, z: torch.Tensor) -> torch.Tensor:
        """z [N,C,h,w] -> uint8 pixels [N,8h,8w,3]: decode with VaeImageProcessor.postprocess (`(x/2+0.5).clamp(0,1)`,
        `(. * 255).round()`, reference flux_pipeline.py:1130) fused into the epilogue of decoder.conv_out."""
        if not z.is_cuda or z.dim() != 4:
            raise _lib.B2FError("vae.decode_u8: CUDA [N,C,h,w] tensor required")
        z = z.to(torch.bfloat16).contiguous()
        if self.use_slicing and z.shape[0] > 1:
            return torch.cat(self._sliced(self.decode_u8, z), dim=0)
        N, _, h, w = z.shape
        ws, n = self._workspace(N, 8 * h, 8 * w)
        img = torch.empty((N, 8 * h, 8 * w, self.config.out_channels), device=self._dev, dtype=torch.uint8)
        check(_lib.lib.b2f_vae_decode_u8(self._h, ptr(z), N, h, w, ptr(img), ptr(ws), n, stream_ptr()), "b2f_vae_decode_u8")
        return img
