"""FluxKontextPipeline — the sampling loop of the reference (univa/utils/flux_pipeline.py:732-1138),
re-hosted over libb2f components.  Same constructor keywords, `__call__` keywords, static helpers
(`_pack_latents`, `_unpack_latents`, `_prepare_latent_image_ids`, `prepare_latents` — also used by
train_denoiser.py:446-454, 1009-1027) and output type as the reference.

The components are protocol objects exactly as in the reference (SURVEY.md §8b):
  transformer  `B200FluxTransformer2DModel`  (C ABI: b2f_flux_forward)
  scheduler    `FlowMatchEulerDiscreteScheduler` (C ABI: b2f_euler_step)
  vae          object with .encode(x).latent_dist.mode(), .decode(z, return_dict=False)[0], .config
What this file adds over the reference loop, without changing results:
  * the AdaLN modulation of all steps is hoisted into one weight-streaming GEMM before the loop
    (`transformer.prepare_schedule`), when the transformer offers it;
  * the transformer is asked for the target tokens only (the reference slices them afterwards,
    flux_pipeline.py:1078), so the Euler update reads a contiguous tensor.
With the transformer's opt-in first-block cache on (`enable_cache`), results change by design: each call resets the
cache and routes the positive forward as branch "cond", the true-CFG negative forward as "uncond".
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Callable, Optional

import numpy as np
import torch

PREFERRED_KONTEXT_RESOLUTIONS = [
    (672, 1568), (688, 1504), (720, 1456), (752, 1392), (800, 1328), (832, 1248), (880, 1184), (944, 1104),
    (1024, 1024), (1104, 944), (1184, 880), (1248, 832), (1328, 800), (1392, 752), (1456, 720), (1504, 688),
    (1568, 672),
]


def stack_prompt_embeds(embeds):
    """Batch prompt embeddings of different lengths: a list of [1, L_b, D] -> (embeds [B, max L_b, D], mask [B, max L_b]
    int64), each item left-padded with zeros as the Qwen processor pads its prompts.  Pass the pair as prompt_embeds and
    prompt_attention_mask: every item then samples what it samples alone on its own embeddings."""
    if not embeds:
        raise ValueError("stack_prompt_embeds: no embeddings")
    if any(e.dim() != 3 or e.shape[0] != 1 or e.shape[1] < 1 or e.shape[2] != embeds[0].shape[2] for e in embeds):
        raise ValueError(f"stack_prompt_embeds: expected [1, L, D] tensors of one D, got {[tuple(e.shape) for e in embeds]}")
    L = max(e.shape[1] for e in embeds)
    out = embeds[0].new_zeros((len(embeds), L, embeds[0].shape[2]))
    mask = torch.zeros((len(embeds), L), dtype=torch.int64, device=embeds[0].device)
    for b, e in enumerate(embeds):
        out[b, L - e.shape[1]:] = e[0]
        mask[b, L - e.shape[1]:] = 1
    return out, mask


def calculate_shift(image_seq_len, base_seq_len: int = 256, max_seq_len: int = 4096, base_shift: float = 0.5,
                    max_shift: float = 1.15):
    """mu is linear in the number of target tokens through (256, 0.5) and (4096, 1.15) (reference :106-116)."""
    slope = (max_shift - base_shift) / (max_seq_len - base_seq_len)
    return image_seq_len * slope + (base_shift - slope * base_seq_len)


def retrieve_timesteps(scheduler, num_inference_steps=None, device=None, timesteps=None, sigmas=None, **kwargs):
    """Reference :120-176 reduced to the two branches FLUX uses (sigmas= or a plain step count)."""
    if timesteps is not None:
        raise ValueError("custom `timesteps` are not supported by FlowMatchEulerDiscreteScheduler; pass `sigmas`")
    if sigmas is not None:
        scheduler.set_timesteps(sigmas=sigmas, device=device, **kwargs)
    else:
        scheduler.set_timesteps(num_inference_steps, device=device, **kwargs)
    return scheduler.timesteps, len(scheduler.timesteps)


class FluxPipelineOutput(SimpleNamespace):
    pass


def randn_tensor(shape, generator=None, device=None, dtype=None):
    """diffusers.utils.torch_utils.randn_tensor as the reference calls it (flux_pipeline.py:703) [dep-spec]: a CPU
    generator draws on the CPU and the result is moved, a CUDA generator cannot serve a CPU tensor, a list of generators
    (a list of one counts as that one) draws one batch item each."""
    shape = tuple(shape)
    device = torch.device(device) if device is not None else torch.device("cpu")
    rand_device = device
    if generator is not None:
        gen_type = (generator[0] if isinstance(generator, list) else generator).device.type
        if gen_type != device.type and gen_type == "cpu":
            rand_device = torch.device("cpu")
        elif gen_type != device.type and gen_type == "cuda":
            raise ValueError(f"Cannot generate a {device} tensor from a generator of type {gen_type}.")
    if isinstance(generator, list) and len(generator) == 1:
        generator = generator[0]
    if isinstance(generator, list):
        one = (1,) + shape[1:]
        parts = [torch.randn(one, generator=generator[i], device=rand_device, dtype=dtype) for i in range(shape[0])]
        return torch.cat(parts, dim=0).to(device)
    return torch.randn(shape, generator=generator, device=rand_device, dtype=dtype).to(device)


class VaeImageProcessor:
    """diffusers' VaeImageProcessor as the reference pipeline configures and reaches it (`VaeImageProcessor(
    vae_scale_factor=16)`, flux_pipeline.py:259: do_resize, lanczos, do_normalize) [dep-spec, SURVEY.md A.4]:
    `get_default_height_width`, `resize`, `preprocess` for tensors, PIL images, arrays and lists of them, and
    `postprocess` to "pt" / "np" / "pil"."""

    def __init__(self, vae_scale_factor: int = 16):
        self.vae_scale_factor = vae_scale_factor

    @staticmethod
    def _is_pil(x):
        return hasattr(x, "resize") and hasattr(x, "height") and not isinstance(x, (torch.Tensor, np.ndarray))

    def get_default_height_width(self, image, height=None, width=None):
        """(height, width) of the input, floored to a multiple of vae_scale_factor (tensors are [.., H, W], arrays
        [N, H, W, C])."""
        if isinstance(image, list):
            image = image[0]
        if height is None:
            height = image.height if self._is_pil(image) else (image.shape[2] if isinstance(image, torch.Tensor)
                                                               else image.shape[1])
        if width is None:
            width = image.width if self._is_pil(image) else (image.shape[3] if isinstance(image, torch.Tensor)
                                                             else image.shape[2])
        f = self.vae_scale_factor
        return int(height) - int(height) % f, int(width) - int(width) % f

    def resize(self, image, height: int, width: int):
        """PIL: lanczos; tensor: nearest `interpolate`; array: through the tensor path; lists element-wise."""
        if isinstance(image, list):
            return [self.resize(i, height, width) for i in image]
        if self._is_pil(image):
            from PIL import Image
            return image.resize((width, height), resample=Image.LANCZOS)
        if isinstance(image, torch.Tensor):
            if image.shape[-2] == height and image.shape[-1] == width:
                return image                      # nearest interpolation to the same size is the identity
            return torch.nn.functional.interpolate(image, size=(height, width))
        t = torch.from_numpy(image.transpose(0, 3, 1, 2) if image.ndim == 4 else image[..., None].transpose(0, 3, 1, 2))
        t = torch.nn.functional.interpolate(t, size=(height, width))
        return t.cpu().permute(0, 2, 3, 1).float().numpy()

    def preprocess(self, image, height=None, width=None) -> torch.Tensor:
        """-> float tensor [N, 3, H, W] in [-1, 1].  PIL / arrays are scaled from [0, 255] / taken as [0, 1], resized to
        (height, width) (default: their own size floored to the scale factor) and normalised; tensors are resized the
        same way and normalised unless they already hold negative values (then they pass as [-1, 1])."""
        if isinstance(image, torch.Tensor) and image.dim() == 3:
            image = image[None]
        if isinstance(image, np.ndarray) and image.ndim == 3:
            image = image[None]
        if self._is_pil(image) or isinstance(image, (torch.Tensor, np.ndarray)):
            image = [image]
        if not isinstance(image, list) or not image:
            raise ValueError("image must be a PIL image, an array, a tensor or a non-empty list of one of them")
        if self._is_pil(image[0]):
            h, w = self.get_default_height_width(image[0], height, width)
            image = [self.resize(i, h, w) for i in image]
            arr = np.stack([np.array(i).astype(np.float32) / 255.0 for i in image], axis=0)
            if arr.ndim == 3:
                arr = arr[..., None]
            x = torch.from_numpy(arr.transpose(0, 3, 1, 2))
        elif isinstance(image[0], np.ndarray):
            arr = np.concatenate(image, axis=0) if image[0].ndim == 4 else np.stack(image, axis=0)
            if arr.ndim == 3:
                arr = arr[..., None]
            x = torch.from_numpy(arr.transpose(0, 3, 1, 2))
            h, w = self.get_default_height_width(x, height, width)
            x = torch.nn.functional.interpolate(x, size=(h, w))
        else:
            x = image[0] if (len(image) == 1 and image[0].dim() == 4) else \
                (torch.cat(image, dim=0) if image[0].dim() == 4 else torch.stack(image, dim=0))
            h, w = self.get_default_height_width(x, height, width)
            x = self.resize(x, h, w)
        if x.min() < 0:              # already [-1, 1] (diffusers warns and skips the normalisation)
            return x
        return 2.0 * x - 1.0

    @staticmethod
    def postprocess(image: torch.Tensor, output_type: str = "pil"):
        if output_type == "latent":
            return image
        if output_type not in ("pt", "np", "pil"):
            raise ValueError(f"output_type={output_type!r}: one of 'pil', 'np', 'pt', 'latent'")
        img = (image.float() / 2 + 0.5).clamp(0, 1)      # fp32 (diffusers denormalises in the VAE's dtype)
        if output_type == "pt":
            return img
        arr = img.cpu().permute(0, 2, 3, 1).numpy()
        if output_type == "np":
            return arr
        from PIL import Image

        arr8 = (arr * 255).round().astype("uint8")
        return [Image.fromarray(a.squeeze(-1), mode="L") if a.shape[-1] == 1 else Image.fromarray(a) for a in arr8]


class FluxKontextPipeline:
    def __init__(self, transformer, vae=None, scheduler=None, text_encoder=None, tokenizer=None, text_encoder_2=None,
                 tokenizer_2=None, image_encoder=None, feature_extractor=None):
        self.transformer = transformer
        self.vae = vae
        self.scheduler = scheduler
        self.text_encoder, self.tokenizer = text_encoder, tokenizer
        self.text_encoder_2, self.tokenizer_2 = text_encoder_2, tokenizer_2
        self.image_encoder, self.feature_extractor = image_encoder, feature_extractor
        boc = getattr(getattr(vae, "config", None), "block_out_channels", (128, 256, 512, 512))
        self.vae_scale_factor = 2 ** (len(boc) - 1)
        self.latent_channels = getattr(getattr(vae, "config", None), "latent_channels", 16)
        self.image_processor = VaeImageProcessor(vae_scale_factor=self.vae_scale_factor * 2)
        self.tokenizer_max_length = getattr(tokenizer, "model_max_length", 77) if tokenizer is not None else 77
        self.default_sample_size = 128
        self._execution_device = getattr(transformer, "device", torch.device("cuda"))
        self._interrupt = False
        self._guidance_scale = None
        self._joint_attention_kwargs = None
        self._num_timesteps = 0
        self._current_timestep = None

    # read-only views of the running call, as the reference exposes them to step callbacks (flux_pipeline.py:710-728)
    guidance_scale = property(lambda self: self._guidance_scale)
    joint_attention_kwargs = property(lambda self: self._joint_attention_kwargs)
    num_timesteps = property(lambda self: self._num_timesteps)
    current_timestep = property(lambda self: self._current_timestep)
    interrupt = property(lambda self: self._interrupt)

    # VAE memory options (reference :615-646) are forwarded to the VAE object, which must offer them
    def enable_vae_slicing(self):
        self.vae.enable_slicing()

    def disable_vae_slicing(self):
        self.vae.disable_slicing()

    def enable_vae_tiling(self):
        self.vae.enable_tiling()

    def disable_vae_tiling(self):
        self.vae.disable_tiling()

    # LoRA (diffusers FluxLoraLoaderMixin, which the reference's pipeline inherits: flux_pipeline.py:30, 193-195).  Only
    # the transformer takes adapters; each call delegates to the matching B200FluxTransformer2DModel method.
    def load_lora_weights(self, pretrained_model_name_or_path_or_dict, adapter_name=None, weight_name=None, **kw):
        """Load a LoRA (diffusers / PEFT, BFL or kohya layout; a dict or a local .safetensors file) onto the transformer.
        The new adapter joins the active set with weight 1.0; see FluxLoraMixin for the rules."""
        return self.transformer.load_lora_adapter(pretrained_model_name_or_path_or_dict, adapter_name=adapter_name,
                                                  weight_name=weight_name, **kw)

    def set_adapters(self, adapter_names, adapter_weights=None):
        self.transformer.set_adapters(adapter_names, adapter_weights)

    def get_active_adapters(self):
        return self.transformer.get_active_adapters()

    def get_list_adapters(self):
        return self.transformer.get_list_adapters()

    def delete_adapters(self, adapter_names):
        self.transformer.delete_adapters(adapter_names)

    def disable_lora(self):
        self.transformer.disable_lora()

    def enable_lora(self):
        self.transformer.enable_lora()

    def unload_lora_weights(self):
        self.transformer.unload_lora()

    @staticmethod
    def _lora_components(components):
        comps = [components] if isinstance(components, str) else list(components)
        bad = [c for c in comps if c != "transformer"]
        if bad:
            raise ValueError(f"LoRA is supported on the transformer only, not on {bad}")

    def fuse_lora(self, components=("transformer",), lora_scale: float = 1.0, adapter_names=None, **kw):
        self._lora_components(components)
        self.transformer.fuse_lora(lora_scale=lora_scale, adapter_names=adapter_names)

    def unfuse_lora(self, components=("transformer",)):
        self._lora_components(components)
        self.transformer.unfuse_lora()

    @classmethod
    def from_pretrained(cls, flux_path, transformer=None, torch_dtype=torch.bfloat16, **kw):
        """Reference univa/serve/cli.py:64-68.  Builds scheduler + VAE from `flux_path` when a
        checkpoint directory exists (safetensors, diffusers key names); the transformer is always the
        one handed in, as in the reference."""
        from .checkpoint import load_pipeline_components

        from .checkpoint import load_text_encoders

        dev = getattr(transformer, "device", "cuda")
        vae, scheduler = load_pipeline_components(flux_path, device=dev)
        clip, tok, t5, tok2 = load_text_encoders(flux_path, device=dev)
        return cls(transformer=transformer, vae=vae, scheduler=scheduler, text_encoder=clip, tokenizer=tok,
                   text_encoder_2=t5, tokenizer_2=tok2)

    def encode_prompt(self, prompt, prompt_2=None, device=None, num_images_per_prompt: int = 1, prompt_embeds=None,
                      pooled_prompt_embeds=None, max_sequence_length: int = 512, lora_scale=None):
        """(prompt_embeds [B*n, L, 4096], pooled [B*n, 768], text_ids [L, 3]) — reference flux_pipeline.py:361-440:
        `prompt` goes to CLIP (pooled output only), `prompt_2 or prompt` to T5."""
        from .text_encoders import _encode_prompt_with_clip, _encode_prompt_with_t5

        device = device or self._execution_device
        if prompt_embeds is None:
            if self.text_encoder is None or self.text_encoder_2 is None or self.tokenizer is None or self.tokenizer_2 is None:
                raise ValueError("string prompts need text_encoder/tokenizer (CLIP) and text_encoder_2/tokenizer_2 (T5); "
                                 "this pipeline was built without them — pass prompt_embeds + pooled_prompt_embeds")
            prompt = [prompt] if isinstance(prompt, str) else prompt
            prompt_2 = prompt_2 or prompt
            # pooled CLIP vector, copies of a prompt adjacent (`repeat(1, n).view(B*n, -1)`, reference :354-355)
            pooled_prompt_embeds = _encode_prompt_with_clip(self.text_encoder, self.tokenizer, prompt, device=device,
                                                            num_images_per_prompt=1)
            pooled_prompt_embeds = pooled_prompt_embeds.repeat(1, num_images_per_prompt).view(
                len(prompt) * num_images_per_prompt, -1)
            prompt_embeds = _encode_prompt_with_t5(self.text_encoder_2, self.tokenizer_2, max_sequence_length, prompt_2,
                                                   num_images_per_prompt, device)
        dtype = self.text_encoder.dtype if self.text_encoder is not None else self.transformer.dtype
        text_ids = torch.zeros(prompt_embeds.shape[1], 3, device=device, dtype=dtype)
        return prompt_embeds, pooled_prompt_embeds, text_ids

    def to(self, *a, **k):
        for comp in (self.transformer, self.vae):
            if comp is not None and hasattr(comp, "to"):
                comp.to(*a, **k)
        return self

    # ------------------------------------------------------------------ argument validation (reference :490-560)
    _callback_tensor_inputs = ("latents", "prompt_embeds")

    def check_inputs(self, prompt, prompt_2, height, width, negative_prompt=None, negative_prompt_2=None, prompt_embeds=None,
                     negative_prompt_embeds=None, pooled_prompt_embeds=None, negative_pooled_prompt_embeds=None,
                     callback_on_step_end_tensor_inputs=None, max_sequence_length=None):
        """Same rejections, in the same order, as the reference's `check_inputs` (ValueError in every case; a size that
        is not a multiple of 16 only warns there and is floored by the size rule)."""
        cb = callback_on_step_end_tensor_inputs
        bad_cb = [k for k in (cb or ()) if k not in self._callback_tensor_inputs]
        if bad_cb:
            raise ValueError(f"`callback_on_step_end_tensor_inputs` has to be in {list(self._callback_tensor_inputs)}, but found {bad_cb}")
        both = "Please make sure to only forward one of the two."
        rules = [
            (prompt is not None and prompt_embeds is not None, f"Cannot forward both `prompt`: {prompt} and `prompt_embeds`. {both}"),
            (prompt_2 is not None and prompt_embeds is not None, f"Cannot forward both `prompt_2`: {prompt_2} and `prompt_embeds`. {both}"),
            (prompt is None and prompt_embeds is None,
             "Provide either `prompt` or `prompt_embeds`. Cannot leave both `prompt` and `prompt_embeds` undefined."),
            (prompt is not None and not isinstance(prompt, (str, list)), f"`prompt` has to be of type `str` or `list` but is {type(prompt)}"),
            (prompt_2 is not None and not isinstance(prompt_2, (str, list)),
             f"`prompt_2` has to be of type `str` or `list` but is {type(prompt_2)}"),
        ]
        for cond, msg in rules:          # the reference chains these with elif: the first hit wins
            if cond:
                raise ValueError(msg)
        if negative_prompt is not None and negative_prompt_embeds is not None:
            raise ValueError(f"Cannot forward both `negative_prompt`: {negative_prompt} and `negative_prompt_embeds`. {both}")
        if negative_prompt_2 is not None and negative_prompt_embeds is not None:
            raise ValueError(f"Cannot forward both `negative_prompt_2`: {negative_prompt_2} and `negative_prompt_embeds`. {both}")
        if prompt_embeds is not None and pooled_prompt_embeds is None:
            raise ValueError("If `prompt_embeds` are provided, `pooled_prompt_embeds` also have to be passed. Make sure to generate "
                             "`pooled_prompt_embeds` from the same text encoder that was used to generate `prompt_embeds`.")
        if negative_prompt_embeds is not None and negative_pooled_prompt_embeds is None:
            raise ValueError("If `negative_prompt_embeds` are provided, `negative_pooled_prompt_embeds` also have to be passed. Make sure "
                             "to generate `negative_pooled_prompt_embeds` from the same text encoder that was used to generate "
                             "`negative_prompt_embeds`.")
        if max_sequence_length is not None and max_sequence_length > 512:
            raise ValueError(f"`max_sequence_length` cannot be greater than 512 but is {max_sequence_length}")

    # ------------------------------------------------------------------ layout helpers (reference :561-598)
    @staticmethod
    def _prepare_latent_image_ids(batch_size, height, width, device, dtype):
        ids = torch.zeros(height, width, 3)
        ids[..., 1] = ids[..., 1] + torch.arange(height)[:, None]
        ids[..., 2] = ids[..., 2] + torch.arange(width)[None, :]
        return ids.reshape(height * width, 3).to(device=device, dtype=dtype)

    @staticmethod
    def _pack_latents(latents, batch_size, num_channels_latents, height, width):
        """[B,C,h,w] -> [B,(h/2)(w/2),C*4]; inside a token the order is (c, dy, dx)."""
        x = latents.view(batch_size, num_channels_latents, height // 2, 2, width // 2, 2)
        x = x.permute(0, 2, 4, 1, 3, 5)
        return x.reshape(batch_size, (height // 2) * (width // 2), num_channels_latents * 4)

    @staticmethod
    def _unpack_latents(latents, height, width, vae_scale_factor):
        batch_size, _, channels = latents.shape
        height = 2 * (int(height) // (vae_scale_factor * 2))
        width = 2 * (int(width) // (vae_scale_factor * 2))
        x = latents.view(batch_size, height // 2, width // 2, channels // 4, 2, 2)
        x = x.permute(0, 3, 1, 4, 2, 5)
        return x.reshape(batch_size, channels // 4, height, width)

    def _encode_vae_image(self, image, generator=None):
        """Mode of the VAE posterior, shifted and scaled (reference :600-613; with a list of generators the reference
        encodes one batch item per call, kept so that the kernels see the same shapes)."""
        image = image if image.dtype == torch.uint8 else image.to(self.vae.dtype)
        if isinstance(generator, list):
            z = torch.cat([self.vae.encode(image[i:i + 1]).latent_dist.mode() for i in range(image.shape[0])], dim=0)
        else:
            z = self.vae.encode(image).latent_dist.mode()
        return (z - self.vae.config.shift_factor) * self.vae.config.scaling_factor

    def prepare_latents(self, image, batch_size, num_channels_latents, height, width, dtype, device, generator=None,
                        latents=None):
        """Reference :648-708."""
        if isinstance(generator, list) and len(generator) != batch_size:
            raise ValueError(f"got {len(generator)} generators for an effective batch size of {batch_size}")
        height = 2 * (int(height) // (self.vae_scale_factor * 2))
        width = 2 * (int(width) // (self.vae_scale_factor * 2))
        shape = (batch_size, num_channels_latents, height, width)
        image_latents = image_ids = None
        if image is not None:
            if image.dtype == torch.uint8:
                image_latents = self._encode_vae_image(image.to(device), generator)
            else:
                image = image.to(device=device, dtype=dtype)
                image_latents = self._encode_vae_image(image, generator) if image.shape[1] != self.latent_channels else image
            n = image_latents.shape[0]
            if batch_size > n and batch_size % n == 0:
                image_latents = torch.cat([image_latents] * (batch_size // n), dim=0)
            elif batch_size > n:
                raise ValueError(f"Cannot duplicate `image` of batch size {n} to {batch_size} text prompts.")
            ih, iw = image_latents.shape[2:]
            image_latents = self._pack_latents(image_latents, batch_size, num_channels_latents, ih, iw)
            image_ids = self._prepare_latent_image_ids(batch_size, ih // 2, iw // 2, device, dtype)
            image_ids[..., 0] = 1  # context image index
        latent_ids = self._prepare_latent_image_ids(batch_size, height // 2, width // 2, device, dtype)
        if latents is None:
            noise = randn_tensor(shape, generator=generator, device=device, dtype=dtype)
            latents = self._pack_latents(noise, batch_size, num_channels_latents, height, width)
        else:
            # a private copy: the Euler kernel updates the latents in place, the caller's tensor must not change
            latents = latents.to(device=device, dtype=dtype).clone()
        return latents, image_latents, latent_ids, image_ids

    # ------------------------------------------------------------------ sampling (reference :732-1138)
    @torch.no_grad()
    def __call__(self, image=None, prompt=None, prompt_2=None, negative_prompt=None, negative_prompt_2=None,
                 true_cfg_scale: float = 1.0, height: Optional[int] = None, width: Optional[int] = None,
                 num_inference_steps: int = 28, sigmas=None, guidance_scale: float = 3.5,
                 num_images_per_prompt: int = 1, generator=None, latents=None, prompt_embeds=None,
                 pooled_prompt_embeds=None, negative_prompt_embeds=None, negative_pooled_prompt_embeds=None,
                 output_type: str = "pil", return_dict: bool = True, joint_attention_kwargs=None,
                 callback_on_step_end: Optional[Callable] = None, callback_on_step_end_tensor_inputs=("latents",),
                 max_sequence_length: int = 512, max_area: int = 1024 ** 2, _auto_resize: bool = True,
                 ip_adapter_image=None, ip_adapter_image_embeds=None, negative_ip_adapter_image=None,
                 negative_ip_adapter_image_embeds=None, prompt_attention_mask=None, negative_prompt_attention_mask=None):
        """prompt_attention_mask / negative_prompt_attention_mask: optional [batch, L] masks of prompt_embeds /
        negative_prompt_embeds (1 = token, 0 = padding; each row one contiguous run of ones, as stack_prompt_embeds
        builds them) for batches of instructions of different lengths: every item samples what it samples alone on its
        unpadded embeddings (B200FluxTransformer2DModel.forward, encoder_attention_mask)."""
        self._interrupt = False                    # reference :907-910: per-call state
        self._guidance_scale = guidance_scale
        self._joint_attention_kwargs = joint_attention_kwargs
        self._current_timestep = None
        if any(a is not None for a in (ip_adapter_image, ip_adapter_image_embeds, negative_ip_adapter_image,
                                       negative_ip_adapter_image_embeds)):
            # the reference forwards these to an image encoder + IP-adapter attention processors (:441-488, 1024-1050);
            # neither cli.py nor the eval drivers ever pass them, and FLUX-Kontext checkpoints ship no IP-adapter
            raise NotImplementedError("IP-adapter inputs are accepted by the reference's pipeline but not built in this engine")
        self.check_inputs(prompt, prompt_2, height, width, negative_prompt=negative_prompt, negative_prompt_2=negative_prompt_2,
                          prompt_embeds=prompt_embeds, negative_prompt_embeds=negative_prompt_embeds,
                          pooled_prompt_embeds=pooled_prompt_embeds, negative_pooled_prompt_embeds=negative_pooled_prompt_embeds,
                          callback_on_step_end_tensor_inputs=list(callback_on_step_end_tensor_inputs or ()),
                          max_sequence_length=max_sequence_length)
        if prompt_embeds is None:
            # string prompts: CLIP pooled + T5 hidden states through the libb2f encoders (reference :925-944)
            prompt_embeds, pooled_prompt_embeds, _ = self.encode_prompt(
                prompt, prompt_2, device=self._execution_device, num_images_per_prompt=1,
                max_sequence_length=max_sequence_length)
        # true classifier-free guidance (reference :925-957): a second forward on the negative prompt per step
        has_neg_prompt = negative_prompt is not None or (negative_prompt_embeds is not None and
                                                         negative_pooled_prompt_embeds is not None)
        do_true_cfg = true_cfg_scale > 1 and has_neg_prompt
        if negative_prompt_embeds is not None and negative_pooled_prompt_embeds is None:
            raise ValueError("If `negative_prompt_embeds` are provided, `negative_pooled_prompt_embeds` also have to be passed.")
        if do_true_cfg and negative_prompt_embeds is None:
            negative_prompt_embeds, negative_pooled_prompt_embeds, _ = self.encode_prompt(
                negative_prompt, negative_prompt_2, device=self._execution_device, num_images_per_prompt=1,
                max_sequence_length=max_sequence_length)
        height = height or self.default_sample_size * self.vae_scale_factor
        width = width or self.default_sample_size * self.vae_scale_factor
        # size rule: rescale to `max_area` keeping aspect, floor to a multiple of 16 (reference :874-889)
        aspect = width / height
        width = round((max_area * aspect) ** 0.5)
        height = round((max_area / aspect) ** 0.5)
        mult = self.vae_scale_factor * 2
        width, height = width // mult * mult, height // mult * mult

        batch_size = prompt_embeds.shape[0]
        device = self._execution_device
        dtype = prompt_embeds.dtype
        if not do_true_cfg:
            negative_prompt_attention_mask = None
        for m, e, name in ((prompt_attention_mask, prompt_embeds, "prompt_attention_mask"),
                           (negative_prompt_attention_mask, negative_prompt_embeds, "negative_prompt_attention_mask")):
            if m is not None and tuple(m.shape) != tuple(e.shape[:2]):
                raise ValueError(f"{name} has shape {tuple(m.shape)}; its embeddings have {tuple(e.shape[:2])}")
        if num_images_per_prompt != 1:
            prompt_embeds = prompt_embeds.repeat_interleave(num_images_per_prompt, dim=0)
            pooled_prompt_embeds = pooled_prompt_embeds.repeat_interleave(num_images_per_prompt, dim=0)
            if prompt_attention_mask is not None:
                prompt_attention_mask = prompt_attention_mask.repeat_interleave(num_images_per_prompt, dim=0)
            if do_true_cfg:
                negative_prompt_embeds = negative_prompt_embeds.repeat_interleave(num_images_per_prompt, dim=0)
                negative_pooled_prompt_embeds = negative_pooled_prompt_embeds.repeat_interleave(num_images_per_prompt, dim=0)
                if negative_prompt_attention_mask is not None:
                    negative_prompt_attention_mask = negative_prompt_attention_mask.repeat_interleave(
                        num_images_per_prompt, dim=0)
        # the masks go to the transformer as the same tensors every step: it validates and uploads each once per call
        pos_kw = {} if prompt_attention_mask is None else {"encoder_attention_mask": prompt_attention_mask}
        neg_kw = {} if negative_prompt_attention_mask is None else {"encoder_attention_mask": negative_prompt_attention_mask}
        text_ids = torch.zeros(prompt_embeds.shape[1], 3, device=device, dtype=dtype)
        negative_text_ids = torch.zeros(negative_prompt_embeds.shape[1], 3, device=device, dtype=dtype) if do_true_cfg else None

        if isinstance(image, torch.Tensor) and image.dtype == torch.uint8:
            # uint8 pixels [N,H,W,3]: normalised inside the VAE's first kernel; only sizes the pipeline would not
            # resize can take this path (anything else goes through the float preprocess like the reference)
            ih, iw = int(image.shape[1]), int(image.shape[2])
            if _auto_resize or ih % mult or iw % mult:
                image = (((image.cpu().permute(0, 3, 1, 2).float() / 255.0) - 0.5) / 0.5).to(image.device)   # host chain of cli.py:99-116
        if isinstance(image, torch.Tensor) and image.dtype == torch.uint8:
            pass
        elif image is not None and not (isinstance(image, torch.Tensor) and image.size(1) == self.latent_channels):
            ih, iw = self.image_processor.get_default_height_width(image)
            if _auto_resize:
                a = iw / ih
                _, iw, ih = min((abs(a - w / h), w, h) for w, h in PREFERRED_KONTEXT_RESOLUTIONS)
            iw, ih = iw // mult * mult, ih // mult * mult
            image = self.image_processor.preprocess(self.image_processor.resize(image, ih, iw), ih, iw)

        B = batch_size * num_images_per_prompt
        num_channels_latents = self.transformer.config.in_channels // 4
        latents, image_latents, latent_ids, image_ids = self.prepare_latents(
            image, B, num_channels_latents, height, width, dtype, device, generator, latents)
        if image_ids is not None:
            latent_ids = torch.cat([latent_ids, image_ids], dim=0)
        latents = latents.contiguous()

        sig = np.linspace(1.0, 1 / num_inference_steps, num_inference_steps) if sigmas is None else sigmas
        n_tgt = latents.shape[1]
        cfgs = self.scheduler.config
        mu = calculate_shift(n_tgt, cfgs.get("base_image_seq_len", 256), cfgs.get("max_image_seq_len", 4096),
                             cfgs.get("base_shift", 0.5), cfgs.get("max_shift", 1.15))
        timesteps, num_inference_steps = retrieve_timesteps(self.scheduler, num_inference_steps, device, sigmas=sig, mu=mu)
        self._num_timesteps = len(timesteps)

        guidance = None
        if self.transformer.config.guidance_embeds:
            guidance = torch.full([1], guidance_scale, device=device, dtype=torch.float32).expand(B)

        if self._joint_attention_kwargs is None:         # reference :1022-1023
            self._joint_attention_kwargs = {}
        jak = dict(joint_attention_kwargs or {})
        hoist = hasattr(self.transformer, "prepare_schedule")
        if hoist:
            # the loop passes timestep = t.to(dtype) / 1000 (reference :1065-1069): hoist with exactly those values
            sched_kw = {"lora_scale": float(jak["scale"])} if "scale" in jak else {}
            self.transformer.prepare_schedule(timesteps.to(dtype) / 1000, guidance, pooled_prompt_embeds, **sched_kw)
            jak["_b2f_out_rows"] = n_tgt
            # first-block cache: every call starts from a full step; the positive and the true-CFG negative forward
            # each keep their own state
            jak["_b2f_cache_branch"] = "cond"
            if hasattr(self.transformer, "cache_reset"):
                self.transformer.cache_reset()

        self.scheduler.set_begin_index(0)
        for i, t in enumerate(timesteps):
            if self._interrupt:
                continue
            self._current_timestep = t
            x_in = latents if image_latents is None else torch.cat([latents, image_latents], dim=1)
            timestep = t.expand(B).to(latents.dtype)
            if hoist:
                jak["_b2f_schedule_step"] = i
            noise_pred = self.transformer(
                hidden_states=x_in, timestep=timestep / 1000, guidance=guidance, pooled_projections=pooled_prompt_embeds,
                encoder_hidden_states=prompt_embeds, txt_ids=text_ids, img_ids=latent_ids, joint_attention_kwargs=jak,
                return_dict=False, **pos_kw)[0]
            noise_pred = noise_pred[:, :n_tgt]
            if do_true_cfg:
                # the hoisted modulation belongs to the positive pooled vector: the negative forward computes its own
                neg_jak = {k: v for k, v in jak.items() if k != "_b2f_schedule_step"}
                if hoist:
                    neg_jak["_b2f_cache_branch"] = "uncond"
                neg_noise_pred = self.transformer(
                    hidden_states=x_in, timestep=timestep / 1000, guidance=guidance,
                    pooled_projections=negative_pooled_prompt_embeds, encoder_hidden_states=negative_prompt_embeds,
                    txt_ids=negative_text_ids, img_ids=latent_ids, joint_attention_kwargs=neg_jak, return_dict=False,
                    **neg_kw)[0]
                neg_noise_pred = neg_noise_pred[:, :n_tgt]
                noise_pred = neg_noise_pred + true_cfg_scale * (noise_pred - neg_noise_pred)
            latents = self.scheduler.step(noise_pred, t, latents, return_dict=False)[0]
            if callback_on_step_end is not None:
                # the tensors named in callback_on_step_end_tensor_inputs, and what the callback may hand back (:1106-1113)
                avail = {"latents": latents, "prompt_embeds": prompt_embeds}
                out = callback_on_step_end(self, i, t, {k: avail[k] for k in callback_on_step_end_tensor_inputs})
                latents = out.pop("latents", latents)
                prompt_embeds = out.pop("prompt_embeds", prompt_embeds)
        self._current_timestep = None

        if output_type == "latent":
            images = latents
        else:
            z = self._unpack_latents(latents, height, width, self.vae_scale_factor)
            z = (z / self.vae.config.scaling_factor) + self.vae.config.shift_factor
            if output_type in ("pil", "u8") and hasattr(self.vae, "decode_u8"):
                # postprocess fused into the last conv: uint8 [N,H,W,3] straight from the decoder
                u8 = self.vae.decode_u8(z.to(self.vae.dtype))
                if output_type == "u8":
                    images = u8
                else:
                    from PIL import Image
                    images = [Image.fromarray(a) for a in u8.cpu().numpy()]
            else:
                images = self.vae.decode(z.to(self.vae.dtype), return_dict=False)[0]
                images = self.image_processor.postprocess(images, output_type=output_type)
        if not return_dict:
            return (images,)
        return FluxPipelineOutput(images=images)


class FluxPipeline(FluxKontextPipeline):
    """Alias kept by the reference for backward compatibility (flux_pipeline.py:1140)."""
