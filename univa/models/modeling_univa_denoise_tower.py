"""`UnivaDenoiseTower` — holder of the FLUX denoiser and the MLP2 projector
(reference univa/models/modeling_univa_denoise_tower.py:13-110), over libb2f.

  .denoiser            B200FluxTransformer2DModel  (handed to the pipeline, reference cli.py:64-68)
  .denoise_projector   Linear(in, 3*out) · SiLU · Linear(3*out, out)   ("mlp2x_gelu" — the activation IS
                       SiLU in the reference, :33-43), run as two wgmma GEMMs with the SiLU fused
  .forward(...)        training-time glue (:49-110): concat [vlm embeds, prefix T5 embeds], zero txt_ids,
                       call the denoiser, return sample
State-dict keys: `denoiser.*` and `denoise_projector.{0,2}.{weight,bias}` as in the reference checkpoint
(train_denoiser.py:112-115, 1232).
"""
from __future__ import annotations

import torch

from gpt_image_edit_b200 import ops
from gpt_image_edit_b200._lib import B2FError
from gpt_image_edit_b200.flux_transformer import B200FluxTransformer2DModel, FluxTransformerConfig

from .configuration_univa_denoise_tower import UnivaDenoiseTowerConfig


class DenoiseProjector(torch.nn.Module):
    def __init__(self, in_features: int, out_features: int, device="cuda"):
        super().__init__()
        mk = lambda *s: torch.zeros(s, device=device, dtype=torch.bfloat16)
        self.w0, self.b0 = mk(3 * out_features, in_features), mk(3 * out_features)
        self.w2, self.b2 = mk(out_features, 3 * out_features), mk(out_features)

    def state_dict(self, *a, **k):
        return {"0.weight": self.w0, "0.bias": self.b0, "2.weight": self.w2, "2.bias": self.b2}

    @torch.no_grad()
    def load_state_dict(self, sd, strict=True, assign=False):
        for k, t in self.state_dict().items():
            t.copy_(sd[k])

    @torch.no_grad()
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        h = ops.linear(x.to(torch.bfloat16), self.w0, self.b0, epilogue=ops.EPI_SILU)
        return ops.linear(h, self.w2, self.b2)


class UnivaDenoiseTower(torch.nn.Module):
    config_class = UnivaDenoiseTowerConfig

    def __init__(self, config: UnivaDenoiseTowerConfig, device="cuda"):
        super().__init__()
        self.config = config
        if config.denoiser_type != "flux":
            raise B2FError(f"denoiser_type={config.denoiser_type!r}: only the FLUX denoiser is built (the reference's "
                           "configs never select sd3, scripts/denoiser/*.yaml)")
        self.denoiser = B200FluxTransformer2DModel(FluxTransformerConfig(**(config.denoiser_config or {})), device=device)
        if getattr(config, "denoise_projector_type", None):
            if config.denoise_projector_type != "mlp2x_gelu":
                raise ValueError(f"Unknown denoise_projector_type: {config.denoise_projector_type}")
            self.denoise_projector = DenoiseProjector(config.input_hidden_size, config.output_hidden_size, device)

    def forward(self, hidden_states, timestep, encoder_hidden_states, pooled_projections, **kwargs):
        prefix = kwargs.pop("prefix_prompt_embeds", None)
        if encoder_hidden_states is not None:
            if prefix is not None:
                encoder_hidden_states = torch.cat([encoder_hidden_states, prefix], dim=1)
        else:
            assert prefix is not None
            encoder_hidden_states = prefix
        txt_ids = torch.zeros(encoder_hidden_states.shape[1], 3, device=hidden_states.device, dtype=hidden_states.dtype)
        # the reference pops BOTH of these and forwards neither (its mask assembly is commented out, :79-100; pinned by
        # tests/golden/tower_ref.pt, which was produced by running that file)
        kwargs.pop("joint_attention_kwargs", None)
        kwargs.pop("enc_attention_mask", None)
        kwargs.pop("return_dict", None)
        return self.denoiser(hidden_states=hidden_states, timestep=timestep, encoder_hidden_states=encoder_hidden_states,
                             pooled_projections=pooled_projections, txt_ids=txt_ids, return_dict=False, **kwargs)[0]
