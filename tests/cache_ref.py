"""Host restatement of the first-block cache (include/b2f.h, b2f_flux_forward_cached) over the float64 oracle.

`CachedOracle.forward` is the oracle's FluxTransformer2DModel.forward split where the engine splits it: the head
(embedders + block 0), the rest (blocks 1..), the tail (norm_out + proj_out over the first n_out image rows), with one
`State` per branch.  `decide` and `replay` are the decision rule alone, used to replay the engine's reported distances.
"""
import math
from dataclasses import dataclass, field

import torch
import torch.nn.functional as F

from oracle import flux_oracle as fo


def residual_distance(r_k: torch.Tensor, r_prev: torch.Tensor) -> float:
    """sum |r_k - r_prev| / sum |r_prev| over every element (the batch pooled), in float64."""
    num = (r_k.double() - r_prev.double()).abs().sum().item()
    den = r_prev.double().abs().sum().item()
    return num / den if den > 0 else math.inf


def decide(dist: float, threshold: float, valid: bool = True) -> bool:
    """Hit iff there is a valid state and dist < threshold (strict); NaN or infinite dist is a miss."""
    return bool(valid and math.isfinite(dist) and dist < threshold)


def replay(log: list, threshold: float) -> list:
    """The decisions the policy takes over one branch's log of (step, dist) in call order since a reset: the first call
    has no state; every later call is compared with the last full step, and `dist` is that comparison."""
    return [decide(e["dist"], threshold, valid=e["step"] > 0) for e in log]


@dataclass
class State:
    valid: bool = False
    shape: tuple = ()
    r_prev: torch.Tensor = None
    R: torch.Tensor = None
    full_steps: int = 0


@dataclass
class CachedOracle:
    sd: dict
    cfg: fo.FluxConfig
    threshold: float
    states: dict = field(default_factory=dict)
    log: list = field(default_factory=list)

    def reset(self):
        self.states.clear()
        self.log.clear()

    def forward(self, branch, hidden_states, encoder_hidden_states, pooled, timestep, img_ids, txt_ids, guidance,
                n_out):
        sd, cfg = self.sd, self.cfg
        st = self.states.setdefault(branch, State())
        B, S_img, _ = hidden_states.shape
        S_txt = encoder_hidden_states.shape[1]
        shape = (B, S_img, S_txt, n_out)
        # head: embedders + block 0
        x = fo._lin(sd, "x_embedder", hidden_states)
        t = timestep.to(x.dtype) * 1000
        g = guidance.to(x.dtype) * 1000 if guidance is not None else None
        temb = fo.time_text_embed(sd, cfg, t, g, pooled)
        c = fo._lin(sd, "context_embedder", encoder_hidden_states)
        ids = torch.cat((txt_ids, img_ids), dim=0)
        cos, sin = fo.rope_tables(ids, cfg.axes_dims_rope, cfg.theta)
        x0 = x
        c, x = fo.double_block(sd, 0, cfg, x, c, temb, cos, sin)
        y0 = x
        r_k = y0 - x0
        valid = st.valid and st.shape == shape
        dist = residual_distance(r_k, st.r_prev) if valid else math.nan
        hit = decide(dist, self.threshold, valid)
        if hit:
            h = y0[:, :n_out] + st.R
        else:
            for i in range(1, cfg.num_layers):
                c, x = fo.double_block(sd, i, cfg, x, c, temb, cos, sin)
            hj = torch.cat([c, x], dim=1)
            for i in range(cfg.num_single_layers):
                hj = fo.single_block(sd, i, cfg, hj, temb, cos, sin)
            h = hj[:, S_txt:S_txt + n_out]
            st.R = h - y0[:, :n_out]
            st.r_prev = r_k
            st.shape = shape
            st.valid = True
            st.full_steps += 1
        self.log.append(dict(branch=branch, step=sum(e["branch"] == branch for e in self.log), dist=dist, hit=hit))
        return self.tail(temb, h)

    def tail(self, temb, h):
        e = fo._lin(self.sd, "norm_out.linear", F.silu(temb).to(h.dtype))
        scale, shift = torch.chunk(e, 2, dim=1)
        return fo._lin(self.sd, "proj_out", fo.layer_norm(h) * (1 + scale)[:, None, :] + shift[:, None, :])
