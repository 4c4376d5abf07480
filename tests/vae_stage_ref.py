"""Float64 references of the FLUX VAE one stage at a time, and the gates that compare a stage's activation with them.

The engine's encode / decode (`b2f_vae_encode` / `b2f_vae_decode`, csrc/vae_model.cu) can stop after any stage of the
numbering in include/b2f.h (`b2f_vae_set_stop_stage`); `B200AutoencoderKL.stage_output` reads that stage's activation.
`stages` lists the same stages as compositions of the oracle's pieces (`vo.resnet_block`, `vo.mid_attention`,
`vo._conv`, `vo._gn`, the downsampler's right / bottom pad, nearest upsampling) in the oracle's op order, so that
chaining them is `vo.encode_moments` / `vo.decode`.  A stage runs in the dtype it is given: float64 for the reference,
bfloat16 for the yardstick (what diffusers in bf16 makes of the same inputs, `F.scaled_dot_product_attention` included
on a GPU).  The stage inputs are the engine's bf16 activations, so an error stays inside the stage that made it.

The gates are train_block_ref's per-tensor rule and per-slice gate at `infer_block_ref.BETA`, over pixel rows (one per
item and position, so a single wrong border pixel shows), channels, and the 32 GroupNorm groups of every item.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

import infer_block_ref as IB
import train_block_ref as TB
from oracle import vae_oracle as vo


def stages(cfg: vo.VaeConfig, side: str) -> list:
    """[(name, prefixes, fn(sd, x) -> y)] of the encoder or the decoder in the engine's stage order; `prefixes` are the
    state-dict prefixes the stage reads."""
    g, boc, L = cfg.norm_num_groups, cfg.block_out_channels, cfg.layers_per_block

    def resnet(n):
        return n, (n + ".",), lambda sd, x: vo.resnet_block(sd, n, x, g)

    def mid(p):
        a = p + ".mid_block.attentions.0"
        return [resnet(p + ".mid_block.resnets.0"), (a, (a + ".",), lambda sd, x: vo.mid_attention(sd, a, x, g)),
                resnet(p + ".mid_block.resnets.1")]

    def tail(p):
        return (p + ".conv_out", (p + ".conv_norm_out.", p + ".conv_out."),
                lambda sd, x: vo._conv(sd, p + ".conv_out", F.silu(vo._gn(sd, p + ".conv_norm_out", x, g))))

    def conv_in(p):
        return p + ".conv_in", (p + ".conv_in.",), lambda sd, x: vo._conv(sd, p + ".conv_in", x)

    def down(i):
        n = f"encoder.down_blocks.{i}.downsamplers.0"
        return n, (n + ".",), lambda sd, x: vo._conv(sd, n + ".conv", F.pad(x, (0, 1, 0, 1)), stride=2, padding=0)

    def up(i):
        n = f"decoder.up_blocks.{i}.upsamplers.0"
        return n, (n + ".",), lambda sd, x: vo._conv(sd, n + ".conv", F.interpolate(x, scale_factor=2.0, mode="nearest"))

    if side == "encoder":
        out = [conv_in("encoder")]
        for i in range(len(boc)):
            out += [resnet(f"encoder.down_blocks.{i}.resnets.{j}") for j in range(L)]
            if i != len(boc) - 1:
                out.append(down(i))
        return out + mid("encoder") + [tail("encoder")]
    out = [conv_in("decoder")] + mid("decoder")
    for i in range(len(boc)):
        out += [resnet(f"decoder.up_blocks.{i}.resnets.{j}") for j in range(L + 1)]
        if i != len(boc) - 1:
            out.append(up(i))
    return out + [tail("decoder")]


def run_stage(sd, stage, x, dtype):
    """one stage of `stages` on x, with its weights and x in `dtype`."""
    _, prefixes, fn = stage
    w = {k: v.to(dtype) for k, v in sd.items() if k.startswith(prefixes)}
    return fn(w, x.to(dtype))


def chain(sd, cfg, side, x, dtype=torch.float64):
    """every stage in turn, each fed the previous one's output: the list of stage outputs."""
    out = []
    for st in stages(cfg, side):
        x = run_stage(sd, st, x, dtype)
        out.append(x)
    return out


def sdpa_backend(q, k, v):
    """the first backend, in torch's default order, that runs F.scaled_dot_product_attention on these inputs."""
    from torch.nn.attention import SDPBackend, sdpa_kernel

    for b in (SDPBackend.FLASH_ATTENTION, SDPBackend.EFFICIENT_ATTENTION, SDPBackend.CUDNN_ATTENTION, SDPBackend.MATH):
        try:
            with sdpa_kernel([b]):
                F.scaled_dot_product_attention(q, k, v)
            return b.name
        except RuntimeError:
            continue
    return "none"


# ------------------------------------------------------------------------------------------------ gates
def _label(N, h, w):
    def f(kind, i):
        if kind == "rows":
            n, p = divmod(i, h * w)
            return f"item {n} pixel (y {p // w}, x {p % w})"
        if kind == "cols":
            return f"channel {i}"
        return f"item {i // 32} group {i % 32}"
    return f


def stage_gates(stage, name, K, R, Y, base=None):
    """gates of an NCHW activation [N, C, h, w]: pixel rows, channels and (C % 32 == 0) the 32 GroupNorm groups of every
    item.  With `base` (the stage input, same shape) the same gates again on the stage's own share K - base."""
    N, C, h, w = K.shape
    pix = lambda t: t.double().permute(0, 2, 3, 1).reshape(-1, C)
    grp = lambda t: t.double().reshape(N * 32, -1)
    lab = _label(N, h, w)
    out = []
    for tag, k, r, y in ((name, K, R, Y),) + (((f"{name} - input", K.double() - base.double(), R.double() - base.double(),
                                                Y.double() - base.double()),) if base is not None else ()):
        out += TB.gate(stage, tag, pix(k), pix(r), pix(y), ("rows", "cols"), lab, beta=IB.BETA)
        if C % 32 == 0:
            out += [c for c in TB.gate(stage, tag, grp(k), grp(r), grp(y), ("chunks",), lab, n_chunks=N * 32,
                                       beta=IB.BETA) if c.kind != "tensor"]
    return out
