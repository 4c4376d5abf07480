"""ctypes binding of libb2f.so (the C ABI declared in include/b2f.h).

The library is the product: there is no Python/torch fallback for any entry point.  If the
shared object is missing or a call returns a negative code, this module raises.
"""
from __future__ import annotations

import ctypes as C
import os
import re
from pathlib import Path

import torch  # noqa: F401  (loads libcudart.so.12 into the process before libb2f.so)

_HERE = Path(__file__).resolve().parent
LIB_PATH = Path(os.environ["B2F_LIB"]) if os.environ.get("B2F_LIB") else _HERE / "lib" / "libb2f.so"   # override: A/B builds
HEADER_PATH = _HERE.parent / "include" / "b2f.h"


class B2FError(RuntimeError):
    pass


def _load() -> C.CDLL:
    if not LIB_PATH.exists():
        raise B2FError(
            f"{LIB_PATH} not found: build it with `make` (or __graft_entry__.build()). "
            "There is no fallback path."
        )
    return C.CDLL(str(LIB_PATH), mode=getattr(os, "RTLD_NOW", 2))


lib = _load()

_vp, _i64, _i32 = C.c_void_p, C.c_int64, C.c_int

class VaeCfg(C.Structure):
    _fields_ = [("block_out", C.c_int * 4), ("layers_per_block", C.c_int), ("latent_channels", C.c_int),
                ("in_channels", C.c_int), ("out_channels", C.c_int)]


class FluxCfg(C.Structure):
    _fields_ = [(n, C.c_int) for n in (
        "num_heads", "head_dim", "num_double", "num_single", "in_channels", "out_channels",
        "joint_dim", "pooled_dim", "guidance_embeds", "mlp_ratio")]


_SIGNATURES = {
    "b2f_strerror": (C.c_char_p, [_i32]),
    "b2f_version": (_i32, []),
    "b2f_device_info": (_i32, [C.POINTER(_i32), C.POINTER(_i32), C.POINTER(_i32), C.POINTER(C.c_size_t)]),
    "b2f_launch_count": (C.c_uint64, []),
    "b2f_prof_enable": (None, [_i32]),
    "b2f_prof_shapes": (_i32, [C.c_char_p, _i32]),
    "b2f_prof_collect": (_i32, [_i32, C.POINTER(C.c_double), C.POINTER(_i64), C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "b2f_gemm_bf16": (_i32, [_vp, _i64, _i64, _vp, _i64, _vp, _vp, _i64, _i64, _i32, _i32, _i32, _i32, _i32, _vp, _i64, _i64, _vp, _i64, _vp]),
    "b2f_gemm_qkv_norm_rope": (_i32, [_vp, _i64, _i64, _vp, _i64, _vp, _vp, _i64, _i64, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _i32, C.c_float, _i32, _vp, _i64, _i64, _i32, _vp]),
    "b2f_ln_modulate": (_i32, [_vp, _i64, _i64, _vp, _vp, _i64, _vp, _i64, _i64, _i32, _i32, _i32, C.c_float, _i32, _vp, _vp, _vp]),
    "b2f_rmsnorm_rope": (_i32, [_vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, C.c_float, _vp]),
    "b2f_euler_step": (_i32, [_vp, _i64, _vp, _i64, _i64, _i32, C.c_float, _vp]),
    "b2f_silu": (_i32, [_vp, _vp, _i64, _vp]),
    "b2f_temb_sinusoid": (_i32, [_vp, _vp, _i32, _vp]),
    "b2f_temb_combine": (_i32, [_vp, _vp, _vp, _vp, _vp, _i64, _vp]),
    "b2f_rope_tables": (_i32, [_vp, _i32, C.POINTER(_i32), C.c_double, _vp, _vp, _vp]),
    "b2f_rmsnorm": (_i32, [_vp, _i64, _vp, _vp, _i64, _i64, _i32, C.c_float, _vp]),
    "b2f_rope_half": (_i32, [_vp, _i64, _i32, _i32, _vp, _vp, _i32, _i64, _i32, _vp]),
    "b2f_swiglu": (_i32, [_vp, _i64, _vp, _i64, _i64, _i32, _vp]),
    "b2f_move_rows": (_i32, [_vp, _i64, _vp, _i64, _vp, _i64, _i32, _i32, _vp]),
    "b2f_conv3x3": (_i32, [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
    "b2f_groupnorm_silu": (_i32, [_vp, _vp, _vp, _vp, _vp, _i32, _i64, _i32, C.c_float, _i32, _vp]),
    "b2f_upsample2x": (_i32, [_vp, _vp, _i32, _i32, _i32, _i32, _vp]),
    "b2f_nchw_to_nhwc_pad": (_i32, [_vp, _i32, _vp, _i32, _i32, _i32, _i32, _i32, _vp]),
    "b2f_softmax_rows": (_i32, [_vp, _i64, _i32, _i32, C.c_float, _vp]),
    "b2f_transpose_bf16": (_i32, [_vp, _i64, _vp, _i64, _i32, _i32, _vp]),
    "b2f_vae_create": (_i32, [C.POINTER(_vp), _vp]),
    "b2f_vae_destroy": (None, [_vp]),
    "b2f_vae_bind_weight": (_i32, [_vp, C.c_char_p, _vp, _i64]),
    "b2f_vae_workspace_bytes": (C.c_size_t, [_vp, _i32, _i32, _i32]),
    "b2f_vae_encode": (_i32, [_vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, C.c_size_t, _vp]),
    "b2f_vae_decode": (_i32, [_vp, _vp, _i32, _i32, _i32, _vp, _vp, C.c_size_t, _vp]),
    "b2f_vae_decode_u8": (_i32, [_vp, _vp, _i32, _i32, _i32, _vp, _vp, C.c_size_t, _vp]),
    "b2f_flux_create": (_i32, [C.POINTER(_vp), _vp]),
    "b2f_flux_destroy": (None, [_vp]),
    "b2f_flux_bind_weight": (_i32, [_vp, C.c_char_p, _vp, _i64]),
    "b2f_flux_finalize": (_i32, [_vp]),
    "b2f_flux_mod_width": (_i64, [_vp]),
    "b2f_flux_set_rope": (_i32, [_vp, _vp, _vp, _i32]),
    "b2f_flux_workspace_bytes": (C.c_size_t, [_vp, _i32, _i32, _i32]),
    "b2f_flux_temb_workspace_bytes": (C.c_size_t, [_vp, _i32]),
    "b2f_flux_temb": (_i32, [_vp, _vp, _vp, _vp, _i64, _i32, _vp, _vp, _vp, C.c_size_t, _vp]),
    "b2f_flux_modulation": (_i32, [_vp, _vp, _i32, _vp, _vp]),
    "b2f_flux_forward": (_i32, [_vp, _vp, _vp, _vp, _i64, _vp, _i32, _i32, _i32, _i32, _vp, C.c_size_t, _i32, _i32, _vp]),
    "b2f_attention_fwd": (_i32, [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _i32, _i32, _i32, _i32, _i32, _i32, C.c_float, _i32, _vp]),
    "b2f_attention_bias_fwd": (_i32, [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _i32, _i32, _i32, _i32, _i32, _i32, C.c_float, _i32,
                                      _vp, _i64, _i64, _vp]),
    "b2f_geglu": (_i32, [_vp, _i64, _vp, _i64, _i64, _i32, _vp]),
    "b2f_layernorm": (_i32, [_vp, _i64, _vp, _vp, _vp, _i64, _i64, _i32, C.c_float, _vp]),
    "b2f_embed": (_i32, [_vp, _i64, _vp, _vp, _i64, _i32, _vp, _i64, _i64, _i32, _vp]),
    # training step
    "b2f_gemm_dgrad": (_i32, [_vp, _i64, _i64, _vp, _i64, _vp, _i64, _i64, _i32, _i32, _i32, _i32, _i32, _vp, _i64, _i64, _vp]),
    "b2f_gemm_wgrad": (_i32, [_vp, _i64, _i64, _vp, _i64, _i64, _vp, _i64, _i32, _i32, _i32, _i32, _i32, _vp]),
    "b2f_attention_fwd_lse": (_i32, [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _i32, _i32, _i32, _i32, _i32, _i32, C.c_float, _i32,
                                     _vp, _i64, _vp]),
    "b2f_attn_delta": (_i32, [_vp, _i64, _vp, _i64, _vp, _vp, _i32, _i32, _i32, _i32, _vp]),
    "b2f_attention_bwd": (_i32, [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64,
                                 _i32, _i32, _i32, _i32, C.c_float, _vp]),
    "b2f_train_chunks": (_i32, [_i32]),
    "b2f_train_ln_chunks": (_i32, [_i32]),
    "b2f_gate_resid_fwd": (_i32, [_vp, _i64, _i64, _vp, _i64, _i64, _vp, _vp, _i64, _vp, _i64, _i64, _i32, _i32, _i32, _i32, _vp]),
    "b2f_gate_bwd": (_i32, [_vp, _i64, _i64, _vp, _i64, _i64, _vp, _vp, _i64, _vp, _i64, _i64, _vp, _i32, _i32, _i32, _i32, _i32, _vp]),
    "b2f_col_reduce": (_i32, [_vp, _i32, _i32, _vp, _i64, _i32, _i32, _vp]),
    "b2f_ln_modulate_bwd": (_i32, [_vp, _i64, _i64, _vp, _i64, _i64, _vp, _vp, _i64, _vp, _i64, _i64, _vp, _i64, _i64, _vp,
                                   _i32, _i32, _i32, C.c_float, _i32, _i32, _vp]),
    "b2f_rmsnorm_rope_out": (_i32, [_vp, _vp, _i64, _i64, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32,
                                    C.c_float, _vp]),
    "b2f_rmsnorm_rope_bwd": (_i32, [_vp, _vp, _i64, _i64, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32,
                                    _i32, C.c_float, _vp]),
    "b2f_gelu_rows": (_i32, [_vp, _i64, _vp, _i64, _i64, _i32, _vp]),
    "b2f_outer_acc": (_i32, [_vp, _i64, _vp, _i64, _vp, _i64, _i32, _i32, _i32, _i32, _vp]),
    "b2f_mse_loss": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, C.c_float, _vp]),
    "b2f_grad_sumsq": (_i32, [_vp, _i64, _vp, _vp, _i32, _vp]),
    "b2f_clip_coef": (_i32, [_vp, C.c_float, C.c_float, _vp, _vp, _vp]),
    "b2f_adamw_step": (_i32, [_vp, _vp, _vp, _vp, _vp, _i64, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, _i32, _vp, _vp]),
    "b2f_cast_bf16_f32": (_i32, [_vp, _vp, _i64, _i32, _vp]),
    "b2f_blend_bf16": (_i32, [_vp, _vp, C.c_float, C.c_float, _vp, _i64, _vp]),
    "b2f_flux_bind_grad": (_i32, [_vp, C.c_char_p, _vp, _i64]),
    "b2f_flux_train_workspace_bytes": (C.c_size_t, [_vp, _i32, _i32, _i32]),
    "b2f_flux_train_forward": (_i32, [_vp, _vp, _vp, _vp, _i64, _vp, _i32, _i32, _i32, _i32, _vp, C.c_size_t, _vp]),
    "b2f_flux_train_backward": (_i32, [_vp, _vp, _vp, _i64, _vp, _i64, _vp, _i32, _i32, _i32, _i32, _i32, _vp, C.c_size_t,
                                       _i32, _i32, _vp]),
    "b2f_flux_train_debug_dh": (_i32, [_vp, _vp, _i32, _i32, _i32, _vp, _vp]),
}


def declared_symbols() -> list[str]:
    """Every function name include/b2f.h declares (used by the CPU-side export test)."""
    text = HEADER_PATH.read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b2f_[a-z0-9_]+)\s*\(", text)))


def _bind() -> None:
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args


_bind()


def check(code: int, what: str = "") -> None:
    if code != 0:
        msg = lib.b2f_strerror(code).decode()
        raise B2FError(f"libb2f {what} failed: {msg} (code {code})")


def stream_ptr(stream: "torch.cuda.Stream | None" = None) -> int:
    s = stream if stream is not None else torch.cuda.current_stream()
    return int(s.cuda_stream)


def ptr(t: "torch.Tensor | None") -> int | None:
    return None if t is None else int(t.data_ptr())


KERNEL_CLASSES = ("gemm", "attention", "ln_modulate", "rmsnorm_rope", "conv", "other")


def prof_enable(on: bool) -> None:
    lib.b2f_prof_enable(int(on))


def prof_collect() -> dict:
    """{class: dict(ms, launches, flops, bytes)} since the last collect (synchronises the events)."""
    out = {}
    for i, name in enumerate(KERNEL_CLASSES):
        ms, n, fl, by = C.c_double(), _i64(), C.c_double(), C.c_double()
        check(lib.b2f_prof_collect(i, C.byref(ms), C.byref(n), C.byref(fl), C.byref(by)), "b2f_prof_collect")
        out[name] = dict(ms=ms.value, launches=n.value, flops=fl.value, bytes=by.value)
    return out


def prof_shapes() -> list:
    """[(tag, launches, ms, tflops)] per GEMM shape since the last call (call before prof_collect)."""
    buf = C.create_string_buffer(1 << 20)
    n = lib.b2f_prof_shapes(buf, len(buf))
    check(min(n, 0), "b2f_prof_shapes")
    out = []
    for line in buf.value.decode().splitlines():
        tag, cnt, ms, tf = line.split("\t")
        out.append((tag, int(cnt), float(ms), float(tf)))
    return out


def launch_count() -> int:
    return int(lib.b2f_launch_count())
