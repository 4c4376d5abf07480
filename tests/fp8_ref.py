"""References of the FP8 (e4m3) path (include/b2f.h, "FP8 linear layers").

  quant_rows      the row rule, bit-exact: what b2f_quant_fp8_rows and b2f_ln_modulate_fp8 must write;
  linear_fp8_emu / qkv_fp8_emu
                  b2f_gemm_fp8 / b2f_gemm_qkv_norm_rope_fp8: fp64 products of the dequantized operands, then the
                  documented bf16 rounding points through kernel_ref's epilogue emulations, with the accumulation floor
                  max(K * 2^-24, 2^-p) * absref: the FP8 tensor cores keep fewer bits than fp32 in their partial sums,
                  an error that does not grow with K (tests/test_fp8_gpu.py measures p);
  fp8_linears()   a context in which the oracle's block linears (every linear inside a transformer block except the
                  AdaLN ones) quantize their input per token and their weight per output channel, as the engine does
                  with FP8 on; the oracle's forward and infer_block_ref's stage functions then give the FP8 emulation.
"""
from __future__ import annotations

import contextlib
import re

import torch
import torch.nn.functional as F

import kernel_ref as R
from oracle import flux_oracle as fo

E4M3 = torch.float8_e4m3fn
E4M3_MAX = 448.0

# linears of a block that run in FP8: the engine's fused qkv / add_qkv / qkv_mlp are the oracle's q, k, v (, proj_mlp)
BLOCK_LINEAR = re.compile(
    r"^(transformer_blocks\.\d+\.(attn\.(to_q|to_k|to_v|add_q_proj|add_k_proj|add_v_proj|to_out\.0|to_add_out)"
    r"|ff\.net\.(0\.proj|2)|ff_context\.net\.(0\.proj|2))"
    r"|single_transformer_blocks\.\d+\.(attn\.(to_q|to_k|to_v)|proj_mlp|proj_out))$")


def quant_rows(x: torch.Tensor):
    """(q e4m3 [..., K], s fp32 [...]) of the row rule over the last dimension of x (evaluated on x.float())."""
    xf = x.float()
    amax = xf.abs().amax(-1, keepdim=True)
    nz = amax > 0
    # fp32 divisions, tensor by tensor: torch's CUDA division by a Python scalar multiplies by its reciprocal
    c448 = torch.full_like(amax, E4M3_MAX)
    inv = torch.where(nz, c448 / amax, torch.zeros_like(amax))
    s = torch.where(nz, amax / c448, torch.ones_like(amax))
    q = (xf * inv).clamp(-E4M3_MAX, E4M3_MAX).to(E4M3)
    q = torch.where(nz, q.float(), torch.zeros_like(xf)).to(E4M3)   # an all-zero row is +0 throughout
    return q, s.squeeze(-1)


def dequant(q: torch.Tensor, s: torch.Tensor, dtype=torch.float64) -> torch.Tensor:
    return q.to(dtype) * s.to(dtype)[..., None]


def fake_quant(x: torch.Tensor) -> torch.Tensor:
    """x through the row rule and back, in x's dtype."""
    q, s = quant_rows(x)
    return dequant(q, s, x.dtype)


@contextlib.contextmanager
def _acc_floor(p: float):
    """kernel_ref's accumulation floor K * 2^-24 * absref, at least 2^-p * absref."""
    old = R.acc_floor
    R.acc_floor = lambda K, absref: max(K * R.U32, 2.0 ** -p) * R.d64(absref)
    try:
        yield
    finally:
        R.acc_floor = old


def linear_fp8_emu(xq, xs, wq, ws, b=None, epi=R.EPI_BIAS, *, p: float, resid=None, gate=None):
    """(emu, floor, math) of b2f_gemm_fp8.  The dequantized products differ from acc * fp32(sa * sw) only by the
    rounding of sa * sw to fp32 (2^-24 relative), which the floor covers."""
    with _acc_floor(p):
        return R.linear_emu(dequant(xq, xs), dequant(wq, ws), b, epi, resid=resid, gate=gate)


def qkv_fp8_emu(xq, xs, wq, ws, b, nw_q, nw_k, cos, sin, *, p: float, rope_row0=0, n_extra=0, epi_extra=R.EPI_BIAS):
    """(emu, floor, math) of b2f_gemm_qkv_norm_rope_fp8."""
    with _acc_floor(p):
        return R.qkv_norm_rope_emu(dequant(xq, xs), dequant(wq, ws), b, nw_q, nw_k, cos, sin, rope_row0=rope_row0,
                                   n_extra=n_extra, epi_extra=epi_extra)


@contextlib.contextmanager
def fp8_linears():
    """The oracle with its block linears in FP8: y = fake_quant(x) fake_quant(W)^T + b in x's dtype."""
    old = fo._lin

    def lin(sd, name, x):
        if not BLOCK_LINEAR.match(name):
            return old(sd, name, x)
        w = sd[name + ".weight"]
        return F.linear(fake_quant(x), fake_quant(w).to(x.dtype), sd.get(name + ".bias"))

    fo._lin = lin
    try:
        yield
    finally:
        fo._lin = old
