"""References of unfused LoRA on the FP8 linears (include/b2f.h, b2f_gemm_fp8_lora).

  down_emu           T = bf16(fp32(x Acat^T) * fp32(colscale * cs_mul)): the bf16 down projection on the linear's bf16
                     input, as lora_ref / test_lora_gpu state it
  linear_fp8_lora_emu / qkv_fp8_lora_emu
                     b2f_gemm_fp8_lora / b2f_gemm_qkv_norm_rope_fp8_lora: fp64 products of the dequantized e4m3 operands
                     plus T Bcat^T with T as given (bf16), then kernel_ref's epilogue emulations, with fp8_ref's
                     accumulation floor max(K * 2^-24, 2^-p) * absref over the whole contraction
  fp8_lora_linears   the oracle with its block linears in FP8 (fp8_ref.fp8_linears) and PEFT-style unfused adapters on
                     every linear (lora_ref.peft_linear) that see the unquantized input x
"""
from __future__ import annotations

import contextlib

import torch

import fp8_ref as Q
import kernel_ref as R
import lora_ref as LR


def down_emu(x, acat, colscale, cs_mul: float = 1.0):
    """fp64 values of T (bf16) for x [..., K], acat [r_pad, K], colscale fp32 [r_pad]."""
    s_eff = (colscale.float() * cs_mul).double()   # fp32(colscale * cs_mul), as the kernel forms it
    return R.bf16r(R.linear_math(x, acat) * s_eff)


def _cat(xq, xs, wq, ws, t, bcat):
    return torch.cat([Q.dequant(xq, xs), R.d64(t)], -1), torch.cat([Q.dequant(wq, ws), R.d64(bcat)], -1)


def linear_fp8_lora_emu(xq, xs, wq, ws, t, bcat, b=None, epi=R.EPI_BIAS, *, p: float, resid=None, gate=None):
    """(emu, floor, math) of b2f_gemm_fp8_lora.  The kernel scales its e4m3 accumulator by fp32(sa * sw) (one more
    fp32 rounding than the fp64 products of the dequantized operands), which the floor covers."""
    x, w = _cat(xq, xs, wq, ws, t, bcat)
    with Q._acc_floor(p):
        return R.linear_emu(x, w, b, epi, resid=resid, gate=gate)


def qkv_fp8_lora_emu(xq, xs, wq, ws, t, bcat, b, nw_q, nw_k, cos, sin, *, p: float, rope_row0=0, n_extra=0,
                     epi_extra=R.EPI_BIAS):
    """(emu, floor, math) of b2f_gemm_qkv_norm_rope_fp8_lora."""
    x, w = _cat(xq, xs, wq, ws, t, bcat)
    with Q._acc_floor(p):
        return R.qkv_norm_rope_emu(x, w, b, nw_q, nw_k, cos, sin, rope_row0=rope_row0, n_extra=n_extra,
                                   epi_extra=epi_extra)


@contextlib.contextmanager
def fp8_lora_linears(loras):
    """fp8_linears() with the adapters of lora_ref.peft_linear(loras) added on top: a block linear gives
    fake_quant(x) fake_quant(W)^T + b + sum s * alpha/r * (x A^T) B^T, every other linear its unquantized PEFT form."""
    with Q.fp8_linears(), LR.peft_linear(loras):
        yield
