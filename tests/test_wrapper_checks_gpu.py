"""The host wrappers of ops.py / train_ops.py against a recording stand-in for libb2f: no kernel launches in this file.

libb2f sees pointers and pitches only, so an operand of the wrong shape, dtype or device would be read or written past
its end on the GPU.  Every malformed operand below must raise B2FError before any libb2f call is made, while the same
call with well-formed operands goes through.  The well-formed calls further down pin the exact argument tuple each
wrapper passes, written out in include/b2f.h's order.  The GPU is needed only to allocate CUDA tensors.
"""
import importlib

import pytest
import torch

pytestmark = pytest.mark.gpu

bf16, f32, E4M3 = torch.bfloat16, torch.float32, torch.float8_e4m3fn
B, M, K, N, R = 2, 5, 16, 24, 64          # GEMMs: batch, rows, k, n, LoRA r_pad
D, E = 128, 256                           # fused QKV: d_model, n_extra
NW = 3 * D + E                            # its weight rows
S, H = 130, 2                             # attention: tokens, heads of 128
EPI_GELU_TANH, EPI_GATE_RESID, EPI_RESID, EPI_DGELU = 1, 3, 4, 8


def _t(*shape, dtype=bf16):
    return torch.zeros(shape, device="cuda", dtype=dtype)


def _cpu(*shape, dtype=bf16):
    return torch.zeros(shape, dtype=dtype)


class _Recorder:
    """Stands in for libb2f: each b2f_* call is recorded as (name, args) and returns 0."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if not name.startswith("b2f_"):
            raise AttributeError(name)
        return lambda *args: self.calls.append((name, args)) or 0


@pytest.fixture
def rec(monkeypatch):
    from gpt_image_edit_b200 import _lib

    r = _Recorder()
    monkeypatch.setattr(_lib, "lib", r)
    return r


# ---------------------------------------------------------------------------------------------------- malformed operands
# wrapper -> (module, well-formed keyword arguments, [(case, replacement arguments)]); each case breaks one rule.
def _epi_ok():
    return dict(bias=_t(N), epilogue=EPI_GATE_RESID, out=_t(B, M, N), resid=_t(B, M, N), gate=_t(B, N))


EPI_BAD = [
    ("bias fp32", lambda: dict(bias=_t(N, dtype=f32))),
    ("bias on the CPU", lambda: dict(bias=_cpu(N))),
    ("bias [N - 8]", lambda: dict(bias=_t(N - 8))),
    ("out fp32", lambda: dict(out=_t(B, M, N, dtype=f32))),
    ("out rows M - 1", lambda: dict(out=_t(B, M - 1, N))),
    ("out columns N - 8", lambda: dict(out=_t(B, M, N - 8))),
    ("out batch 1", lambda: dict(out=_t(1, M, N))),
    ("resid on the CPU", lambda: dict(resid=_cpu(B, M, N))),
    ("resid rows M - 1", lambda: dict(resid=_t(B, M - 1, N))),
    ("resid columns N - 8", lambda: dict(resid=_t(B, M, N - 8))),
    ("RESID without resid", lambda: dict(epilogue=EPI_RESID, resid=None)),
    ("gate fp32", lambda: dict(gate=_t(B, N, dtype=f32))),
    ("gate [B, N - 8]", lambda: dict(gate=_t(B, N - 8))),
    ("gate [N - 8]", lambda: dict(gate=_t(N - 8))),
    ("gate [B + 1, N]", lambda: dict(gate=_t(B + 1, N))),
]


def _w_bad(name, rows, dtype):
    return [(f"{name} [.., K + 8]", lambda: {name: _t(rows, K + 8, dtype=dtype)}),
            (f"{name} on the CPU", lambda: {name: _cpu(rows, K, dtype=dtype)}),
            (f"{name} fp32", lambda: {name: _t(rows, K, dtype=f32)})]


def _lora_ok(n):
    return dict(t=_t(B, M, R), bcat=_t(n, R))


def _lora_bad(n):
    return [("t on the CPU", lambda: dict(t=_cpu(B, M, R))),
            ("t rows M - 1", lambda: dict(t=_t(B, M - 1, R))),
            ("t batch 1", lambda: dict(t=_t(1, M, R))),
            ("t columns != bcat's", lambda: dict(t=_t(B, M, R + 64))),
            ("bcat fp32", lambda: dict(bcat=_t(n, R, dtype=f32))),
            ("bcat rows - 8", lambda: dict(bcat=_t(n - 8, R)))]


def _qkv_ok():
    return dict(bias=_t(NW), cos=_t(M + 3, 128, dtype=f32), sin=_t(M + 3, 128, dtype=f32), rope_row0=3,
                out=_t(B, M, 3 * D), out_extra=_t(B, M, E), epi_extra=EPI_GELU_TANH)


def _qkv_bad(w, nq, nk, dtype):
    return _w_bad(w, NW, dtype) + [
        ("weight rows - n_extra not a multiple of 3", lambda: {w: _t(NW + 8, K, dtype=dtype), "bias": _t(NW + 8)}),
        ("bias fp32", lambda: dict(bias=_t(NW, dtype=f32))),
        ("bias on the CPU", lambda: dict(bias=_cpu(NW))),
        ("bias [3 d]", lambda: dict(bias=_t(3 * D))),
        (f"{nq} fp32", lambda: {nq: _t(128, dtype=f32)}),
        (f"{nq} on the CPU", lambda: {nq: _cpu(128)}),
        (f"{nk} [64]", lambda: {nk: _t(64)}),
        ("cos/sin rows < rope_row0 + M", lambda: dict(cos=_t(M + 2, 128, dtype=f32), sin=_t(M + 2, 128, dtype=f32))),
        ("sin rows != cos rows", lambda: dict(sin=_t(M + 4, 128, dtype=f32))),
        ("cos bf16", lambda: dict(cos=_t(M + 3, 128))),
        ("cos/sin [.., 64]", lambda: dict(cos=_t(M + 3, 64, dtype=f32), sin=_t(M + 3, 64, dtype=f32))),
        ("out rows M - 1", lambda: dict(out=_t(B, M - 1, 3 * D))),
        ("out fp32", lambda: dict(out=_t(B, M, 3 * D, dtype=f32))),
        ("out_extra fp32", lambda: dict(out_extra=_t(B, M, E, dtype=f32))),
        ("out_extra on the CPU", lambda: dict(out_extra=_cpu(B, M, E))),
        ("out_extra rows M - 1", lambda: dict(out_extra=_t(B, M - 1, E))),
    ]


def _bf16_x():
    return dict(x=_t(B, M, K))


def _fp8_x():
    return dict(xq=_t(B, M, K, dtype=E4M3), x_scale=_t(B, M, dtype=f32))


def _fp8_w(n):
    return dict(wq=_t(n, K, dtype=E4M3), w_scale=_t(n, dtype=f32))


def _attn_ok():
    return dict(q=_t(B, S, H, 128), k=_t(B, S, H, 128), v=_t(B, S, H, 128), out=_t(B, S, H * 128))


ATTN_OUT_BAD = [
    ("out fp32", lambda: dict(out=_t(B, S, H * 128, dtype=f32))),
    ("out on the CPU", lambda: dict(out=_cpu(B, S, H * 128))),
    ("out rows S - 1", lambda: dict(out=_t(B, S - 1, H * 128))),
    ("out batch 1", lambda: dict(out=_t(1, S, H * 128))),
    ("out columns H * 128 - 8", lambda: dict(out=_t(B, S, H * 128 - 8))),
    ("out [B, S, H, 64]", lambda: dict(out=_t(B, S, H, 64))),
    ("out batch stride S + 2 rows", lambda: dict(out=_t(B, S + 2, H * 128)[:, :S])),
]


def _bwd_ok():
    return dict(q=_t(B, S, H, 128), k=_t(B, S, H, 128), v=_t(B, S, H, 128), o=_t(B, S, H * 128),
                dout=_t(B, S, H * 128), lse=_t(B, H, 256, dtype=f32), dq=_t(B, S, H, 128), dk=_t(B, S, H, 128),
                dv=_t(B, S, H, 128))


def _fp8_bufs():
    return dict(q8=_t(B, S, H, 128, dtype=E4M3), k8=_t(B, S, H, 128, dtype=E4M3), sq=_t(B, H, dtype=f32),
                sk=_t(B, H, dtype=f32), v8t=_t(B, H, 128, 256, dtype=E4M3), sv=_t(B, H, 128, dtype=f32))


TABLE = {
    "linear": ("ops", lambda: _bf16_x() | dict(weight=_t(N, K)) | _epi_ok(), EPI_BAD + _w_bad("weight", N, bf16)),
    "linear_lora": ("ops", lambda: _bf16_x() | dict(weight=_t(N, K)) | _epi_ok() | _lora_ok(N),
                    EPI_BAD + _w_bad("weight", N, bf16) + _lora_bad(N)),
    "linear_fp8": ("ops", lambda: _fp8_x() | _fp8_w(N) | _epi_ok(), EPI_BAD + _w_bad("wq", N, E4M3)),
    "linear_fp8_lora": ("ops", lambda: _fp8_x() | _fp8_w(N) | _epi_ok() | _lora_ok(N),
                        EPI_BAD + _w_bad("wq", N, E4M3) + _lora_bad(N)),
    "linear_qkv_norm_rope": ("ops", lambda: _bf16_x() | dict(weight=_t(NW, K), wq=_t(128), wk=_t(128)) | _qkv_ok(),
                             _qkv_bad("weight", "wq", "wk", bf16)),
    "linear_qkv_norm_rope_lora": ("ops", lambda: _bf16_x() | dict(weight=_t(NW, K), wq=_t(128), wk=_t(128)) | _qkv_ok()
                                  | _lora_ok(NW), _qkv_bad("weight", "wq", "wk", bf16) + _lora_bad(NW)),
    "linear_qkv_norm_rope_fp8": ("ops", lambda: _fp8_x() | _fp8_w(NW) | dict(nq=_t(128), nk=_t(128)) | _qkv_ok(),
                                 _qkv_bad("wq", "nq", "nk", E4M3)),
    "linear_qkv_norm_rope_fp8_lora": ("ops", lambda: _fp8_x() | _fp8_w(NW) | dict(nq=_t(128), nk=_t(128)) | _qkv_ok()
                                      | _lora_ok(NW), _qkv_bad("wq", "nq", "nk", E4M3) + _lora_bad(NW)),
    "lora_down": ("ops", lambda: _bf16_x() | dict(acat=_t(R, K), colscale=_t(R, dtype=f32), out=_t(B, M, R)), [
        ("acat [.., K + 8]", lambda: dict(acat=_t(R, K + 8))),
        ("colscale [r_pad - 8]", lambda: dict(colscale=_t(R - 8, dtype=f32))),
        ("out fp32", lambda: dict(out=_t(B, M, R, dtype=f32))),
        ("out on the CPU", lambda: dict(out=_cpu(B, M, R))),
        ("out rows M - 1", lambda: dict(out=_t(B, M - 1, R))),
        ("out columns r_pad - 8", lambda: dict(out=_t(B, M, R - 8))),
    ]),
    "linear_dgrad": ("train_ops", lambda: dict(dy=_t(B, M, K), weight=_t(K, N), epilogue=EPI_DGELU, aux=_t(B, M, N),
                                               out=_t(B, M, N)), [
        ("out fp32", lambda: dict(out=_t(B, M, N, dtype=f32))),
        ("out rows M - 1", lambda: dict(out=_t(B, M - 1, N))),
        ("out columns N - 8", lambda: dict(out=_t(B, M, N - 8))),
        ("aux rows M - 1", lambda: dict(aux=_t(B, M - 1, N))),
        ("aux columns N - 8", lambda: dict(aux=_t(B, M, N - 8))),
        ("aux batch 1", lambda: dict(aux=_t(1, M, N))),
    ]),
    "linear_wgrad": ("train_ops", lambda: dict(dy=_t(B, M, N), x=_t(B, M, K), out=_t(N, K, dtype=f32),
                                               accumulate=True), [
        ("out bf16", lambda: dict(out=_t(N, K))),
        ("out [N, K - 8]", lambda: dict(out=_t(N, K - 8, dtype=f32))),
        ("out [N - 8, K]", lambda: dict(out=_t(N - 8, K, dtype=f32))),
        ("out [N * K]", lambda: dict(out=_t(N * K, dtype=f32))),
    ]),
    "attention": ("ops", _attn_ok, ATTN_OUT_BAD + [
        ("q heads not contiguous", lambda: dict(q=_t(B, S, H, 256)[..., :128])),
        ("v rows S - 1", lambda: dict(v=_t(B, S - 1, H, 128))),
        ("k, v batch 1", lambda: dict(k=_t(1, S, H, 128), v=_t(1, S, H, 128))),
    ]),
    "attention_fwd_lse": ("train_ops", _attn_ok, ATTN_OUT_BAD + [
        ("k batch stride S + 2 rows", lambda: dict(k=_t(B, S + 2, H, 128)[:, :S])),
        ("v rows S - 1", lambda: dict(v=_t(B, S - 1, H, 128))),
    ]),
    "attention_bwd": ("train_ops", _bwd_ok, [
        ("k rows S - 1", lambda: dict(k=_t(B, S - 1, H, 128), v=_t(B, S - 1, H, 128))),
        ("o on the CPU", lambda: dict(o=_cpu(B, S, H * 128))),
        ("o rows S - 1", lambda: dict(o=_t(B, S - 1, H * 128))),
        ("o columns H * 128 - 8", lambda: dict(o=_t(B, S, H * 128 - 8))),
        ("dout rows S - 1", lambda: dict(dout=_t(B, S - 1, H * 128))),
        ("dout batch stride S + 2 rows", lambda: dict(dout=_t(B, S + 2, H * 128)[:, :S])),
        ("lse bf16", lambda: dict(lse=_t(B, H, 256))),
        ("lse S_pad < S", lambda: dict(lse=_t(B, H, 128, dtype=f32))),
        ("lse S_pad not a multiple of 128", lambda: dict(lse=_t(B, H, 200, dtype=f32))),
        ("lse heads H + 1", lambda: dict(lse=_t(B, H + 1, 256, dtype=f32))),
        ("lse batch 1", lambda: dict(lse=_t(1, H, 256, dtype=f32))),
        ("lse not contiguous", lambda: dict(lse=_t(B, H, 512, dtype=f32)[..., :256])),
        ("dq heads not contiguous", lambda: dict(dq=_t(B, S, H, 256)[..., :128])),
        ("dq rows S - 1", lambda: dict(dq=_t(B, S - 1, H, 128))),
        ("dk heads H + 1", lambda: dict(dk=_t(B, S, H + 1, 128))),
        ("dv rows S - 1", lambda: dict(dv=_t(B, S - 1, H, 128))),
    ]),
    "attn_quant_fp8": ("ops", lambda: {n: t for n, t in _attn_ok().items() if n != "out"} | _fp8_bufs(), [
        ("k, v rows S - 1", lambda: dict(k=_t(B, S - 1, H, 128), v=_t(B, S - 1, H, 128))),
        ("v heads H + 1", lambda: dict(v=_t(B, S, H + 1, 128))),
        ("sv [B, H, 64]", lambda: dict(sv=_t(B, H, 64, dtype=f32))),
    ]),
    "attention_fp8": ("ops", lambda: _fp8_bufs() | dict(out=_t(B, S, H * 128)), ATTN_OUT_BAD),
}
CASES = [(w, case) for w, (_, _, bad) in TABLE.items() for case, _ in bad]


@pytest.mark.parametrize("wrapper,case", CASES, ids=[f"{w}: {c}" for w, c in CASES])
def test_malformed_operand_refused_before_libb2f(rec, wrapper, case):
    from gpt_image_edit_b200 import _lib

    module, ok, bad = TABLE[wrapper]
    fn = getattr(importlib.import_module(f"gpt_image_edit_b200.{module}"), wrapper)
    fn(**ok())
    assert rec.calls, "the well-formed call did not reach libb2f"
    rec.calls.clear()
    with pytest.raises(_lib.B2FError):
        fn(**(ok() | dict(bad)[case]()))
    assert rec.calls == [], f"{case}: reached {rec.calls[0][0]}"


# ---------------------------------------------------------------------------------------------------- argument tuples
def _p(t):
    return t.data_ptr()


def _one_call(rec, name):
    assert [c[0] for c in rec.calls] == [name]
    return rec.calls[0][1]


def _st():
    return int(torch.cuda.current_stream().cuda_stream)


def test_args_gemm_bf16_batched_strided_views_1d_gate(rec):
    from gpt_image_edit_b200 import ops

    xa, oa, ra = _t(B, M + 4, 32), _t(B, M + 3, 40), _t(B, M + 1, 48)
    x, out, resid = xa[:, 2:2 + M, :K], oa[:, 1:1 + M, 8:8 + N], ra[:, :M, :N]
    w, bias, gate = _t(N, K), _t(N), _t(N)
    assert ops.linear(x, w, bias, epilogue=EPI_GATE_RESID, out=out, resid=resid, gate=gate) is out
    assert _one_call(rec, "b2f_gemm_bf16") == (
        _p(x), 32, (M + 4) * 32, _p(w), K, _p(bias), _p(out), 40, (M + 3) * 40, B, M, N, K,
        EPI_GATE_RESID, _p(resid), 48, (M + 1) * 48, _p(gate), 0, _st())


def test_args_gemm_qkv_norm_rope_out_extra(rec):
    from gpt_image_edit_b200 import ops

    x, w, bias, wq, wk = _t(B, M, K), _t(NW, K), _t(NW), _t(128), _t(128)
    cos, sin = _t(M + 3, 128, dtype=f32), _t(M + 3, 128, dtype=f32)
    cat = _t(B, M, D + E)
    extra = cat[:, :, D:]
    out = ops.linear_qkv_norm_rope(x, w, bias, wq, wk, cos, sin, rope_row0=3, out_extra=extra,
                                   epi_extra=EPI_GELU_TANH)
    assert out.shape == (B, M, 3 * D)
    assert _one_call(rec, "b2f_gemm_qkv_norm_rope") == (
        _p(x), K, M * K, _p(w), K, _p(bias), _p(out), 3 * D, M * 3 * D, B, M, D, K,
        _p(wq), _p(wk), _p(cos), _p(sin), 3, 1e-6, E, _p(extra), D + E, M * (D + E), EPI_GELU_TANH, _st())


def test_args_gemm_colscale(rec):
    from gpt_image_edit_b200 import ops

    x, acat, cs = _t(M, K), _t(R, K), _t(R, dtype=f32)
    t = ops.lora_down(x, acat, cs, cs_mul=0.5)
    assert t.shape == (M, R)
    assert _one_call(rec, "b2f_gemm_colscale") == (
        _p(x), K, M * K, _p(acat), K, _p(t), R, M * R, 1, M, R, K, _p(cs), 0.5, _st())


def test_args_gemm_bf16_lora(rec):
    from gpt_image_edit_b200 import ops

    x, w, resid = _t(M, K), _t(N, K), _t(M, N)
    tb, bcat = _t(M, R + 8), _t(N, R)
    t = tb[:, :R]
    out = ops.linear_lora(x, w, None, t, bcat, epilogue=EPI_RESID, resid=resid)
    assert _one_call(rec, "b2f_gemm_bf16_lora") == (
        _p(x), K, M * K, _p(w), K, None, _p(out), N, M * N, 1, M, N, K, EPI_RESID, _p(resid), N, M * N, None, 0,
        _p(t), R + 8, M * (R + 8), _p(bcat), R, R, _st())


def test_args_gemm_qkv_norm_rope_lora(rec):
    from gpt_image_edit_b200 import ops

    x, w, bias, wq, wk = _t(1, M, K), _t(3 * D, K), _t(3 * D), _t(128), _t(128)
    cos, sin = _t(M, 128, dtype=f32), _t(M, 128, dtype=f32)
    t, bcat = _t(1, M, R), _t(3 * D, R)
    out = _t(1, M, 3 * D)
    ops.linear_qkv_norm_rope_lora(x, w, bias, wq, wk, cos, sin, t, bcat, out=out, eps=1e-5)
    assert _one_call(rec, "b2f_gemm_qkv_norm_rope_lora") == (
        _p(x), K, M * K, _p(w), K, _p(bias), _p(out), 3 * D, M * 3 * D, 1, M, D, K,
        _p(wq), _p(wk), _p(cos), _p(sin), 0, 1e-5, 0, None, 0, 0, 0,
        _p(t), R, M * R, _p(bcat), R, R, _st())


def test_args_gemm_fp8_2d_gate(rec):
    from gpt_image_edit_b200 import ops

    xq, xs, wq, ws = _t(B, M, K, dtype=E4M3), _t(B, M, dtype=f32), _t(N, K, dtype=E4M3), _t(N, dtype=f32)
    mod = _t(B, 3 * N)
    gate, out = mod[:, N:2 * N], _t(B, M, N)
    ops.linear_fp8(xq, xs, wq, ws, None, epilogue=EPI_GATE_RESID, out=out, resid=out, gate=gate)
    assert _one_call(rec, "b2f_gemm_fp8") == (
        _p(xq), K, M * K, _p(xs), M, _p(wq), K, _p(ws), None, _p(out), N, M * N, B, M, N, K,
        EPI_GATE_RESID, _p(out), N, M * N, _p(gate), 3 * N, _st())


def test_args_gemm_qkv_norm_rope_fp8(rec):
    from gpt_image_edit_b200 import ops

    xq, xs = _t(B, M, K, dtype=E4M3), _t(B, M, dtype=f32)
    wq, ws, bias, nq, nk = _t(NW, K, dtype=E4M3), _t(NW, dtype=f32), _t(NW), _t(128), _t(128)
    cos, sin = _t(M, 128, dtype=f32), _t(M, 128, dtype=f32)
    out, extra = _t(B, M, 3 * D), _t(B, M, E)
    ops.linear_qkv_norm_rope_fp8(xq, xs, wq, ws, bias, nq, nk, cos, sin, out=out, out_extra=extra, epi_extra=EPI_GELU_TANH)
    assert _one_call(rec, "b2f_gemm_qkv_norm_rope_fp8") == (
        _p(xq), K, M * K, _p(xs), M, _p(wq), K, _p(ws), _p(bias), _p(out), 3 * D, M * 3 * D, B, M, D, K,
        _p(nq), _p(nk), _p(cos), _p(sin), 0, 1e-6, E, _p(extra), E, M * E, EPI_GELU_TANH, _st())


def test_args_gemm_fp8_lora(rec):
    from gpt_image_edit_b200 import ops

    xq, xs, wq, ws, bias = _t(M, K, dtype=E4M3), _t(M, dtype=f32), _t(N, K, dtype=E4M3), _t(N, dtype=f32), _t(N)
    t, bcat = _t(M, R), _t(N, R)
    out = ops.linear_fp8_lora(xq, xs, wq, ws, bias, t, bcat, epilogue=EPI_GELU_TANH)
    assert _one_call(rec, "b2f_gemm_fp8_lora") == (
        _p(xq), K, M * K, _p(xs), M, _p(wq), K, _p(ws), _p(bias), _p(out), N, M * N, 1, M, N, K,
        EPI_GELU_TANH, None, 0, 0, None, 0, _p(t), R, M * R, _p(bcat), R, R, _st())


def test_args_gemm_qkv_norm_rope_fp8_lora(rec):
    from gpt_image_edit_b200 import ops

    xq, xs = _t(B, M, K, dtype=E4M3), _t(B, M, dtype=f32)
    wq, ws, nq, nk = _t(NW, K, dtype=E4M3), _t(NW, dtype=f32), _t(128), _t(128)
    cos, sin = _t(M + 2, 128, dtype=f32), _t(M + 2, 128, dtype=f32)
    t, bcat, extra = _t(B, M, R), _t(NW, R), _t(B, M, E)
    out = ops.linear_qkv_norm_rope_fp8_lora(xq, xs, wq, ws, None, nq, nk, cos, sin, t, bcat, rope_row0=2,
                                            out_extra=extra, epi_extra=EPI_GELU_TANH)
    assert _one_call(rec, "b2f_gemm_qkv_norm_rope_fp8_lora") == (
        _p(xq), K, M * K, _p(xs), M, _p(wq), K, _p(ws), None, _p(out), 3 * D, M * 3 * D, B, M, D, K,
        _p(nq), _p(nk), _p(cos), _p(sin), 2, 1e-6, E, _p(extra), E, M * E, EPI_GELU_TANH,
        _p(t), R, M * R, _p(bcat), R, R, _st())


def test_args_gemm_dgrad_strided(rec):
    from gpt_image_edit_b200 import train_ops as T

    dya = _t(B, M + 2, 3 * K)
    dy, w, aux = dya[:, 2:, K:2 * K], _t(K, N), _t(B, M, N)
    out = T.linear_dgrad(dy, w, epilogue=EPI_DGELU, aux=aux)
    assert _one_call(rec, "b2f_gemm_dgrad") == (
        _p(dy), 3 * K, (M + 2) * 3 * K, _p(w), N, _p(out), N, M * N, B, M, N, K, EPI_DGELU, _p(aux), N, M * N, _st())


def test_args_gemm_wgrad(rec):
    from gpt_image_edit_b200 import train_ops as T

    dy, x, buf = _t(B, M, N), _t(B, M, K), _t(N, K + 8, dtype=f32)
    dw = buf[:, :K]
    assert T.linear_wgrad(dy, x, out=dw, accumulate=True) is dw
    assert _one_call(rec, "b2f_gemm_wgrad") == (
        _p(dy), N, M * N, _p(x), K, M * K, _p(dw), K + 8, B, M, N, K, 1, _st())


def _qkv_slices(Bq, Sq, Hq):
    """q, k, v as head-split column slices of one [B, S, 3 H 128] projection buffer."""
    qkv = _t(Bq, Sq, 3 * Hq * 128)
    return [qkv[:, :, i * Hq * 128:(i + 1) * Hq * 128].unflatten(-1, (Hq, 128)) for i in range(3)]


def test_args_attention_fwd(rec):
    from gpt_image_edit_b200 import ops

    q, k, v = _qkv_slices(B, S, H)
    wide = _t(B, S, 3 * H * 128)
    out = wide[:, :, :H * 128]
    assert ops.attention(q, k, v, out=out, causal=True) is out
    ld = 3 * H * 128
    assert _one_call(rec, "b2f_attention_fwd") == (
        _p(q), ld, _p(k), ld, _p(v), ld, _p(out), ld, B, H, H, S, S, 128, 128 ** -0.5, 1, _st())


def test_args_attention_fwd_gqa_4d_out(rec):
    from gpt_image_edit_b200 import ops

    q, k, v = _t(1, 3, 4, 128), _t(1, S, 2, 128), _t(1, S, 2, 128)
    out = _t(1, 3, 4, 128)
    ops.attention(q, k, v, out=out, scale=0.25)
    assert _one_call(rec, "b2f_attention_fwd") == (
        _p(q), 512, _p(k), 256, _p(v), 256, _p(out), 512, 1, 4, 2, 3, S, 128, 0.25, 0, _st())


def test_args_attention_fwd_window(rec):
    from gpt_image_edit_b200 import ops

    q, k, v = _qkv_slices(B, S, H)
    win = _t(B, 2, dtype=torch.int32)
    out = ops.attention(q, k, v, win=win, S_txt=40)
    ld = 3 * H * 128
    assert _one_call(rec, "b2f_attention_fwd_window") == (
        _p(q), ld, _p(k), ld, _p(v), ld, _p(out), H * 128, B, H, H, S, S, 128, 128 ** -0.5, _p(win), 40, _st())


def test_args_attention_bias_fwd(rec):
    from gpt_image_edit_b200 import ops

    q, k, v = _qkv_slices(B, S, H)
    bias = _t(H, S, S + 6)[:, :, :S]
    out = ops.attention(q, k, v, scale=1.0, bias=bias)
    ld = 3 * H * 128
    assert _one_call(rec, "b2f_attention_bias_fwd") == (
        _p(q), ld, _p(k), ld, _p(v), ld, _p(out), H * 128, B, H, H, S, S, 128, 1.0, 0, _p(bias), S * (S + 6), S + 6,
        _st())


def test_args_attention_fwd_lse(rec):
    from gpt_image_edit_b200 import train_ops as T

    q, k, v = _qkv_slices(B, S, H)
    out, lse = T.attention_fwd_lse(q, k, v, scale=0.5)
    assert lse.shape == (B, H, 256) and out.shape == (B, S, H * 128)
    ld = 3 * H * 128
    assert _one_call(rec, "b2f_attention_fwd_lse") == (
        _p(q), ld, _p(k), ld, _p(v), ld, _p(out), H * 128, B, H, H, S, S, 128, 0.5, 0, _p(lse), 256, _st())


def test_args_attention_fp8_pair(rec):
    from gpt_image_edit_b200 import ops

    q, k, v = _qkv_slices(B, S, H)
    bufs = ops.attn_quant_fp8(q, k, v)
    q8, k8, sq, sk, v8t, sv = bufs
    assert v8t.shape == (B, H, 128, 256)
    ld = 3 * H * 128
    assert _one_call(rec, "b2f_attn_quant_fp8") == (
        _p(q), ld, _p(k), ld, _p(v), ld, _p(q8), _p(k8), _p(sq), _p(sk), _p(v8t), _p(sv), B, H, S, 128, _st())
    rec.calls.clear()
    cat = _t(B, S, 2 * H * 128)
    out = cat[:, :, :H * 128]
    assert ops.attention_fp8(*bufs, out=out) is out
    assert _one_call(rec, "b2f_attention_fp8") == (
        _p(q8), _p(k8), _p(sq), _p(sk), _p(v8t), _p(sv), _p(out), 2 * H * 128, B, H, S, 128, 128 ** -0.5, 0, _st())
