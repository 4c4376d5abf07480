"""GPU parity: b2f_gemm_bf16 (wgmma) against a torch fp32 reference of the same op.

Tolerance: inputs are bf16, accumulation fp32, one bf16 rounding on the output, so the result must
match round_bf16(fp32 reference) to within 1 bf16 ulp of the largest magnitude in the row-block
(rel-L2 <= 4e-3, i.e. about one bf16 rounding: 2^-8 = 3.9e-3).
"""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel_l2(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-20)).item()


def _mk(M, N, K, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.05).bfloat16()
    b = torch.randn(N, device="cuda", generator=g).bfloat16()
    return x, w, b


@pytest.mark.parametrize(
    "M,N,K",
    [
        (128, 128, 64),      # single tile, single k-block
        (128, 256, 128),
        (256, 512, 256),
        (544, 3072, 4096),   # context_embedder
        (1000, 136, 72),     # ragged everything (M, N, K tails)
        (8736, 3072, 3072),  # to_q at C1024
        (28, 18432, 3072),   # hoisted AdaLN (weight streaming)
        (4096, 64, 3072),    # proj_out
        (8192, 3072, 64),    # x_embedder
    ],
)
def test_gemm_bias(M, N, K):
    from gpt_image_edit_b200 import ops

    x, w, b = _mk(M, N, K)
    out = ops.linear(x, w, b)
    ref = (x.float() @ w.float().t() + b.float())
    assert out.shape == (M, N)
    err = _rel_l2(out, ref)
    assert err < 4e-3, f"rel-L2 {err}"
    # against the bf16-rounded reference nearly everything is identical
    max_abs = (out.float() - ref).abs().max().item()
    assert max_abs <= 2.0 ** -7 * ref.abs().max().item() + 1e-3


def test_gemm_no_bias_and_pitched_output():
    from gpt_image_edit_b200 import ops

    x, w, _ = _mk(300, 256, 192, seed=1)
    big = torch.zeros(300, 1024, device="cuda", dtype=torch.bfloat16)
    view = big[:, 512:768]
    ops.linear(x, w, None, out=view)
    ref = x.float() @ w.float().t()
    assert _rel_l2(view, ref) < 4e-3
    assert big[:, :512].abs().max().item() == 0 and big[:, 768:].abs().max().item() == 0


def test_gemm_gelu_silu():
    from gpt_image_edit_b200 import ops

    x, w, b = _mk(640, 768, 512, seed=2)
    lin = (x.float() @ w.float().t() + b.float()).bfloat16()
    out = ops.linear(x, w, b, epilogue=ops.EPI_GELU_TANH)
    ref = torch.nn.functional.gelu(lin.float(), approximate="tanh")
    assert _rel_l2(out, ref) < 6e-3
    out = ops.linear(x, w, b, epilogue=ops.EPI_SILU)
    ref = torch.nn.functional.silu(lin.float())
    assert _rel_l2(out, ref) < 6e-3


def test_gemm_gate_resid_batched_views():
    """Batched rows: A, out and resid are row-slices of a wider [B, S_all, *] buffer (the joint
    [txt;img] activation layout of the model), gate is per batch item."""
    from gpt_image_edit_b200 import ops

    B, S_all, S0, S, N, K = 2, 420, 40, 300, 384, 256
    g = torch.Generator(device="cuda").manual_seed(3)
    xa = torch.randn(B, S_all, K, device="cuda", generator=g).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.05).bfloat16()
    b = torch.randn(N, device="cuda", generator=g).bfloat16()
    ha = torch.randn(B, S_all, N, device="cuda", generator=g).bfloat16()
    gate = torch.randn(B, N, device="cuda", generator=g).bfloat16()
    x, h = xa[:, S0:S0 + S], ha[:, S0:S0 + S]
    h_before = ha.clone()
    lin = (x.float() @ w.float().t() + b.float()).bfloat16()
    ref = h.float() + (gate.float()[:, None] * lin.float()).bfloat16().float()
    ops.linear(x, w, b, epilogue=ops.EPI_GATE_RESID, resid=h, gate=gate, out=h)  # in place
    assert _rel_l2(h, ref) < 6e-3
    # rows outside the slice untouched
    assert torch.equal(ha[:, :S0], h_before[:, :S0]) and torch.equal(ha[:, S0 + S:], h_before[:, S0 + S:])


@pytest.mark.parametrize("B,M,H,K,row0", [(1, 200, 2, 256, 0), (2, 300, 3, 384, 40), (1, 8736, 24, 3072, 0)])
def test_gemm_qkv_norm_rope_equals_unfused_path(B, M, H, K, row0):
    """Fused epilogue == GEMM(bias) followed by the standalone rmsnorm_rope kernel (same rounding chain)."""
    from gpt_image_edit_b200 import ops

    d = H * 128
    g = torch.Generator(device="cuda").manual_seed(H)
    x = torch.randn(B, M, K, device="cuda", generator=g).bfloat16()
    w = (torch.randn(3 * d, K, device="cuda", generator=g) * 0.05).bfloat16()
    b = torch.randn(3 * d, device="cuda", generator=g).bfloat16()
    wq, wk = ((1 + 0.1 * torch.randn(128, device="cuda", generator=g)).bfloat16() for _ in range(2))
    S = row0 + M
    ids = torch.zeros(S, 3, device="cuda")
    ids[:, 1] = torch.arange(S, device="cuda") % 97
    ids[:, 2] = torch.arange(S, device="cuda") % 53
    cos, sin = ops.rope_tables(ids)
    fused = ops.linear_qkv_norm_rope(x, w, b, wq, wk, cos, sin, rope_row0=row0)
    ref = ops.linear(x, w, b)
    ops.rmsnorm_rope_(ref, H, wq, wk, cos[row0:].contiguous(), sin[row0:].contiguous())
    mism = (fused != ref).float().mean().item()
    assert mism < 1e-3, f"{mism:.4%} elements differ"
    assert torch.equal(fused[..., 2 * d:], ref[..., 2 * d:])      # V untouched by norm/rope
