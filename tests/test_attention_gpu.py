"""GPU parity: b2f_attention_fwd (wgmma, S/P/O in registers) against an fp32 softmax-attention
reference of the same op (plain matmul + softmax in fp32 on the bf16 inputs).

Tolerance: P is rounded to bf16 before P·V and the output is rounded to bf16, so the error budget is
two bf16 roundings: rel-L2 <= 8e-3 against the fp32 reference; torch's own bf16 SDPA on the same
inputs sits at 3-5e-3.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(q, k, v, causal=False):
    # q [B,Sq,H,dh], k/v [B,Skv,Hkv,dh] -> [B,Sq,H*dh], fp32 math
    B, Sq, H, dh = q.shape
    Hkv = k.shape[2]
    qf = q.float().permute(0, 2, 1, 3)
    kf = k.float().permute(0, 2, 1, 3).repeat_interleave(H // Hkv, dim=1)
    vf = v.float().permute(0, 2, 1, 3).repeat_interleave(H // Hkv, dim=1)
    s = qf @ kf.transpose(-1, -2) / math.sqrt(dh)
    if causal:
        mask = torch.ones(Sq, k.shape[1], device=q.device, dtype=torch.bool).tril()
        s = s.masked_fill(~mask, float("-inf"))
    o = torch.softmax(s, dim=-1) @ vf
    return o.permute(0, 2, 1, 3).reshape(B, Sq, H * dh)


def _rel_l2(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm()).item()


@pytest.mark.parametrize(
    "B,H,Hkv,Sq,Skv,causal",
    [
        (1, 1, 1, 128, 128, False),
        (1, 2, 2, 256, 256, False),
        (1, 2, 2, 256, 512, False),
        (2, 3, 3, 300, 300, False),     # ragged tail in q and kv, batch > 1
        (1, 2, 2, 1056, 1056, False),   # 256^2 config: S = 1056 = 8*128 + 32
        (1, 24, 24, 2592, 2592, False), # 512^2 config, all heads
        (1, 4, 4, 8736, 8736, False),   # C1024 sequence length (4 of 24 heads)
        (2, 2, 2, 640, 640, False),     # batch > 1, last 128-row tile partial
        (1, 4, 2, 768, 1000, False),    # GQA, Sq != Skv, ragged kv tail
        (1, 4, 2, 384, 384, True),      # causal + GQA (Qwen2.5-VL style)
        (2, 28, 4, 290, 290, True),     # Qwen2.5-VL-7B head layout, L=290
    ],
)
def test_attention_matches_fp32_reference(B, H, Hkv, Sq, Skv, causal):
    from gpt_image_edit_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(Sq + H)
    q = torch.randn(B, Sq, H, 128, device="cuda", generator=g).bfloat16()
    k = torch.randn(B, Skv, Hkv, 128, device="cuda", generator=g).bfloat16()
    v = torch.randn(B, Skv, Hkv, 128, device="cuda", generator=g).bfloat16()
    out = ops.attention(q, k, v, causal=causal)
    ref = _ref(q, k, v, causal)
    assert out.shape == ref.shape
    assert torch.isfinite(out.float()).all()
    err = _rel_l2(out, ref)
    assert err < 8e-3, f"rel-L2 {err}"


def test_attention_strided_qkv_and_output_slice():
    """Q/K/V as column slices of one [B,S,3*H*128] projection buffer; O into a wider buffer."""
    from gpt_image_edit_b200 import ops

    B, S, H = 1, 700, 3
    g = torch.Generator(device="cuda").manual_seed(5)
    qkv = torch.randn(B, S, 3 * H * 128, device="cuda", generator=g).bfloat16()
    q = qkv[:, :, : H * 128].unflatten(-1, (H, 128))
    k = qkv[:, :, H * 128 : 2 * H * 128].unflatten(-1, (H, 128))
    v = qkv[:, :, 2 * H * 128 :].unflatten(-1, (H, 128))
    wide = torch.zeros(B, S, 5 * H * 128, device="cuda", dtype=torch.bfloat16)
    ops.attention(q, k, v, out=wide[:, :, : H * 128])
    ref = _ref(q, k, v)
    assert _rel_l2(wide[:, :, : H * 128], ref) < 8e-3
    assert wide[:, :, H * 128 :].abs().max().item() == 0


def test_attention_peaked_softmax_rows():
    """Large-magnitude logits exercise the running-max / lazy-rescale path."""
    from gpt_image_edit_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(11)
    B, S, H = 1, 1024, 2
    q = (torch.randn(B, S, H, 128, device="cuda", generator=g) * 4).bfloat16()
    k = (torch.randn(B, S, H, 128, device="cuda", generator=g) * 4).bfloat16()
    # make later keys systematically larger so the row max keeps growing block after block
    k = (k.float() * torch.linspace(0.2, 2.0, S, device="cuda")[None, :, None, None]).bfloat16()
    v = torch.randn(B, S, H, 128, device="cuda", generator=g).bfloat16()
    out = ops.attention(q, k, v)
    ref = _ref(q, k, v)
    assert torch.isfinite(out.float()).all()
    assert _rel_l2(out, ref) < 1e-2
