"""The FP8 attention references (tests/attn_fp8_ref.py) on the CPU: the v8t token order, its padding, the per-head /
per-channel quantization against the row rule, and the online emulation against the direct formulas."""
import math

import pytest
import torch

import attn_fp8_ref as A
import fp8_ref as Q
import kernel_ref as R


def _qkv(B, S, H, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(B, S, H, 128, generator=g) * scale).bfloat16() for _ in range(3)]


def test_v8t_order_is_a_bijection_per_group():
    perm = A.V8T_TOKEN
    assert sorted(perm.tolist()) == list(range(32))
    # the documented fragment rule: k-positions 4t..4t+3 hold {2t, 2t+1, 8+2t, 9+2t}, 16+4t.. the same plus 16
    for t in range(4):
        assert perm[4 * t:4 * t + 4].tolist() == [2 * t, 2 * t + 1, 8 + 2 * t, 9 + 2 * t]
        assert perm[16 + 4 * t:20 + 4 * t].tolist() == [16 + 2 * t, 17 + 2 * t, 24 + 2 * t, 25 + 2 * t]
    idx = A.v8t_order(256)
    assert sorted(idx.tolist()) == list(range(256))
    assert torch.equal(idx // 32, torch.arange(256) // 32)        # never leaves its group
    x = torch.arange(256, dtype=torch.uint8).view(Q.E4M3)
    assert torch.equal(A.v8t_tokens(x[idx], 256).view(torch.uint8), torch.arange(256, dtype=torch.uint8))


@pytest.mark.parametrize("S", [1, 127, 128, 129, 300])
def test_quant_attn_is_the_row_rule(S):
    B, H = 2, 3
    q, k, v = _qkv(B, S, H, S)
    k[1, :, 2] = 0                                                 # an all-zero head: scale 1, +0 bytes
    q8, k8, sq, sk, v8t, sv = A.quant_attn(q, k, v)
    P = A.s_pad(S)
    assert v8t.shape == (B, H, 128, P) and sv.shape == (B, H, 128) and sq.shape == (B, H)
    for x, x8, s in ((q, q8, sq), (k, k8, sk)):
        r8, rs = Q.quant_rows(x.permute(0, 2, 1, 3).reshape(B, H, S * 128))
        assert torch.equal(x8.permute(0, 2, 1, 3).reshape(B, H, -1).view(torch.uint8), r8.view(torch.uint8))
        assert torch.equal(s, rs)
    assert sk[1, 2] == 1 and not k8[1, :, 2].view(torch.uint8).any()
    r8, rs = Q.quant_rows(v.permute(0, 2, 3, 1))
    assert torch.equal(A.v8t_tokens(v8t, S).view(torch.uint8), r8.view(torch.uint8)) and torch.equal(sv, rs)
    pad = v8t.view(torch.uint8)[..., A.v8t_order(P) >= S]
    assert pad.numel() == B * H * 128 * (P - S) and not pad.any()  # +0 (byte 0x00), not -0 (0x80)


def test_emulation_without_quantization_is_attention_math():
    """Identity quantization (unit scales, unrounded P) reproduces attention_math."""
    B, S, H = 1, 300, 2
    q, k, v = (x.double() for x in _qkv(B, S, H, 7, scale=2.0))
    hm = lambda x: x.permute(0, 2, 1, 3)
    ones = torch.ones(B, H, dtype=torch.float32)
    o = A.attention_fp8_core(hm(q), hm(k), ones, ones, hm(v), torch.ones(B, H, 128), 128 ** -0.5,
                             quant_p=False)
    mth, _ = R.attention_math(q, k, v)
    flat = o.permute(0, 2, 1, 3).reshape(B, S, H * 128)
    assert R.rel_l2(flat, mth) < 1e-6    # the score scale is rounded to fp32 as the kernel rounds it


@pytest.mark.parametrize("Skv", [1, 77, 128])
def test_online_emulation_in_one_block_is_the_direct_formula(Skv):
    """With one KV block the online softmax is out = sv / 256 * e4m3(256 * 2^(t - max t)) V8 / sum 2^(t - max t)."""
    B, H = 2, 2
    q, k, v = _qkv(B, Skv, H, Skv, scale=3.0)
    q8, k8, sq, sk, v8t, sv = A.quant_attn(q, k, v)
    hm = lambda x: x.permute(0, 2, 1, 3).to(torch.float64)
    v8 = A.v8t_tokens(v8t, Skv).transpose(-1, -2).to(torch.float64)
    o = A.attention_fp8_core(hm(q8), hm(k8), sq, sk, v8, sv, 128 ** -0.5)
    t = hm(q8) @ hm(k8).transpose(-1, -2) * A.score_scale(sq, sk, 128 ** -0.5)[..., None, None]
    p = torch.exp2(t - t.amax(-1, keepdim=True))
    p8 = (p * 256).float().to(Q.E4M3).double()
    direct = (p8 @ v8) * (sv.double()[..., None, :] / 256) / p.sum(-1, keepdim=True)
    assert torch.equal(o, direct)


def test_fp8_attention_context_quantizes_the_oracle():
    """fp8_attention() swaps the oracle's attention for the FP8 one and restores it; the result stays close to the
    unquantized attention (a few e4m3 steps)."""
    from oracle import flux_oracle as fo

    q, k, v = (x.permute(0, 2, 1, 3).double() for x in _qkv(1, 200, 2, 3))
    ref = fo.attention(q, k, v)
    with A.fp8_attention():
        f8 = fo.attention(q, k, v)
    assert fo.attention(q, k, v).equal(ref)
    e = R.rel_l2(f8, ref)
    assert 1e-3 < e < 0.1, e
    assert math.isfinite(e)
