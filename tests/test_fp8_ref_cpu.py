"""The FP8 references of tests/fp8_ref.py on the CPU: the row rule at its rounding and saturation edges, and the FP8
variant of the oracle's forward at a toy width."""
import torch

import fp8_ref as Q
import infer_block_ref as IB
import kernel_ref as R
from oracle import flux_oracle as fo


def _bytes(q):
    return q.view(torch.uint8).tolist()


def _row(vals, amax=448.0):
    """a bf16 row whose amax is `amax` (so inv = 448 / amax) followed by `vals`."""
    return torch.tensor([amax] + list(vals), dtype=torch.float32).bfloat16()


def test_row_rule_ties_round_to_even():
    # amax = 448: inv = 1, s = 1.  e4m3 spacing in [1, 2) is 1/8: 1.0625 ties 1.0 (0x38) / 1.125 (0x39) -> even 0x38;
    # 1.1875 ties 1.125 / 1.25 (0x3a) -> 0x3a; -1.0625 -> 0xb8
    q, s = Q.quant_rows(_row([1.0625, 1.1875, -1.0625, 1.0]))
    assert s.item() == 1.0
    assert _bytes(q) == [0x7E, 0x38, 0x3A, 0xB8, 0x38]


def test_row_rule_subnormal_outputs():
    # e4m3 subnormals are multiples of 2^-9: 2^-9 -> 0x01; 1.5 * 2^-9 ties 0x01 / 0x02 -> 0x02; 0.5 * 2^-9 ties 0 / 0x01
    # -> 0; 2^-7 - 2^-9 = 3 * 2^-9 -> 0x03; 2^-6 is the smallest normal (0x08)
    u = 2.0 ** -9
    q, _ = Q.quant_rows(_row([u, 1.5 * u, 0.5 * u, 3 * u, 2.0 ** -6, -u]))
    assert _bytes(q) == [0x7E, 0x01, 0x02, 0x00, 0x03, 0x08, 0x81]


def test_row_rule_scale_and_saturation_edge():
    # amax * fp32(448 / amax) rounds above 448 for some amax: the product must saturate to 448 (0x7e), never NaN (0x7f),
    # and torch's own conversion would map it to 448 as well below 464
    x = torch.linspace(0.5, 3.0, 20001, dtype=torch.float32).bfloat16().unique()
    inv = torch.full_like(x.float(), 448.0) / x.float()
    over = x[(x.float() * inv) > 448.0]
    assert over.numel() > 0
    q, s = Q.quant_rows(over[:, None].expand(-1, 4).contiguous())
    assert (q.view(torch.uint8) == 0x7E).all()
    assert torch.equal(s, over.float() / 448.0)
    assert (torch.tensor([449.0, 463.9]).to(Q.E4M3).float() == 448.0).all()   # the saturation torch applies itself


def test_row_rule_zero_rows():
    x = torch.zeros(3, 48, dtype=torch.bfloat16)
    x[1] = -0.0
    x[2, 5] = 3.0
    q, s = Q.quant_rows(x)
    assert s.tolist()[:2] == [1.0, 1.0] and s[2] == torch.tensor(3.0) / 448.0
    assert (q[:2].view(torch.uint8) == 0).all()
    assert q[2].view(torch.uint8)[5].item() == 0x7E


def test_row_rule_batched_is_per_row():
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(2, 5, 96, generator=g) * torch.logspace(-3, 3, 5)[None, :, None]).bfloat16()
    q, s = Q.quant_rows(x)
    for b in range(2):
        for r in range(5):
            q1, s1 = Q.quant_rows(x[b, r])
            assert torch.equal(q[b, r].view(torch.uint8), q1.view(torch.uint8)) and s[b, r] == s1
    err = (Q.dequant(q, s) - x.double()).abs() / x.double().abs().amax(-1, keepdim=True)
    assert err.max() <= 2.0 ** -4   # half an e4m3 ulp at the top binade, relative to amax


def test_linear_fp8_emu_is_scaled_integer_product():
    g = torch.Generator().manual_seed(1)
    x, w, b = torch.randn(7, 64, generator=g).bfloat16(), torch.randn(24, 64, generator=g).bfloat16(), torch.randn(24, generator=g).bfloat16()
    xq, xs = Q.quant_rows(x)
    wq, ws = Q.quant_rows(w)
    emu, floor, pre = Q.linear_fp8_emu(xq, xs, wq, ws, b, p=12)
    acc = xq.double() @ wq.double().T
    ref = acc * (xs.double()[:, None] * ws.double()[None, :]) + b.double()
    assert torch.allclose(pre, ref, rtol=1e-12, atol=0)
    assert torch.equal(emu, R.bf16r(pre))
    absref = (xq.double().abs() @ wq.double().abs().T) * (xs.double()[:, None] * ws.double()[None, :]) + b.double().abs()
    assert torch.allclose(floor, 2.0 ** -12 * absref, rtol=1e-12)            # 2^-12 > 64 * 2^-24
    assert torch.allclose(Q.linear_fp8_emu(xq, xs, wq, ws, b, p=20)[1], 64 * R.U32 * absref, rtol=1e-12)


def test_fp8_oracle_quantizes_block_linears_only():
    cfg = fo.FluxConfig(num_layers=1, num_single_layers=1, attention_head_dim=128, num_attention_heads=2,
                        joint_attention_dim=64, pooled_projection_dim=32, in_channels=16, out_channels=16)
    sd = {k: v.double() for k, v in fo.make_synthetic_state_dict(cfg, seed=0, dtype=torch.bfloat16).items()}
    g = torch.Generator().manual_seed(2)
    B, S_txt, n = 1, 8, 16
    hs, enc = torch.randn(B, n, 16, generator=g, dtype=torch.float64), torch.randn(B, S_txt, 64, generator=g, dtype=torch.float64)
    pooled = torch.randn(B, 32, generator=g, dtype=torch.float64)
    ids = torch.zeros(n, 3)
    ids[:, 1], ids[:, 2] = torch.arange(n) // 4, torch.arange(n) % 4
    args = (hs, enc, pooled, torch.tensor([0.5]), ids, torch.zeros(S_txt, 3))
    ref = fo.flux_forward(sd, cfg, *args, guidance=torch.tensor([3.5]))
    with Q.fp8_linears():
        q8 = fo.flux_forward(sd, cfg, *args, guidance=torch.tensor([3.5]))
        assert torch.equal(fo._lin(sd, "x_embedder", hs), Q.F.linear(hs, sd["x_embedder.weight"], sd["x_embedder.bias"]))
    # a double block's 6 projections, to_out, to_add_out and 4 MLP linears; a single block's q, k, v, proj_mlp, proj_out
    quantized = [k for k in sd if k.endswith(".weight") and Q.BLOCK_LINEAR.match(k[:-len(".weight")])]
    assert len(quantized) == 12 + 5, quantized
    e = R.rel_l2(q8, ref)
    assert 1e-4 < e < 0.1, e
    # the stage functions of infer_block_ref pick up the same quantization
    mod = torch.randn(B, 12 * cfg.inner_dim + 3 * cfg.inner_dim + 2 * cfg.inner_dim, generator=g, dtype=torch.float64) * 0.1
    cos, sin = fo.rope_tables(torch.cat([torch.zeros(S_txt, 3), ids]), cfg.axes_dims_rope, cfg.theta)
    h = torch.randn(B, S_txt + n, cfg.inner_dim, generator=g, dtype=torch.float64)
    plain = IB.double_stage(sd, cfg, 0, h, mod, cos, sin, S_txt, torch.float64)["h"]
    with Q.fp8_linears():
        quant = IB.double_stage(sd, cfg, 0, h, mod, cos, sin, S_txt, torch.float64)["h"]
    assert 1e-5 < R.rel_l2(quant, plain) < 0.1
