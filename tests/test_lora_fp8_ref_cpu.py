"""The references of tests/lora_fp8_ref.py on the CPU, against independent fp64 restatements."""
import torch

import fp8_ref as Q
import infer_block_ref as IB
import kernel_ref as R
import lora_fp8_ref as LQ
import lora_ref as LR
from oracle import flux_oracle as fo


def _operands(seed, M=9, K=256, N=40, r_pad=64):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(2, M, K, generator=g).bfloat16()
    w = (torch.randn(N, K, generator=g) * K ** -0.5).bfloat16()
    acat = (torch.randn(r_pad, K, generator=g) * K ** -0.5).bfloat16()
    bcat = (torch.randn(N, r_pad, generator=g) * 0.1).bfloat16()
    cs = torch.rand(r_pad, generator=g) * 2 - 1
    return x, w, acat, bcat, cs, torch.randn(N, generator=g).bfloat16()


def test_down_emu_is_rounded_scaled_product():
    x, _, acat, _, cs, _ = _operands(0)
    t = LQ.down_emu(x, acat, cs, 0.7)
    ref = (x.double() @ acat.double().T) * (cs * 0.7).double()
    assert torch.equal(t, ref.float().bfloat16().double())


def test_linear_fp8_lora_emu_restated():
    """emu = bf16(sa sw (xq wq^T) + T Bcat^T + b) in fp64, floor = max(K_all 2^-24, 2^-p) * absref."""
    x, w, acat, bcat, cs, b = _operands(1)
    xq, xs = Q.quant_rows(x)
    wq, ws = Q.quant_rows(w)
    t = LQ.down_emu(x, acat, cs, 0.5).bfloat16()
    sc = xs.double()[..., :, None] * ws.double()[None, None, :]
    pre = (xq.double() @ wq.double().T) * sc + t.double() @ bcat.double().T + b.double()
    absref = (xq.double().abs() @ wq.double().abs().T) * sc + t.double().abs() @ bcat.double().abs().T + b.double().abs()
    emu, floor, math = LQ.linear_fp8_lora_emu(xq, xs, wq, ws, t, bcat, b, p=11)
    assert torch.allclose(math, pre, rtol=1e-12, atol=0)
    assert torch.equal(emu, R.bf16r(pre))
    assert torch.allclose(floor, 2.0 ** -11 * absref, rtol=1e-12)             # 2^-11 > (256 + 64) * 2^-24
    # an adapter with Bcat = 0 gives the plain FP8 emulation
    z = LQ.linear_fp8_lora_emu(xq, xs, wq, ws, t, torch.zeros_like(bcat), b, p=11)[0]
    assert torch.equal(z, Q.linear_fp8_emu(xq, xs, wq, ws, b, p=11)[0])
    # epilogues run on the same pre-activation
    resid, gate = torch.randn(2, 9, 40).bfloat16(), torch.randn(2, 40).bfloat16()
    e = LQ.linear_fp8_lora_emu(xq, xs, wq, ws, t, bcat, b, R.EPI_GATE_RESID, p=11, resid=resid, gate=gate)[0]
    y = R.bf16r(pre)
    assert torch.equal(e, R.bf16r(resid.double() + R.bf16r(gate.double()[:, None, :] * y)))


def test_qkv_fp8_lora_emu_is_qkv_emu_of_the_sum():
    g = torch.Generator().manual_seed(2)
    d, K, M = 256, 128, 5
    x = torch.randn(1, M, K, generator=g).bfloat16()
    w = (torch.randn(3 * d, K, generator=g) * K ** -0.5).bfloat16()
    b = torch.randn(3 * d, generator=g).bfloat16()
    t = torch.randn(1, M, 64, generator=g).bfloat16()
    bcat = (torch.randn(3 * d, 64, generator=g) * 0.1).bfloat16()
    nq = nk = torch.ones(128).bfloat16()
    ang = torch.rand(M, 64, generator=g) * 6.28
    cos, sin = ang.cos().repeat_interleave(2, 1), ang.sin().repeat_interleave(2, 1)
    xq, xs = Q.quant_rows(x)
    wq, ws = Q.quant_rows(w)
    emu, _, math = LQ.qkv_fp8_lora_emu(xq, xs, wq, ws, t, bcat, b, nq, nk, cos, sin, p=11)
    pre = Q.dequant(xq, xs) @ Q.dequant(wq, ws).T + t.double() @ bcat.double().T + b.double()
    ref = R.qkv_norm_rope_emu(pre, torch.eye(3 * d, dtype=torch.float64), None, nq, nk, cos, sin)[0]
    assert torch.equal(emu, ref)


def test_fp8_lora_oracle_adds_unquantized_update():
    """Block linears: fake-quantized base plus the adapter on the unquantized input; other linears: PEFT as is."""
    cfg = fo.FluxConfig(num_layers=1, num_single_layers=1, attention_head_dim=128, num_attention_heads=2,
                        joint_attention_dim=64, pooled_projection_dim=32, in_channels=16, out_channels=16)
    sd = {k: v.double() for k, v in fo.make_synthetic_state_dict(cfg, seed=0, dtype=torch.bfloat16).items()}
    lora = LR.make_lora(cfg, rank=4, seed=3, alpha=8.0, a_std=0.1, b_std=0.1)
    g = torch.Generator().manual_seed(4)
    for name in ("transformer_blocks.0.attn.to_q", "single_transformer_blocks.0.proj_out", "x_embedder",
                 "transformer_blocks.0.norm1.linear"):
        k = sd[name + ".weight"].shape[1]
        x = torch.randn(3, k, generator=g, dtype=torch.float64)
        A, B, alpha = lora[name]
        upd = 0.7 * alpha / A.shape[0] * (x @ A.double().T) @ B.double().T
        with LQ.fp8_lora_linears([(lora, 0.7)]):
            y = fo._lin(sd, name, x)
        with Q.fp8_linears():
            base = fo._lin(sd, name, x)
        assert torch.allclose(y - base, upd, rtol=1e-9, atol=1e-12), name
        quantized = Q.BLOCK_LINEAR.match(name) is not None
        plain = torch.nn.functional.linear(x, sd[name + ".weight"], sd[name + ".bias"])
        assert torch.equal(base, plain) != quantized, name
    # the stage functions pick the adapters up
    S_txt, n = 4, 8
    mod = torch.randn(1, 17 * cfg.inner_dim, generator=g, dtype=torch.float64) * 0.1
    ids = torch.zeros(S_txt + n, 3)
    ids[S_txt:, 2] = torch.arange(n)
    cos, sin = fo.rope_tables(ids, cfg.axes_dims_rope, cfg.theta)
    h = torch.randn(1, S_txt + n, cfg.inner_dim, generator=g, dtype=torch.float64)
    with Q.fp8_linears():
        q8 = IB.double_stage(sd, cfg, 0, h, mod, cos, sin, S_txt, torch.float64)["h"]
    with LQ.fp8_lora_linears([(lora, 0.7)]):
        q8l = IB.double_stage(sd, cfg, 0, h, mod, cos, sin, S_txt, torch.float64)["h"]
    assert R.rel_l2(q8l, q8) > 1e-4
