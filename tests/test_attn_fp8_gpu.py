"""FP8 attention on the GPU: b2f_attn_quant_fp8 bit for bit against the reference quantization (tests/attn_fp8_ref.py),
b2f_attention_fp8 element by element against its fp64 emulation, its accuracy against fp64 unquantized attention, and
the FLUX forward with FP8 attention stage by stage and end to end.

Accumulation floor.  P8 V8 accumulates e4m3 products on the FP8 tensor cores into the running fp32 O, as the FP8 GEMM
accumulates (tests/test_fp8_gpu.py).  test_attention_fp8_accumulation_precision measures the error on outputs whose exact
value is 0 and holds it to the emulation's floor max(Skv 2^-24, 2^-11) * absref.
"""
import math

import pytest
import torch

import attn_fp8_ref as A
import fp8_ref as Q
import infer_block_ref as IB
import kernel_ref as R
from oracle import flux_oracle as fo
from test_flux_blocks_gpu import CASES, _fwd, _report, _setup, _temb_mod

pytestmark = pytest.mark.gpu

P_ACC = 11.0                      # tests/test_fp8_gpu.py: the FP8 tensor cores' accumulation floor 2^-11 * absref
TH_ATTN = dict(max_ulp=2, share_gt1=1e-3, mean_ulp=0.05)
BHSD = ("b", "token", "head", "col")
f64, bf16 = torch.float64, torch.bfloat16


def _g(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _qkv_buffer(B, S, H, g, scale=1.0):
    """q, k, v as the model holds them: head-split column slices of one qkv [B, S, 3 H 128] buffer."""
    d = H * 128
    qkv = (torch.randn(B, S, 3 * d, device="cuda", generator=g) * scale).bfloat16()
    return [qkv[:, :, i * d:(i + 1) * d].unflatten(-1, (H, 128)) for i in range(3)]


def _u8(t):
    return t.view(torch.uint8)


# ---------------------------------------------------------------------------------------------------- quantizer
@pytest.mark.parametrize("S", [1, 127, 128, 129, 4641])
@pytest.mark.parametrize("H", [1, 3])
def test_attn_quant_fp8_bit_exact(S, H):
    """The model's strided [B, S, 3d] views; one all-zero head; rows spanning 4 decades; amaxes of either sign (their
    element lands exactly on +-448)."""
    from gpt_image_edit_b200 import ops

    B = 2
    g = _g(S * 10 + H)
    q, k, v = _qkv_buffer(B, S, H, g)
    span = torch.logspace(-2, 2, S, device="cuda")[torch.randperm(S, device="cuda", generator=g)]
    v.mul_(span[None, :, None, None].bfloat16())
    k[1, :, H - 1] = 0
    q[0, S // 2, 0, 5] = -1000.0
    q8, k8, sq, sk, v8t, sv = ops.attn_quant_fp8(q, k, v)
    r = A.quant_attn(q, k, v)
    c = R.Checker(f"attn quant B{B} S{S} H{H}")
    for n, a, b in zip(("q8", "k8", "sq", "sk", "v8t", "sv"), (q8, k8, sq, sk, v8t, sv), r):
        c.equal(n, _u8(a) if a.dtype == Q.E4M3 else a, _u8(b) if b.dtype == Q.E4M3 else b)
    c.equal("-448 at the q amax", q8[0, S // 2, 0, 5].float(), torch.tensor(-448.0, device="cuda"))
    c.equal("zero head scale", sk[1, H - 1], torch.tensor(1.0, device="cuda"))
    c.finish()


# ---------------------------------------------------------------------------------------------------- attention
def _attn_fp8_check(name, q, k, v, *, ldo_mult=5, th=TH_ATTN):
    from gpt_image_edit_b200 import ops

    B, S, H, D = q.shape
    d = H * D
    cat = torch.full((B, S, ldo_mult * d), float("nan"), device="cuda", dtype=bf16)
    out = ops.attention_fp8(*ops.attn_quant_fp8(q, k, v), out=cat[:, :, :d])
    emu, floor, mth = A.attention_fp8_emu(q, k, v)
    c = R.Checker(name)
    shp = (B, S, H, D)
    # against fp64 math, within 1.15x of what the quantization itself costs (the emulation's rel-L2)
    c.bf16("o", out.reshape(shp), emu.view(shp), floor.view(shp), math_ref=mth.view(shp),
           rel_l2_max=1.15 * R.rel_l2(emu, mth), dims=BHSD, **th)
    c.equal("columns outside the slice", torch.isnan(cat[:, :, d:]).all(), torch.tensor(True, device="cuda"))
    c.finish()
    return out, emu, mth


@pytest.mark.parametrize("B,S", [(1, 1), (2, 64), (1, 127), (2, 128), (2, 129), (1, 255), (2, 1000), (1, 4641)])
def test_attention_fp8_matches_emulation(B, S):
    """Query tiles and KV blocks at their edges (128 rows each, two slots: the phase flips at block 3), batch items,
    output into a pitched cat slice (ldo = 5d)."""
    q, k, v = _qkv_buffer(B, S, 2, _g(S + B), scale=2.0)
    _attn_fp8_check(f"attn fp8 B{B} S{S}", q, k, v)


def test_attention_fp8_peaked_softmax_rows():
    """Large logits whose row max keeps growing block after block (test_attention_peaked_softmax_rows' construction)."""
    g = _g(11)
    B, S, H = 1, 1024, 2
    q = (torch.randn(B, S, H, 128, device="cuda", generator=g) * 4).bfloat16()
    k = (torch.randn(B, S, H, 128, device="cuda", generator=g) * 4).bfloat16()
    k = (k.float() * torch.linspace(0.2, 2.0, S, device="cuda")[None, :, None, None]).bfloat16()
    v = torch.randn(B, S, H, 128, device="cuda", generator=g).bfloat16()
    _attn_fp8_check("attn fp8 peaked", q, k, v)


@pytest.mark.parametrize("S", [1024, 8736])
def test_attention_fp8_accumulation_precision(S):
    """q = 0 gives p = 1 for every key (P8 = 256 exactly) and v = [a; -a] along the tokens makes every exact output 0
    while the running O is not: the output is the P.V accumulation error (times sv / 256 / l) rounded once to bf16."""
    from gpt_image_edit_b200 import ops

    g = _g(S)
    B, H = 1, 2
    q = torch.zeros(B, S, H, 128, device="cuda", dtype=bf16)
    k = torch.randn(B, S, H, 128, device="cuda", generator=g).bfloat16()
    a = torch.randn(B, S // 2, H, 128, device="cuda", generator=g).bfloat16()
    v = torch.cat([a, -a], 1)
    bufs = ops.attn_quant_fp8(q, k, v)
    out = ops.attention_fp8(*bufs).double().view(B, S, H, 128)
    absref = (A.v8t_tokens(bufs[4], S).double().abs().mean(-1) * bufs[5].double())[:, None]   # sum_j P_j |v~_j|
    err = (out.abs() / absref).max().item()
    p = -math.log2(max(err, 2.0 ** -60))
    print(f"KREF fp8 attention accumulation Skv={S}: worst |err| = 2^-{p:.2f} * absref = Skv * 2^-{p + math.log2(S):.2f}"
          f" * absref; nonzero outputs {(out != 0).double().mean().item():.3g}")
    assert err <= max(S * R.U32, 2.0 ** -P_ACC), f"accumulation error 2^-{p:.2f} * absref exceeds the floor"


def test_attention_fp8_kernel_accuracy():
    """S = 4641 with realistic, peaked logits (RMSNorm'd q / k of unit rms per head times a weight of rms 2.5): the
    engine's rel-L2 to fp64 unquantized attention is at most 1.15x that of the fp64 emulation of the same scheme."""
    from gpt_image_edit_b200 import ops

    g = _g(4641)
    B, S, H = 1, 4641, 2
    q, k, v = (torch.randn(B, S, H, 128, device="cuda", generator=g) for _ in range(3))
    w = (1 + 2 * torch.rand(128, device="cuda", generator=g)) * 1.25                  # norm weights: rms ~2.5
    q, k = ((x / x.pow(2).mean(-1, keepdim=True).sqrt() * w).bfloat16() for x in (q, k))
    v = v.bfloat16()
    out = ops.attention_fp8(*ops.attn_quant_fp8(q, k, v))
    emu, _, mth = A.attention_fp8_emu(q, k, v)
    bf = ops.attention(q, k, v)
    e_eng, e_emu, e_bf = R.rel_l2(out, mth), R.rel_l2(emu, mth), R.rel_l2(bf, mth)
    pmax = torch.softmax(q[0, :512, 0].double() @ k[0, :, 0].double().T * 128 ** -0.5, -1).amax(-1).median().item()
    print(f"KREF fp8 attention accuracy S={S}: engine {e_eng:.4g}, fp64 emulation {e_emu:.4g}, bf16 kernel {e_bf:.4g} "
          f"(median row max p {pmax:.3g})")
    assert e_eng <= 1.15 * e_emu


# ---------------------------------------------------------------------------------------------------- refusals
def test_attention_fp8_refusals():
    from gpt_image_edit_b200 import _lib, ops

    g = _g(3)
    q, k, v = _qkv_buffer(1, 200, 2, g)
    bufs = ops.attn_quant_fp8(q, k, v)
    with pytest.raises(_lib.B2FError, match="unsupported"):
        ops.attention_fp8(*bufs, causal=True)
    with pytest.raises(_lib.B2FError, match="bias"):
        ops.attention_fp8(*bufs, bias=torch.zeros(2, 200, 200, device="cuda", dtype=bf16))
    q64 = torch.randn(1, 200, 2, 64, device="cuda", generator=g).bfloat16()
    with pytest.raises(_lib.B2FError, match="unsupported"):
        ops.attn_quant_fp8(q64, q64, q64)
    lib = _lib.lib
    p = [t.data_ptr() for t in bufs]
    out = torch.empty(1, 200, 2 * 128 + 8, device="cuda", dtype=bf16)
    s = _lib.stream_ptr()
    assert lib.b2f_attention_fp8(*p, out.data_ptr(), 264, 1, 2, 200, 64, 0.1, 0, s) == -3     # head_dim 64
    # misaligned pointers and pitches
    assert lib.b2f_attention_fp8(p[0] + 8, p[1], p[2], p[3], p[4], p[5], out.data_ptr(), 264, 1, 2, 200, 128,
                                 0.1, 0, s) == -4
    assert lib.b2f_attention_fp8(*p, out.data_ptr() + 2, 264, 1, 2, 200, 128, 0.1, 0, s) == -4
    assert lib.b2f_attention_fp8(*p, out.data_ptr(), 260, 1, 2, 200, 128, 0.1, 0, s) == -4
    qp = q.data_ptr()
    assert lib.b2f_attn_quant_fp8(qp + 2, 768, k.data_ptr(), 768, v.data_ptr(), 768, *p, 1, 2, 200, 128, s) == -4
    assert lib.b2f_attn_quant_fp8(qp, 765, k.data_ptr(), 768, v.data_ptr(), 768, *p, 1, 2, 200, 128, s) == -4
    assert lib.b2f_attn_quant_fp8(qp, 768, k.data_ptr(), 768, v.data_ptr(), 768, p[0], p[1], p[2], p[3], p[4] + 4, p[5],
                                  1, 2, 200, 128, s) == -4
    # buffers that do not match the operands raise instead of being written past
    names = ("q8", "k8", "sq", "sk", "v8t", "sv")
    bad = {"q8": torch.empty(1, 199, 2, 128, device="cuda", dtype=Q.E4M3), "sk": torch.empty(1, 1, device="cuda"),
           "v8t": torch.empty(1, 2, 128, 128, device="cuda", dtype=Q.E4M3), "sv": torch.empty(1, 2, 64, device="cuda")}
    for n, t in bad.items():
        with pytest.raises(_lib.B2FError):
            ops.attn_quant_fp8(q, k, v, **(dict(zip(names, bufs)) | {n: t}))
    with pytest.raises(_lib.B2FError):
        ops.attention_fp8(*bufs, out=torch.empty(1, 100, 256, device="cuda", dtype=bf16))


# ---------------------------------------------------------------------------------------------------- the model
def _model_inputs(s):
    return dict(hidden_states=s.hs, encoder_hidden_states=s.enc, pooled_projections=s.pooled, timestep=s.t,
                img_ids=s.img_ids, txt_ids=s.txt_ids, guidance=s.gd, return_dict=False)


@pytest.mark.parametrize("linears", [False, True])
def test_fp8_attention_forward_stagewise(linears):
    """Each block's output against the fp64 FP8 emulation (fp8_attention(), with fp8_linears() when the linears run in
    FP8 too) from the engine's own input to that block, at d = 3072 with ragged S_txt / S_img and B = 2."""
    import contextlib

    s = _setup(*CASES["ragged"])
    s.model.enable_fp8(linears=linears, attention=True)
    _, mod, _ = _temb_mod(s, s.t, s.gd, s.pooled)
    _fwd(s, (0, 0))
    h = s.model.debug_buffers(s.B, s.S_img, s.S_txt).h.clone()
    checks = []
    d = s.ocfg.inner_dim
    for blk in range(s.nblk):
        h_in = h
        _fwd(s, (blk, blk + 1))
        bufs = s.model.debug_buffers(s.B, s.S_img, s.S_txt)
        K = {"h": bufs.h.clone(), "qkv": bufs.qkv.clone(), "attn": bufs.cat[..., :d].clone(),
             "mlp": bufs.cat[..., d:].clone()}
        h = K["h"]
        if blk < s.ocfg.num_layers:
            name, f = f"double{blk}", (lambda sd, dt: IB.double_stage(sd, s.ocfg, blk, h_in, mod, s.cos, s.sin,
                                                                       s.S_txt, dt))
        else:
            si = blk - s.ocfg.num_layers
            name, f = f"single{si}", (lambda sd, dt: IB.single_stage(sd, s.ocfg, si, h_in, mod, s.cos, s.sin, dt))
        with A.fp8_attention(), (Q.fp8_linears() if linears else contextlib.nullcontext()):
            Rf, Yf = f(s.sd, f64), f(s.sd, bf16)
        checks += IB.token_gates(name, "h", K["h"], Rf["h"], Yf["h"], s.S_txt, base=h_in)
        for n in ("qkv", "attn"):
            checks += IB.token_gates(name, n, K[n], Rf[n], Yf[n], s.S_txt, heads=True)
        checks += IB.token_gates(name, "mlp", K["mlp"], Rf["mlp"], Yf["mlp"], s.S_txt)
        del K, Rf, Yf
    bad = _report(f"fp8 attention stagewise (linears {linears})", s, checks)
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("linears", [False, True])
def test_fp8_attention_forward_quality_gate(linears):
    """rel-L2 of the engine with FP8 attention (and FP8 linears) to the fp64 unquantized forward <= E_emu (fp64 emulation
    of the same scheme vs fp64) + E_bf16 (the bf16 engine vs fp64); inputs as in test_fp8_forward_quality_gate."""
    import contextlib

    s = _setup(*CASES["ragged"])
    s.gd = torch.tensor([4.0, 2.0], device="cuda")
    for x in (s.t, s.gd):
        assert torch.equal(s.model._times1000(x).double(), x.double() * 1000), "x1000 not exact in bf16"
    out_bf16 = s.model(**_model_inputs(s))[0].clone()
    s.model.enable_fp8(linears=linears, attention=True)
    out_fp8 = s.model(**_model_inputs(s))[0].clone()
    sd64 = {k: v.double() for k, v in s.sd.items()}
    args = (s.hs.double(), s.enc.double(), s.pooled.double(), s.t, s.img_ids, s.txt_ids)
    ref = fo.flux_forward(sd64, s.ocfg, *args, guidance=s.gd)
    with A.fp8_attention(), (Q.fp8_linears() if linears else contextlib.nullcontext()):
        emu = fo.flux_forward(sd64, s.ocfg, *args, guidance=s.gd)
    e_emu, e_bf16, e_fp8 = R.rel_l2(emu, ref), R.rel_l2(out_bf16, ref), R.rel_l2(out_fp8, ref)
    print(f"KREF fp8 attention quality (linears {linears}): E_emu={e_emu:.4g} E_bf16={e_bf16:.4g} "
          f"engine={e_fp8:.4g} (engine vs emulation {R.rel_l2(out_fp8, emu):.4g})")
    assert e_fp8 <= e_emu + e_bf16


def test_fp8_attention_switching():
    """enable -> disable gives the never-enabled bits; the workspace grows only while the switch is on; an unfused LoRA
    adapter runs with FP8 attention and matches fp8_attention() over the LoRA oracle; training is refused."""
    import lora_ref as LR
    from gpt_image_edit_b200 import _lib
    from gpt_image_edit_b200.training import FluxTrainGraph

    s = _setup(*CASES["toy_text_of_one"])
    m, inp = s.model, _model_inputs(s)
    lib, h = _lib.lib, m._h
    ws = lambda: int(lib.b2f_flux_workspace_bytes(h, s.B, s.S_img, s.S_txt))
    base, ws0 = m(**inp)[0].clone(), ws()
    m.enable_fp8(linears=False, attention=True)
    assert m.fp8_attention_enabled and not m.fp8_enabled
    S, d, H = s.S_img + s.S_txt, s.ocfg.inner_dim, s.ocfg.num_attention_heads
    assert ws() == ws0 + s.B * d * (2 * S + A.s_pad(S)) + s.B * (2 * H + d) * 4 + 256
    f8 = m(**inp)[0].clone()
    assert not torch.equal(f8, base)
    m.disable_fp8()
    assert not m.fp8_attention_enabled and ws() == ws0 and torch.equal(m(**inp)[0], base)
    m.enable_fp8()                                           # linears only: attention stays bf16
    assert m.fp8_enabled and not m.fp8_attention_enabled
    m.disable_fp8()

    # an unfused adapter with FP8 attention, against fp8_attention() over the fp64 oracle on merged weights, in the form
    # of the quality gate: E_engine <= E_emu + E_bf16 (E_bf16: the same adapter with bf16 attention)
    la = LR.make_lora(s.ocfg, rank=8, seed=3, alpha=16.0, a_std=0.03, b_std=0.03)
    m.load_lora_adapter(LR.to_diffusers(la), adapter_name="a")
    out_bf16 = m(**inp)[0].clone()
    m.enable_fp8(linears=False, attention=True)
    assert m.lora_unfused_active()
    out = m(**inp)[0].clone()
    sd64 = LR.merged({k: v.double() for k, v in s.sd.items()}, [(la, 1.0)])
    args = (s.hs.double(), s.enc.double(), s.pooled.double(), s.t, s.img_ids, s.txt_ids)
    ref = fo.flux_forward(sd64, s.ocfg, *args, guidance=s.gd)
    with A.fp8_attention():
        emu = fo.flux_forward(sd64, s.ocfg, *args, guidance=s.gd)
    e_emu, e_bf16, e_eng = R.rel_l2(emu, ref), R.rel_l2(out_bf16, ref), R.rel_l2(out, ref)
    print(f"KREF fp8 attention + unfused LoRA: E_emu={e_emu:.4g} E_bf16={e_bf16:.4g} engine={e_eng:.4g} "
          f"(engine vs emulation {R.rel_l2(out, emu):.4g})")
    assert e_eng <= e_emu + e_bf16
    m.unload_lora()

    # training refuses while FP8 attention is on
    den = type("Tower", (), {})()
    den.denoiser = m
    model = type("M", (), {})()
    model.denoise_tower = den
    with pytest.raises(_lib.B2FError, match="disable_fp8"):
        FluxTrainGraph(model, [])
    m.disable_fp8()
