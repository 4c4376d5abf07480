"""The FLUX inference forward (`b2f_flux_forward`) checked stage by stage, at the 1024^2 edit's widths and lengths and at
ragged ones, against float64 references of the oracle per token, per channel, per head and per modulation chunk.

The module's own forward is driven one stage per call with `_b2f_block_range`: `(0, 0)` runs the embedders, `(blk,
blk + 1)` one block, `(nblk, nblk)` the tail (norm_out + proj_out over the first n_out image rows).  After every call
the joint activation buffer and the intermediates the block left in the workspace are read through `debug_buffers`.
silu(temb) and `mod` come from `_temb_mod` and are stages of their own, and so are the rows of hoisted schedules.  Each
stage is compared with its float64 reference (tests/infer_block_ref.py) fed with the engine's bf16 inputs to that
stage, with torch-bf16 of the same stage as the yardstick: the per-tensor rule rel-L2(engine) <= 2 rel-L2(bf16) + 1e-2
and the per-slice gate max_s e_s <= 2 max_s y_s + 1e-3 (`infer_block_ref.BETA`).  Block outputs are also gated as the
block's own share, h_out - h_in.

Exact checks, bit for bit: the stage-by-stage forward equals one call; a forward into a NaN-filled workspace equals one
into a zero-filled workspace; an n_out < S_img output is the first n_out rows of the n_out = S_img one; batch item b of
a batched forward is the forward of that item alone.
"""
import contextlib
from types import SimpleNamespace

import pytest
import torch

import infer_block_ref as IB
import lora_ref as LR
from oracle import flux_oracle as fo
from test_flux_gpu import _heavy_tailed
from test_train_blocks_gpu import _ids, _synthetic_sd

pytestmark = pytest.mark.gpu

f64, bf16 = torch.float64, torch.bfloat16
FULL = dict(attention_head_dim=128, num_attention_heads=24, joint_attention_dim=4096, pooled_projection_dim=768)
TOYW = dict(attention_head_dim=128, num_attention_heads=2, joint_attention_dim=256, pooled_projection_dim=64)

# name: (width, B, S_txt, latent h, w, n_out, double, single, heavy q/k, LoRA)
CASES = {
    "c1024": (FULL, 1, 544, 64, 64, 4096, 2, 2, False, False),        # the edit's shapes: S = 8736, the GEMMs bench.py times
    "ragged": (FULL, 2, 77, 9, 10, 90, 2, 2, False, False),           # B = 2, S_txt % 8 != 0, S = 257 = 2 * 128 + 1
    "ragged_heavy": (FULL, 2, 77, 9, 10, 90, 2, 2, True, False),      # peaked attention rows
    "full_depth": (FULL, 1, 32, 8, 8, 64, 19, 38, False, False),      # every modulation offset of the real model
    "toy_text_of_one": (TOYW, 3, 1, 8, 8, 64, 2, 2, False, False),    # text GEMMs with M = 1, B = 3, S = 129
    "ragged_lora": (FULL, 2, 77, 9, 10, 90, 2, 2, False, True),       # two unfused adapters on every target
}


def _setup(width, B, S_txt, hl, wl, n_out, nd, ns, heavy, lora, seed=0):
    from gpt_image_edit_b200.flux_transformer import B200FluxTransformer2DModel, FluxTransformerConfig

    kw = dict(width, num_layers=nd, num_single_layers=ns)
    ocfg = fo.FluxConfig(**kw)
    model = B200FluxTransformer2DModel(FluxTransformerConfig(**kw))
    sd = _synthetic_sd(ocfg, seed)
    if heavy:
        sd = _heavy_tailed(sd, ocfg)
    model.load_state_dict(sd)
    del sd                       # the model's own storage serves as the bf16 state dict (24 GB at full depth)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    S_img = 2 * hl * wl
    s = SimpleNamespace(
        ocfg=ocfg, model=model, sd=model.state_dict(), sd64=None, yard=contextlib.nullcontext, B=B, S_txt=S_txt,
        S_img=S_img, S=S_txt + S_img, n_out=n_out, nblk=nd + ns, scale=None,
        hs=torch.randn(B, S_img, ocfg.in_channels, device="cuda", generator=g).bfloat16(),
        enc=torch.randn(B, S_txt, ocfg.joint_attention_dim, device="cuda", generator=g).bfloat16(),
        pooled=torch.randn(B, ocfg.pooled_projection_dim, device="cuda", generator=g).bfloat16(),
        t=torch.tensor([0.5, 0.25, 0.75][:B], device="cuda").bfloat16(),   # t * 1000 exact in bf16
        gd=torch.tensor([4.0, 3.5, 2.5][:B], device="cuda"),
        img_ids=_ids(hl, wl), txt_ids=torch.zeros(S_txt, 3, device="cuda", dtype=bf16))
    if lora:
        la = LR.make_lora(ocfg, rank=16, seed=11, alpha=32.0, a_std=0.03, b_std=0.03)
        lb = LR.make_lora(ocfg, rank=8, seed=12, alpha=None, a_std=0.03, b_std=0.03)
        model.load_lora_adapter(LR.to_diffusers(la), adapter_name="a")
        model.load_lora_adapter(LR.to_bfl(ocfg, lb), adapter_name="b")
        s.scale, wb = 0.6, 0.5
        model.set_adapters(["a", "b"], [1.0, wb])
        loras = [(la, s.scale), (lb, s.scale * wb)]
        s.sd64 = LR.merged(s.sd, loras)
        s.yard = lambda: LR.peft_linear(loras)
    ids = torch.cat([s.txt_ids.float(), s.img_ids.float()])
    s.cos, s.sin = fo.rope_tables(ids, ocfg.axes_dims_rope, ocfg.theta)
    return s


def _fwd(s, rng=(0, -1), n_out=None, inp=None):
    jak = {"_b2f_block_range": rng, "_b2f_out_rows": n_out or s.n_out}
    if s.scale is not None:
        jak["scale"] = s.scale
    i = inp or dict(hidden_states=s.hs, encoder_hidden_states=s.enc, pooled_projections=s.pooled, timestep=s.t,
                    guidance=s.gd)
    return s.model(**i, img_ids=s.img_ids, txt_ids=s.txt_ids, return_dict=False, joint_attention_kwargs=jak)[0]


def _bufs(s):
    b = s.model.debug_buffers(s.B, s.S_img, s.S_txt)
    d = s.ocfg.inner_dim
    return {"h": b.h.clone(), "xn": b.xn.clone(), "qkv": b.qkv.clone(), "attn": b.cat[..., :d].clone(),
            "mlp": b.cat[..., d:].clone()}


def _ref(s, f):
    """(float64 reference, torch-bf16 yardstick) of one stage: f(state dict, dtype)."""
    R = f(s.sd64 if s.sd64 is not None else s.sd, f64)
    with s.yard():
        Y = f(s.sd, bf16)
    return R, Y


def _temb_mod(s, t, g, pooled):
    m = s.model
    m._set_lora_scale(1.0 if s.scale is None else s.scale)
    return m._temb_mod(m._times1000(t), m._times1000(g), pooled, want_silu=True)


def _head_checks(s, t, g, pooled, stage):
    """temb, silu(temb) and mod of rows (t, g, pooled) against their references."""
    temb, mod, stemb = _temb_mod(s, t, g, pooled)
    m = s.model
    R, Y = _ref(s, lambda sd, dt: IB.temb_stage(sd, s.ocfg, m._times1000(t), m._times1000(g), pooled, dt))
    out = IB.row_gates(stage, "temb", temb, R["temb"], Y["temb"])
    out += IB.row_gates(stage, "silu(temb)", stemb, R["silu"], Y["silu"])
    R, Y = _ref(s, lambda sd, dt: IB.modulation_stage(sd, s.ocfg, stemb, dt))
    return out + IB.mod_gates(stage, mod, R["mod"], Y["mod"], s.ocfg), mod


def _report(case, s, checks):
    print(f"\n[{case}] d={s.ocfg.inner_dim} B={s.B} S_txt={s.S_txt} S_img={s.S_img} n_out={s.n_out} blocks={s.nblk}")
    print("\n".join(str(c) for c in checks))
    return [str(c) for c in checks if not c.ok]


@pytest.mark.parametrize("case", list(CASES))
def test_stagewise_forward_matches_fp64(case):
    s = _setup(*CASES[case])
    checks, mod = _head_checks(s, s.t, s.gd, s.pooled, "head")

    # embedders
    _fwd(s, (0, 0))
    h = s.model.debug_buffers(s.B, s.S_img, s.S_txt).h.clone()
    R, Y = _ref(s, lambda sd, dt: IB.embed_stage(sd, s.hs, s.enc, dt))
    checks += IB.token_gates("embed", "h", h, R["h"], Y["h"], s.S_txt)
    # blocks
    for blk in range(s.nblk):
        h_in = h
        _fwd(s, (blk, blk + 1))
        K = _bufs(s)
        h = K["h"]
        if blk < s.ocfg.num_layers:
            name = f"double{blk}"
            f = lambda sd, dt: IB.double_stage(sd, s.ocfg, blk, h_in, mod, s.cos, s.sin, s.S_txt, dt)
        else:
            si = blk - s.ocfg.num_layers
            name = f"single{si}"
            f = lambda sd, dt: IB.single_stage(sd, s.ocfg, si, h_in, mod, s.cos, s.sin, dt)
        R, Y = _ref(s, f)
        if blk == s.nblk - 1:
            # this call ran the tail too: norm_out overwrote xn's first n_out image rows (the tail's own check reads
            # them), so the block's xn is gated over the rest; its image labels count from token n_out
            keep = torch.cat([torch.arange(s.S_txt), torch.arange(s.S_txt + s.n_out, s.S)]).cuda()
            for D in (K, R, Y):
                D["xn"] = D["xn"][:, keep]
        checks += IB.block_gates(name, K, R, Y, h_in, s.S_txt)
        del K, R, Y
    # tail
    out = _fwd(s, (s.nblk, s.nblk)).clone()
    xn = s.model.debug_buffers(s.B, s.S_img, s.S_txt).xn[:, s.S_txt:s.S_txt + s.n_out].clone()
    R, Y = _ref(s, lambda sd, dt: IB.tail_stage(sd, s.ocfg, h, mod, s.S_txt, s.n_out, dt))
    checks += IB.token_gates("tail", "xn", xn, R["xn"], Y["xn"], 0)
    checks += IB.token_gates("tail", "out", out, R["out"], Y["out"], 0)
    del R, Y
    bad = _report(case, s, checks)

    # bit for bit: one call, into a NaN-filled and into a zero-filled workspace, gives the stage-by-stage result
    ws = s.model._ws["fwd"]
    for fill in (255, 0):                 # 0xffff is a bf16 NaN
        ws.fill_(fill)
        full = _fwd(s).clone()
        assert torch.equal(full, out), f"one forward call into a workspace of bytes {fill:#x} != the stagewise forward"
        assert torch.equal(s.model.debug_buffers(s.B, s.S_img, s.S_txt).h, h), f"final h (workspace bytes {fill:#x})"
    # the n_out rows of the target are the first rows of the whole image's output
    if s.n_out < s.S_img:
        assert torch.equal(_fwd(s, n_out=s.S_img)[:, :s.n_out], out)
    # every launch is row- or (batch, head)-independent: batch item b alone gives the same bits
    if s.B > 1:
        for b in range(s.B):
            one = dict(hidden_states=s.hs[b:b + 1], encoder_hidden_states=s.enc[b:b + 1],
                       pooled_projections=s.pooled[b:b + 1], timestep=s.t[b:b + 1], guidance=s.gd[b:b + 1])
            assert torch.equal(_fwd(s, inp=one), out[b:b + 1]), f"batch item {b} alone"
    assert not bad, f"[{case}] " + "\n".join(bad)


@pytest.mark.parametrize("steps", [28, 65])
def test_hoisted_schedule_rows_match_fp64(steps):
    """The modulation of a whole schedule (prepare_schedule: M = steps x B rows, 56 and 130 here) against its reference:
    the AdaLN GEMM at M past one 128-row tile, and every row in (step, batch) order."""
    s = _setup(*CASES["ragged"])
    ts = (torch.linspace(1.0, 1.0 / steps, steps, device="cuda") * 1000).bfloat16() / 1000
    sched = s.model.prepare_schedule(ts, s.gd, s.pooled)
    t = ts.reshape(steps, 1).expand(steps, s.B).reshape(-1)
    g = s.gd.reshape(1, s.B).expand(steps, s.B).reshape(-1)
    pooled = s.pooled.repeat(steps, 1).contiguous()
    checks, mod = _head_checks(s, t, g, pooled, f"M={steps * s.B}")
    assert torch.equal(sched.mod.reshape(steps * s.B, -1), mod)
    bad = _report(f"schedule {steps} steps", s, checks)
    assert not bad, "\n".join(bad)
