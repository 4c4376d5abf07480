"""The FLUX training backward (`b2f_flux_train_backward`) checked stage by stage, at the widths and lengths of the
training workload and at ragged ones, against float64 autograd of the oracle per token, per channel and per element.

The backward is driven directly on the context and workspace of a `FluxTrainGraph` after its forward, one stage per
call: the tail (norm_out + proj_out), then each block from the last to block 0 (whose call also writes d_enc), reading
the residual-stream gradient dh after every call.  Each stage is compared with its own float64 reference
(tests/train_block_ref.py) fed with the engine's bf16 inputs to that stage: the block input from the inference path
(`_b2f_block_range=(0, blk)`, so the training checkpoints are checked too), the engine's dh from the previous stage, and
`mod` / silu(temb) from the graph.  The graph's own backward then supplies d_enc to MLP2, which is checked the same way.

Every gradient passes two gates against the same reference, with torch-bf16 autograd of the same stage as yardstick:
the per-tensor rule rel-L2(engine) <= 2 rel-L2(bf16) + 1e-2, and the per-slice gate max_s e_s <= 2 max_s y_s + 1e-2 over
token rows, weight rows and columns, modulation chunks and single bias / norm elements.
"""
from types import SimpleNamespace

import pytest
import torch

import train_block_ref as TB
from oracle import flux_oracle as fo
from test_flux_gpu import _heavy_tailed
from test_train_flux_gpu import _ref_for

pytestmark = pytest.mark.gpu

FULL = dict(attention_head_dim=128, num_attention_heads=24, joint_attention_dim=4096, pooled_projection_dim=768)
TOYW = dict(attention_head_dim=128, num_attention_heads=2, joint_attention_dim=256, pooled_projection_dim=64)

# name: (width, B, S_txt, latent h, w, n_out, heavy, VLM width)
CASES = {
    "bench": (FULL, 1, 288, 32, 32, 1024, False, 3584),     # the train512 workload: S = 2336, S_pad 2432
    "ragged": (FULL, 2, 77, 9, 10, 90, False, 3584),        # S_txt % 8 != 0, S = 257 = 2*128 + 1
    "ragged_heavy": (FULL, 2, 77, 9, 10, 90, True, 3584),   # peaked attention rows in the backward
    "toy_width": (TOYW, 2, 1, 8, 8, 64, False, 128),        # d = 256, text GEMMs with M = 1, S = 129
}


def _synthetic_sd(ocfg, seed):
    """make_synthetic_state_dict's distributions, drawn on the device (the full-width stacks hold ~1e9 weights); norm
    weights and AdaLN biases non-trivial so that every gradient path carries signal."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    sd = {}
    for name, shape in fo.state_dict_spec(ocfg).items():
        t = torch.randn(shape, device="cuda", generator=g)
        if "norm_q" in name or "norm_k" in name or "norm_added" in name:
            t = 1.0 + 0.2 * t
        else:
            t = t * 0.02
        sd[name] = t.bfloat16()
    return sd


def _ids(h, w):
    ids = torch.zeros(h, w, 3)
    ids[..., 1] += torch.arange(h)[:, None]
    ids[..., 2] += torch.arange(w)[None, :]
    ids = ids.reshape(-1, 3)
    ctx = ids.clone()
    ctx[:, 0] = 1
    return torch.cat([ids, ctx]).to("cuda", torch.bfloat16)


def _setup(width, B, S_txt, hl, wl, n_out, heavy, vlm, nd=2, ns=2, seed=0):
    from gpt_image_edit_b200 import training as tr
    from gpt_image_edit_b200.flux_transformer import B200FluxTransformer2DModel, FluxTransformerConfig
    from univa.models.modeling_univa_denoise_tower import DenoiseProjector

    kw = dict(width, num_layers=nd, num_single_layers=ns)
    ocfg = fo.FluxConfig(**kw)
    sd = _synthetic_sd(ocfg, seed)
    if heavy:
        sd = _heavy_tailed(sd, ocfg)
    den = B200FluxTransformer2DModel(FluxTransformerConfig(**kw))
    den.load_state_dict(sd)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    proj = DenoiseProjector(vlm, ocfg.joint_attention_dim)
    for t in proj.state_dict().values():
        t.copy_((torch.randn(t.shape, device="cuda", generator=g) * 0.02).bfloat16())
    model = SimpleNamespace(denoise_tower=SimpleNamespace(denoiser=den, denoise_projector=proj))
    params = tr.trainable_params(model)
    for p in params:
        p.grad = torch.zeros(p.storage.shape, device="cuda", dtype=torch.float32)
    S_img = 2 * hl * wl
    return SimpleNamespace(
        ocfg=ocfg, sd=sd, den=den, proj=proj, model=model, params=params, B=B, S_txt=S_txt, S_img=S_img, S=S_txt + S_img,
        n_out=n_out, nblk=nd + ns,
        x=torch.randn(B, S_txt, vlm, device="cuda", generator=g).bfloat16(),
        hs=torch.randn(B, S_img, 64, device="cuda", generator=g).bfloat16(),
        pooled=torch.randn(B, ocfg.pooled_projection_dim, device="cuda", generator=g).bfloat16(),
        img_ids=_ids(hl, wl),
        t=torch.tensor([0.5, 0.25][:B], device="cuda").bfloat16(),       # per-item timesteps, t * 1000 exact in bf16
        gd=torch.full((B,), 1.0, device="cuda"),                          # the training config's guidance
        target=torch.randn(B, n_out, 64, device="cuda", generator=g))


def _graph(s):
    from gpt_image_edit_b200 import training as tr
    graph = tr.FluxTrainGraph(s.model, s.params)
    pred = graph.forward(s.x, s.hs, s.t, s.gd, s.pooled, s.img_ids, s.n_out)
    _, dpred = tr.flow_matching_loss(pred, s.target)
    return graph, dpred


def _stage(graph, dpred, d_enc, first, last, accumulate=0):
    from gpt_image_edit_b200 import _lib
    c, h = graph._ctx, graph.den._h
    _lib.check(_lib.lib.b2f_flux_train_backward(
        h, _lib.ptr(dpred), _lib.ptr(c["mod"]), c["mod"].stride(0), _lib.ptr(c["stemb"]), c["stemb"].stride(0),
        _lib.ptr(d_enc), c["B"], c["S_img"], c["S_txt"], c["n_out"], accumulate, _lib.ptr(c["ws"]), c["nws"], first, last,
        _lib.stream_ptr()), f"backward ({first}, {last})")


def _dh(graph):
    from gpt_image_edit_b200 import _lib
    c = graph._ctx
    dst = torch.empty(c["B"], c["S_img"] + c["S_txt"], graph.den.inner_dim, device="cuda", dtype=torch.bfloat16)
    _lib.check(_lib.lib.b2f_flux_train_debug_dh(graph.den._h, _lib.ptr(dst), c["B"], c["S_img"], c["S_txt"],
                                                _lib.ptr(c["ws"]), _lib.stream_ptr()), "debug_dh")
    return dst


def _stagewise(graph, dpred, s):
    """tail, then every block from the last to 0, one call each: ({stage: dh after it}, d_enc)."""
    d_enc = torch.full((s.B, s.S_txt, s.ocfg.joint_attention_dim), float("nan"), device="cuda", dtype=torch.bfloat16)
    dh = {}
    _stage(graph, dpred, d_enc, s.nblk, s.nblk)
    dh["tail"] = _dh(graph)
    for blk in range(s.nblk - 1, -1, -1):
        if blk == 0:
            assert torch.isnan(d_enc.float()).all(), "d_enc written before the block-0 call"
        _stage(graph, dpred, d_enc, blk, blk + 1)
        dh[blk] = _dh(graph)
    return dh, d_enc


def _h_in(s, blk):
    """the block input h of block `blk` (blk = nblk: the input of norm_out) from the inference path."""
    txt_ids = torch.zeros(s.S_txt, 3, device="cuda", dtype=torch.bfloat16)
    s.den(hidden_states=s.hs, encoder_hidden_states=s.enc, pooled_projections=s.pooled, timestep=s.t, img_ids=s.img_ids,
          txt_ids=txt_ids, guidance=s.gd, return_dict=False,
          joint_attention_kwargs={"_b2f_block_range": (0, blk), "_b2f_out_rows": s.n_out})
    return s.den.debug_hidden(s.B, s.S_img, s.S_txt).clone()


def _block_params(s, blk):
    return [p for p in s.params if p.bucket == blk]


def _param_gates(stage, s, ps, grads, r64, r16):
    d, hd = s.ocfg.inner_dim, s.ocfg.attention_head_dim
    out = []
    for p in ps:
        ref, yard = _ref_for(p.name, r64, {}), _ref_for(p.name, r16, {})
        short = p.name.split(".", 2)[2]
        if p.name.endswith("linear.weight"):
            names = TB.CHUNKS["double" if p.name.startswith("transformer_blocks") else "single"]
            out += TB.gate(stage, short, grads[p.name], ref, yard, ("chunks",), TB.chunk_label(names), n_chunks=len(names))
        elif p.name.endswith(".weight") and p.grad.dim() == 2:
            lab = TB.qkv_label(d, hd) if "to_q|to_k|to_v" in p.name else None
            out += TB.gate(stage, short, grads[p.name], ref, yard, ("rows", "cols"), lab)
        else:
            out += TB.gate(stage, short, grads[p.name], ref, yard, ("elems",))
    return out


@pytest.mark.parametrize("case", list(CASES))
def test_stagewise_backward_matches_fp64(case):
    s = _setup(*CASES[case])
    graph, dpred = _graph(s)
    s.enc = graph._ctx["enc"]
    mod, stemb = graph._ctx["mod"], graph._ctx["stemb"]

    # stage by stage, into NaN-filled gradient buffers: accumulate=0 must write every element
    for p in s.params:
        p.grad.fill_(float("nan"))
    dh, d_enc = _stagewise(graph, dpred, s)
    grads = {p.name: p.grad.clone() for p in s.params if p.bind_key is not None}
    for n, g in grads.items():
        assert torch.isfinite(g).all(), f"{n}: elements left unwritten"
    assert torch.isfinite(d_enc.float()).all()
    # the tail writes only the image rows of the target tokens
    tail = dh["tail"]
    assert not tail[:, :s.S_txt].any() and not tail[:, s.S_txt + s.n_out:].any()

    # one call over every stage, into zero-filled buffers, then MLP2: the same bits
    for p in s.params:
        p.grad.zero_()
    d_enc_full = graph.backward(dpred)
    torch.cuda.synchronize()
    assert torch.equal(d_enc_full, d_enc)
    for p in s.params:
        if p.bind_key is not None:
            assert torch.equal(p.grad, grads[p.name]), p.name
    mlp2 = {p.name: p.grad.clone() for p in s.params if p.bind_key is None}

    ids = torch.cat([torch.zeros(s.S_txt, 3, device="cuda"), s.img_ids.float()])
    cos, sin = fo.rope_tables(ids, s.ocfg.axes_dims_rope, s.ocfg.theta)
    checks = []

    # tail
    h_fin = _h_in(s, s.nblk)
    r = [TB.tail_stage(s.sd, s.ocfg, h_fin, dpred, mod, s.S_txt, s.n_out, dt)["dh"] for dt in (torch.float64, torch.bfloat16)]
    checks += TB.dh_gates("tail", tail, *r, None, s.B, s.S_txt)
    dh_out = tail
    # blocks, last to first
    for blk in range(s.nblk - 1, -1, -1):
        h_in = _h_in(s, blk)
        if blk < s.ocfg.num_layers:
            f = lambda dt: TB.double_stage(s.sd, s.ocfg, blk, h_in, dh_out, mod, stemb, cos, sin, s.S_txt, dt)
            name = f"double{blk}"
        else:
            si = blk - s.ocfg.num_layers
            f = lambda dt: TB.single_stage(s.sd, s.ocfg, si, h_in, dh_out, mod, stemb, cos, sin, dt)
            name = f"single{si}"
        r64, r16 = f(torch.float64), f(torch.bfloat16)
        checks += TB.dh_gates(name, dh[blk], r64["dh"], r16["dh"], dh_out, s.B, s.S_txt)
        checks += _param_gates(name, s, _block_params(s, blk), grads, r64, r16)
        dh_out = dh[blk]
        del r64, r16
    # head: d_enc from the engine's dh after block 0
    r = [TB.head_stage(s.sd, dh[0], s.S_txt, dt) for dt in (torch.float64, torch.bfloat16)]
    checks += TB.gate("head", "d_enc", d_enc, *r, ("rows",), TB.token_label(s.B, s.S_txt, s.S_txt))
    # MLP2 from the engine's d_enc
    pw = s.proj.state_dict()
    r = [TB.mlp2_stage(pw, s.x, d_enc, dt) for dt in (torch.float64, torch.bfloat16)]
    for p in s.params:
        if p.bind_key is None:
            k = p.name[len("denoise_projector."):]
            kinds = ("rows", "cols") if k.endswith("weight") else ("elems",)
            checks += TB.gate("mlp2", k, mlp2[p.name], r[0][k], r[1][k], kinds)

    print(f"\n[{case}] d={s.ocfg.inner_dim} B={s.B} S_txt={s.S_txt} S_img={s.S_img} n_out={s.n_out}")
    print("\n".join(str(c) for c in checks))
    bad = [str(c) for c in checks if not c.ok]
    assert not bad, f"[{case}] " + "\n".join(bad)


def _bound_run(s, graph, dpred, fill):
    for p in s.params:
        p.grad.fill_(fill)
    dh, d_enc = _stagewise(graph, dpred, s)
    return dh, d_enc, {p.name: p.grad.clone() for p in s.params if p.bind_key is not None}


def test_partial_binding_changes_nothing_else():
    """Unbinding norm_q / norm_k of a double block (its RMSNorm backward then writes no weight partials) and every
    gradient of a single block leaves every other gradient and every stage's dh unchanged, bit for bit."""
    from gpt_image_edit_b200 import _lib

    s = _setup(*CASES["toy_width"])
    graph, dpred = _graph(s)
    dh0, d_enc0, g0 = _bound_run(s, graph, dpred, 0.0)
    dropped = {"transformer_blocks.1.attn.norm_q.weight", "transformer_blocks.1.attn.norm_k.weight"}
    dropped |= {p.bind_key for p in s.params if p.bind_key and p.bind_key.startswith("single_transformer_blocks.0.")}
    for k in dropped:
        _lib.check(_lib.lib.b2f_flux_bind_grad(graph.den._h, k.encode(), None, 0), f"unbind {k}")
    dh1, d_enc1, g1 = _bound_run(s, graph, dpred, 7.0)
    assert torch.equal(d_enc1, d_enc0)
    for k in dh0:
        assert torch.equal(dh1[k], dh0[k]), f"dh after stage {k}"
    keys = {p.name: p.bind_key for p in s.params if p.bind_key}
    for n, g in g1.items():
        if keys[n] in dropped:
            assert (g == 7.0).all(), f"{n}: unbound gradient was written"
        else:
            assert torch.equal(g, g0[n]), n


def test_accumulate_adds_to_every_buffer():
    """accumulate=1 onto random fp32 contents P gives P + G0 to within one fp32 rounding of the sum, per element, where G0
    is the accumulate=0 result: every kernel that writes a gradient (wgrad, bias and norm column sums, the AdaLN outer
    product, MLP2) reads what is there."""
    s = _setup(*CASES["toy_width"])
    graph, dpred = _graph(s)
    for p in s.params:
        p.grad.zero_()
    graph.backward(dpred)
    g0 = {p.name: p.grad.clone() for p in s.params}
    gen = torch.Generator(device="cuda").manual_seed(3)
    pre = {}
    for p in s.params:
        scale = g0[p.name].abs().max().clamp_min(1e-30)
        pre[p.name] = torch.randn(p.grad.shape, device="cuda", generator=gen) * scale
        p.grad.copy_(pre[p.name])
    graph.backward(dpred, accumulate=True)
    torch.cuda.synchronize()
    for p in s.params:
        P, G0 = pre[p.name].double(), g0[p.name].double()
        err = (p.grad.double() - (P + G0)).abs()
        bound = 2.0 ** -22 * (P.abs() + G0.abs())
        worst = int((err - bound).argmax())
        assert (err <= bound).all(), f"{p.name}: element {worst} err {err.view(-1)[worst]:.3e} bound {bound.view(-1)[worst]:.3e}"
