"""The Qwen2.5-VL conditioning path (gpt_image_edit_b200/qwen2p5vl.py) checked stage by stage at full width and reduced
depth against float64 references of the oracle per token, per channel, per attention window and per head
(tests/qwen_stage_ref.py), at the ragged image grids the processor makes of real photos and at padded prompt batches.

Every stage runs through the engine's own methods (`_vision_embed`, `_vision_block`, `_vision_merge`, `_decoder_layer`,
`_decode_step`'s pieces); its reference is fed the engine's input to that stage, with torch-bf16 of the same stage as the
yardstick: the per-tensor rule rel-L2(engine) <= 2 rel-L2(bf16) + 1e-2 and the per-slice gate max_s e_s <= 2 max_s y_s +
1e-3.  Exact checks: the stagewise run is the one call bit for bit, the padding slots of the ViT's 128-wide heads and
3424-wide MLP stay zero, the KV cache holds the post-RoPE K / V, a decode step writes only its own cache row and reads
nothing outside [lo, past], and a padded prompt's padding rows get a zero attention output.
"""
import pytest
import torch

import qwen_stage_ref as QS
import vae_stage_ref as VS
from oracle import qwen_oracle as qo

pytestmark = pytest.mark.gpu

f64, bf16 = torch.float64, torch.bfloat16
IMG, VSTART, VEND = 151655, 151652, 151653


def _cfgs(depth=4, full=(1, 3), layers=2, vocab=152064, hidden=3584, vit_hidden=1280, vit_heads=16, vit_inter=3420,
          heads=28, kv=4, inter=18944):
    from gpt_image_edit_b200.qwen2p5vl import QwenTextConfig, QwenVisionConfig

    tc = QwenTextConfig(num_hidden_layers=layers, vocab_size=vocab, hidden_size=hidden, num_attention_heads=heads,
                        num_key_value_heads=kv, intermediate_size=inter)
    vc = QwenVisionConfig(depth=depth, fullatt_block_indexes=full, hidden_size=vit_hidden, num_heads=vit_heads,
                          intermediate_size=vit_inter, out_hidden_size=hidden)
    return tc, vc


def _model(tc, vc, seed=0):
    from gpt_image_edit_b200.qwen2p5vl import B200Qwen2p5VL

    sd = qo.make_synthetic_state_dict(tc, vc, seed=seed, dtype=bf16, device="cuda")
    m = B200Qwen2p5VL(tc, vc)
    m.load_state_dict(sd)
    return sd, m


def _pixels(grid, seed):
    T = sum(t * h * w for t, h, w in grid)
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(T, 1176, device="cuda", generator=g).bfloat16()


def _report(title, checks):
    print(f"\n[{title}]")
    print("\n".join(str(c) for c in checks))
    return [str(c) for c in checks if not c.ok]


def _summary(title, checks):
    """worst e / y and the smallest margin 2y + beta - e per tensor family"""
    fam = {}
    for c in checks:
        if c.kind == "tensor":
            continue
        k = f"{c.tensor} {c.kind}"
        r = c.e / c.y if c.y > 0 else 0.0
        m = 2 * c.y + QS.IB.BETA - c.e
        a, b = fam.get(k, (0.0, float("inf")))
        fam[k] = (max(a, r), min(b, m))
    print(f"\n[{title} summary] " + "; ".join(f"{k}: e/y {a:.2f} margin {b:.2e}" for k, (a, b) in sorted(fam.items())))


# ------------------------------------------------------------------------------------------------ vision tower
VIT = {
    "vit_448": ([(1, 32, 32)], 4, (1, 3)),                   # 16 windows of 64, full attention over 1024
    "vit_1000x1500": ([(1, 26, 38)], 4, (1, 3)),             # windows 64 / 48 / 16 / 12, full attention over 988
    "vit_1456x720": ([(1, 44, 22)], 4, (1, 3)),              # windows 64 / 48 / 32 / 24
    "vit_two_images": ([(1, 26, 38), (1, 2, 2)], 4, (1, 3)),  # a 4-patch image; two unequal full-attention segments
    "vit_full_depth": ([(1, 8, 12)], 32, (7, 15, 23, 31)),   # the real block schedule
}
TOY_VIT = dict(vit_hidden=1280, vit_heads=16, vit_inter=340, hidden=256, heads=2, kv=1, inter=512, vocab=1000)


def _vit_case(tc, vc, grid, seed=1):
    sd, m = _model(tc, vc, seed)
    pix = _pixels(grid, seed)
    nh, inter = vc.num_heads, vc.intermediate_size
    hd = vc.hidden_size // nh
    widx, cu_win, cu_full, _ = QS.vit_context(vc, grid)
    x, ctx = m._vision_embed(pix, grid)
    assert torch.equal(ctx.window_index, widx) and ctx.cu_win == cu_win and ctx.cu_full == cu_full
    checks = QS.vit_gates("embed", "x", x, QS.vit_embed_stage(sd, vc, pix, grid, f64),
                          QS.vit_embed_stage(sd, vc, pix, grid, bf16), cu_win)
    for i in range(vc.depth):
        x_in = x.clone()
        keep = {}
        m._vision_block(i, x, ctx, keep)
        for name, t in QS.vit_padding(keep, nh, inter, hd).items():
            assert not bool(t.any()), f"block {i}: {name} is not zero"
        R = QS.vit_block_stage(sd, vc, i, x_in, grid, f64)
        Y = QS.vit_block_stage(sd, vc, i, x_in, grid, bf16)
        cu = cu_full if i in vc.fullatt_block_indexes else cu_win
        st = f"vit {i}"
        checks += QS.vit_gates(st, "h", x, R["h"], Y["h"], cu, base=x_in)
        checks += QS.vit_gates(st, "qkv", QS.vit_qkv(keep["qkv"], nh, hd), R["qkv"], Y["qkv"], cu, heads=(3 * nh, hd))
        checks += QS.vit_gates(st, "attn", QS.vit_heads(keep["attn_out"], nh, hd), R["attn"], Y["attn"], cu, heads=(nh, hd))
        checks += QS.vit_gates(st, "a", QS.vit_mlp(keep["a"], inter), R["a"], Y["a"], cu)
        del R, Y
    keep = {}
    out = m._vision_merge(x, ctx, keep)
    R, Y = QS.vit_merge_stage(sd, vc, x, grid, f64), QS.vit_merge_stage(sd, vc, x, grid, bf16)
    checks += QS.TB.gate("merge", "merged", keep["merged"], R["merged"], Y["merged"], ("rows", "cols"), beta=QS.IB.BETA)
    assert torch.equal(out, keep["merged"][torch.argsort(widx).cuda()])
    assert torch.equal(m.forward_visual(pix, grid), out)
    return checks


@pytest.mark.parametrize("case", list(VIT))
def test_vit_stages_match_fp64(case):
    grid, depth, full = VIT[case]
    tc, vc = _cfgs(depth=depth, full=full, layers=0, vocab=1000)
    checks = _vit_case(tc, vc, grid)
    q = torch.randn(1, vc.num_heads, 64, 80, device="cuda", dtype=bf16)
    print(f"\nyardstick SDPA backend: {VS.sdpa_backend(q, q, q)}")
    _summary(case, checks)
    bad = _report(f"{case} grid {grid}", checks)
    assert not bad, "\n".join(bad)


def test_vit_stages_toy_width():
    """80-wide heads in 128-wide slots and an MLP of 340 (padded to 344) at two blocks: the launch shapes
    compute-sanitizer runs over.  The hidden width stays 1280: b2f_rmsnorm takes multiples of 256, and 1280 is the
    smallest that is also a multiple of 80."""
    tc, vc = _cfgs(**TOY_VIT, layers=0, depth=2, full=(1,))
    bad = _report("toy vit", _vit_case(tc, vc, [(1, 26, 38), (1, 2, 2)]))
    assert not bad, "\n".join(bad)


# ------------------------------------------------------------------------------------------------ decoder prefill
def _prompt(grids, text, tail, g):
    ids = torch.randint(1000, 150000, (text,), generator=g).tolist()
    for t, h, w in grids:
        ids += [VSTART] + [IMG] * (t * h * w // 4) + [VEND] + torch.randint(1000, 150000, (3,), generator=g).tolist()
    return ids + torch.randint(1000, 150000, (tail,), generator=g).tolist()


def _batch(rows, side, pad=151643):
    L = max(len(r) for r in rows)
    ids = torch.full((len(rows), L), pad, dtype=torch.long)
    mask = torch.zeros(len(rows), L, dtype=torch.long)
    for b, r in enumerate(rows):
        sl = slice(0, len(r)) if side == "right" else slice(L - len(r), L)
        ids[b, sl], mask[b, sl] = torch.tensor(r), 1
    return ids, mask


def _engine_prefill(m, ids, mask, pix, grid, cache=None, layer_cb=None):
    """forward() stage by stage: -> (final-norm hidden [B, L, d], image embeds, pos, deltas, spans)"""
    from gpt_image_edit_b200 import ops
    from gpt_image_edit_b200.qwen2p5vl import get_rope_index, padding_spans

    tc = m.tc
    B, L = ids.shape
    spans = None if mask is None or bool((mask == 1).all()) else padding_spans(mask)
    idc = ids.cuda()
    x = ops.gather_rows(m.W["model.embed_tokens"], idc.reshape(-1).contiguous())
    emb = None
    if pix is not None:
        emb = m.forward_visual(pix, grid)
        ops.scatter_rows_(x, (idc.reshape(-1) == IMG).nonzero().squeeze(1).contiguous(), emb)
    pos, deltas = get_rope_index(idc, torch.tensor(grid) if pix is not None else None, mask,
                                 image_token_id=IMG, vision_start_token_id=VSTART)
    cos, sin = m._rope_tables(pos)
    o = m._attn_buffer(B, L, 0, spans)
    for i in range(tc.num_hidden_layers):
        x_in = x.clone()
        keep = {}
        m._decoder_layer(i, x, o, cos, sin, B, L, cache, 0, spans, keep)
        if layer_cb is not None:
            layer_cb(i, x_in, x, keep)
    return ops.rmsnorm(x, m.W["model.norm"], eps=tc.rms_norm_eps).view(B, L, -1), emb, pos, deltas, spans


def _layer_gates(sd, tc, i, x_in, x, keep, pos, parts, spans, B, L):
    R = QS.decoder_stage(sd, tc, i, x_in.view(B, L, -1), pos, f64, spans)
    Y = QS.decoder_stage(sd, tc, i, x_in.view(B, L, -1), pos, bf16, spans)
    v3 = lambda t: t.view(B, L, -1)
    nq, nkv = tc.num_attention_heads, tc.num_key_value_heads
    st = f"dec {i}"
    c = QS.dec_gates(st, "h", v3(x), R["h"], Y["h"], parts, base=x_in.view(B, L, -1))
    c += QS.dec_gates(st, "qkv", v3(keep["qkv"]), R["qkv"], Y["qkv"], parts, heads=(QS.qkv_head_labels(nq, nkv), 128))
    c += QS.dec_gates(st, "attn", v3(keep["attn_out"]), R["attn"], Y["attn"], parts,
                      heads=([f"head {h}" for h in range(nq)], 128))
    c += QS.dec_gates(st, "a", v3(keep["a"]), R["a"], Y["a"], parts)
    return c


def _projector(d, out=4096, seed=5):
    from univa.models.modeling_univa_denoise_tower import DenoiseProjector

    g = torch.Generator(device="cuda").manual_seed(seed)
    pw = {"0.weight": torch.randn(3 * out, d, device="cuda", generator=g) * d ** -0.5,
          "0.bias": torch.randn(3 * out, device="cuda", generator=g) * 0.1,
          "2.weight": torch.randn(out, 3 * out, device="cuda", generator=g) * (3 * out) ** -0.5,
          "2.bias": torch.randn(out, device="cuda", generator=g) * 0.1}
    pw = {k: v.bfloat16() for k, v in pw.items()}
    proj = DenoiseProjector(d, out)
    proj.load_state_dict(pw)
    return pw, proj


# name: (rows as (grids, text, tail), padding side)
PREFILL = {
    "edit_prompt": ([([(1, 26, 38)], 20, 30)], None),                                    # L 301, 247 image tokens
    "padded_pair": ([([(1, 26, 38), (1, 44, 22)], 12, 14), ([], 0, 200)], "right"),       # L 528, B*L 1056
    "text_of_one": ([([], 1, 0)] * 3, None),                                               # M = 3 GEMMs
}


@pytest.mark.parametrize("case", list(PREFILL))
def test_decoder_prefill_stages_match_fp64(case):
    spec, side = PREFILL[case]
    tc, vc = _cfgs()
    sd, m = _model(tc, vc, seed=2)
    g = torch.Generator().manual_seed(7)
    rows = [_prompt(gr, t, tl, g) for gr, t, tl in spec]
    ids, mask = _batch(rows, side or "right")
    grid = [gg for gr, _, _ in spec for gg in gr]
    pix = _pixels(grid, 3) if grid else None
    B, L = ids.shape
    real = mask.bool()
    parts = {"text": real & (ids != IMG), "image": ids == IMG, "padding": ~real}
    from gpt_image_edit_b200 import ops
    from gpt_image_edit_b200.qwen2p5vl import get_rope_index, padding_spans

    pos = get_rope_index(ids, torch.tensor(grid) if grid else None, mask if side else None, image_token_id=IMG,
                         vision_start_token_id=VSTART)[0]
    spans = padding_spans(mask) if side else None
    checks = []
    last = {}

    def cb(i, x_in, x, keep):
        if side is not None:
            assert not bool(keep["attn_out"].view(B, L, -1)[~real.cuda()].any()), "padding rows' attention output"
        checks.extend(_layer_gates(sd, tc, i, x_in, x, keep, pos, parts, spans, B, L))
        last["x"] = x.clone()

    h, emb, pos_e, _, spans_e = _engine_prefill(m, ids, mask if side else None, pix, grid, layer_cb=cb)
    assert torch.equal(pos_e.cpu(), pos) and spans_e == spans
    x_fin = last["x"].view(B, L, -1)
    checks += QS.dec_gates("norm", "h", h, QS.norm_stage(sd, tc, x_fin, f64), QS.norm_stage(sd, tc, x_fin, bf16), parts)
    one = m(ids.cuda(), pixel_values=pix, attention_mask=mask.cuda() if side else None,
            image_grid_thw=torch.tensor(grid) if grid else None)
    assert torch.equal(one, h)
    # MLP2 on the hidden state, and on it with the image rows blended with the ViT output (vlm_residual_image_factor)
    pw, proj = _projector(tc.hidden_size)
    flat = h.reshape(-1, tc.hidden_size)
    for f in ((0.0, 0.3) if grid else (0.0,)):
        inp = flat.clone()
        if f:
            where = (ids.reshape(-1) == IMG).nonzero().squeeze(1).cuda()
            ops.scatter_rows_(inp, where, ops.blend(ops.gather_rows(inp, where), emb.contiguous(), 1.0 - f, f))
            R = (1 - f) * flat[where].double() + f * emb.double()
            Y = ((1 - f) * flat[where].float() + f * emb.float()).bfloat16()
            checks += QS.TB.gate(f"blend {f}", "h", inp[where], R, Y, ("rows", "cols"), beta=QS.IB.BETA)
        K = proj(inp.view(B, L, -1))
        R, Y = QS.mlp2_stage(pw, inp, f64), QS.mlp2_stage(pw, inp, bf16)
        checks += QS.dec_gates(f"mlp2 {f}", "enc", K, R.view(B, L, -1), Y.view(B, L, -1), parts)
    _summary(case, checks)
    bad = _report(f"{case} B {B} L {L}", checks)
    assert not bad, "\n".join(bad)



def test_massive_activation_layer_matches_fp64():
    """one decoder layer fed a residual stream with 4 channels at +-2000 (Qwen2's outlier channels): RMSNorm's statistics
    and the in-place residual GEMMs where a bf16 ulp of the stream is 16"""
    tc, vc = _cfgs(layers=1, depth=0, full=())
    sd, m = _model(tc, vc, seed=4)
    B, L = 1, 300
    g = torch.Generator(device="cuda").manual_seed(9)
    x = torch.randn(B * L, tc.hidden_size, device="cuda", generator=g)
    for c, s in ((17, 2000.0), (458, -2000.0), (1201, 2000.0), (3000, -2000.0)):
        x[:, c] = s * (1 + 0.01 * torch.randn(B * L, device="cuda", generator=g))
    x = x.bfloat16()
    pos = torch.arange(L).view(1, 1, L).expand(3, B, L)
    cos, sin = m._rope_tables(pos)
    x_in = x.clone()
    keep = {}
    m._decoder_layer(0, x, m._attn_buffer(B, L), cos, sin, B, L, keep=keep)
    parts = {"text": torch.ones(B, L, dtype=torch.bool)}
    checks = _layer_gates(sd, tc, 0, x_in, x, keep, pos, parts, None, B, L)
    _summary("massive_activation", checks)
    bad = _report("massive activation", checks)
    assert not bad, "\n".join(bad)


def test_decoder_prefills_reach_both_gemm_tiles():
    """which tile each Qwen linear runs on in a single-image edit prompt (L 301) and a padded pair (B*L 1056)"""
    from test_gemm_wide_gpu import _tags

    tc, vc = _cfgs(layers=1, depth=1, full=(0,))
    _, m = _model(tc, vc, seed=6)
    pw, proj = _projector(tc.hidden_size)
    seen = set()
    for case in ("edit_prompt", "padded_pair"):
        spec, side = PREFILL[case]
        g = torch.Generator().manual_seed(7)
        ids, mask = _batch([_prompt(gr, t, tl, g) for gr, t, tl in spec], side or "right")
        grid = [gg for gr, _, _ in spec for gg in gr]
        tags = _tags(lambda: proj(m(ids.cuda(), pixel_values=_pixels(grid, 3), attention_mask=mask.cuda() if side else None,
                                    image_grid_thw=torch.tensor(grid))))
        print(f"\n{case} B*L {ids.numel()}: " + ", ".join(tags))
        seen |= {t.rsplit(" ", 1)[-1] for t in tags}
    assert {"t128", "t256"} <= seen, seen


# ------------------------------------------------------------------------------------------------ decode
def test_decode_steps_match_fp64():
    """B 2, left-padded text prompts of 300 and 181 tokens, 4 teacher-forced steps: each step's layers as stages, the new
    cache rows against the reference K / V, the lm_head logits per (step, sequence) in vocab chunks, and the argmax
    wherever the float64 top-2 margin is clear."""
    from gpt_image_edit_b200 import ops

    tc, vc = _cfgs(depth=0, full=())
    sd, m = _model(tc, vc, seed=8)
    g = torch.Generator().manual_seed(11)
    ids, mask = _batch([_prompt([], 300, 0, g), _prompt([], 181, 0, g)], "left")
    B, L = ids.shape
    steps = 4
    forced = torch.randint(1000, 150000, (B, steps), generator=g)
    nkv, hd = tc.num_key_value_heads, m.thd
    cache = torch.full((tc.num_hidden_layers, 2, B, L + steps, nkv, hd), float("nan"), device="cuda", dtype=bf16)
    qkvs = []
    h, _, pos, deltas, spans = _engine_prefill(m, ids, mask, None, [], cache,
                                               layer_cb=lambda i, xi, x, keep: qkvs.append(keep["qkv"].clone()))
    nq = tc.num_attention_heads
    for i, qkv in enumerate(qkvs):            # the cache holds the post-RoPE K and V columns of the layer's qkv
        k = qkv[:, nq * hd:(nq + nkv) * hd].view(B, L, nkv, hd)
        v = qkv[:, (nq + nkv) * hd:].view(B, L, nkv, hd)
        assert torch.equal(cache[i, 0, :, :L], k) and torch.equal(cache[i, 1, :, :L], v)
    checks, logits_k, logits_r, logits_y = [], [], [], []
    last = h[:, -1]
    lo = [s[0] for s in spans]
    for t in range(steps):
        logits_k.append(m.lm_logits(last).float())
        logits_r.append(QS.lm_head_stage(sd, last, f64))
        logits_y.append(QS.lm_head_stage(sd, last, bf16))
        if t == steps - 1:
            break
        past = L + t
        nxt = forced[:, t].cuda()
        # the same step on a cache whose rows outside [lo, past) are NaN and on one where they are zero
        nan_c, zero_c = cache.clone(), cache.clone()
        for b in range(B):
            nan_c[:, :, b, :lo[b]], zero_c[:, :, b, :lo[b]] = float("nan"), 0
        nan_c[:, :, :, past:], zero_c[:, :, :, past:] = float("nan"), 0
        ref_step = m._decode_step(nxt, nan_c, past, deltas, spans)
        assert torch.equal(ref_step, m._decode_step(nxt, zero_c, past, deltas, spans)), "read outside [lo, past]"
        before = cache.clone()
        # text continues after the prompt's largest position on all three axes
        pos_t = (pos.amax(dim=(0, 2)).cpu() + 1 + t).view(1, B, 1).expand(3, B, 1)
        assert torch.equal(pos_t[0, :, 0], past + deltas.cpu().view(B))
        cos, sin = m._rope_tables(pos_t)
        x = ops.gather_rows(m.W["model.embed_tokens"], nxt.contiguous())
        o = m._attn_buffer(B, 1, past, spans)
        for i in range(tc.num_hidden_layers):
            x_in = x.clone()
            keep = {}
            m._decoder_layer(i, x, o, cos, sin, B, 1, cache, past, spans, keep)
            kv = (cache[i, 0, :, :past], cache[i, 1, :, :past])
            R = QS.decoder_stage(sd, tc, i, x_in.view(B, 1, -1), pos_t, f64, past_kv=kv, past_lo=lo)
            Y = QS.decoder_stage(sd, tc, i, x_in.view(B, 1, -1), pos_t, bf16, past_kv=kv, past_lo=lo)
            st = f"step {t} dec {i}"
            lab = lambda kind, j: f"sequence {j}" if kind == "rows" else f"{kind[:-1]} {j}"
            checks += QS.TB.gate(st, "h", x, R["h"][:, 0], Y["h"][:, 0], ("rows", "cols"), lab, beta=QS.IB.BETA)
            checks += QS.TB.gate(st, "attn", keep["attn_out"], R["attn"][:, 0], Y["attn"][:, 0], ("rows", "cols"), lab,
                                 beta=QS.IB.BETA)
            checks += QS.TB.gate(st, "cache k", cache[i, 0, :, past].reshape(B, -1), R["k"].reshape(B, -1),
                                 Y["k"].reshape(B, -1), ("rows",), lab, beta=QS.IB.BETA)
            checks += QS.TB.gate(st, "cache v", cache[i, 1, :, past].reshape(B, -1), R["v"].reshape(B, -1),
                                 Y["v"].reshape(B, -1), ("rows",), lab, beta=QS.IB.BETA)
        changed = (cache != before) & ~(torch.isnan(cache) & torch.isnan(before))
        assert not bool(changed[:, :, :, :past].any()) and not bool(changed[:, :, :, past + 1:].any()), "wrote outside row past"
        last = ops.rmsnorm(x, m.W["model.norm"], eps=tc.rms_norm_eps)
        assert torch.equal(last, ref_step)
    K, R, Y = torch.cat(logits_k), torch.cat(logits_r), torch.cat(logits_y)
    lab = lambda kind, j: f"step {j // B} sequence {j % B}" if kind == "rows" else f"vocab {j}"
    checks += QS.logits_gates("lm_head", K, R, Y, lab)
    top2 = R.topk(2, dim=-1)
    clear = (top2.values[:, 0] - top2.values[:, 1]) > 8 * (K.double() - R).abs().max(-1).values
    assert torch.equal(K.argmax(-1)[clear], top2.indices[clear, 0])
    print(f"\nargmax checked on {int(clear.sum())} of {clear.numel()} (step, sequence) rows")
    # the stagewise run is generate() with the same forced tokens
    _, scores = m.generate(ids.cuda(), attention_mask=mask.cuda(), forced_tokens=forced, output_scores=True,
                           eos_token_id=(999999,))
    for t in range(steps):
        assert torch.equal(scores[t], logits_k[t]), f"step {t}"
    _summary("decode", checks)
    bad = _report(f"decode B {B} L {L} steps {steps}", checks)
    assert not bad, "\n".join(bad)
