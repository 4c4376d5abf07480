"""CPU checks of the stage references and gates in train_block_ref.py (no GPU needed).

- double_block_mod / single_block_mod fed the modulation rows double_block / single_block compute give the same bits;
  apply_rotary_emb keeps float64 inputs in float64.
- Each float64 stage reference agrees with central finite differences of the oracle along random directions, for
  every gradient family the engine produces: block input, fused q|k|v weight and bias (perturbing to_q / to_k / to_v),
  to_out, norm_q / norm_k, the AdaLN linears through dmod (perturbing norm1.linear / norm.linear / norm_out.linear
  themselves, so the chunk order is checked), d_enc and MLP2.
- At the proportions of the training workload (S_txt 288, S_img 2048, n_out 1024; d = 256 to keep it small) the
  per-slice gate fails on three errors: one target token's gradient dropped, one image token modulated with the text
  stream's chunks, one 128-row head block of the q|k|v weight gradient scaled by 0.9.  What the per-tensor rule makes
  of each is printed and asserted as measured.
"""
import pytest
import torch
import torch.nn.functional as F

import train_block_ref as TB
from oracle import flux_oracle as fo


def _ids(h, w):
    ids = torch.zeros(h, w, 3)
    ids[..., 1] += torch.arange(h)[:, None]
    ids[..., 2] += torch.arange(w)[None, :]
    ids = ids.reshape(-1, 3)
    ctx = ids.clone()
    ctx[:, 0] = 1
    return torch.cat([ids, ctx])


def _full_mod(sd, cfg, temb):
    """`mod` as b2f_flux_modulation lays it out: every AdaLN linear of silu(temb), in block order."""
    st = F.silu(temb)
    rows = []
    for i in range(cfg.num_layers):
        rows += [fo._lin(sd, f"transformer_blocks.{i}.norm1.linear", st), fo._lin(sd, f"transformer_blocks.{i}.norm1_context.linear", st)]
    rows += [fo._lin(sd, f"single_transformer_blocks.{i}.norm.linear", st) for i in range(cfg.num_single_layers)]
    return torch.cat(rows + [fo._lin(sd, "norm_out.linear", st)], 1)


def _problem(dtype, B=2, S_txt=3, hl=2, wl=2, seed=0, **kw):
    cfg = fo.FluxConfig.toy(**kw)
    sd = fo.make_synthetic_state_dict(cfg, seed=seed, dtype=dtype, bias_std=0.2, norm_jitter=0.2)
    g = torch.Generator().manual_seed(seed + 1)
    S_img = 2 * hl * wl
    S = S_txt + S_img
    d = cfg.inner_dim
    cos, sin = fo.rope_tables(torch.cat([torch.zeros(S_txt, 3), _ids(hl, wl)]), cfg.axes_dims_rope, cfg.theta)
    temb = torch.randn(B, d, generator=g, dtype=torch.float64).to(dtype)
    return dict(cfg=cfg, sd=sd, B=B, S_txt=S_txt, S_img=S_img, S=S, d=d, cos=cos, sin=sin, temb=temb,
                h=torch.randn(B, S, d, generator=g, dtype=torch.float64).to(dtype),
                dh=torch.randn(B, S, d, generator=g, dtype=torch.float64).to(dtype), g=g)


def test_mod_wrappers_match_the_blocks_bit_for_bit():
    P = _problem(torch.float32)
    cfg, sd, S_txt, temb = P["cfg"], P["sd"], P["S_txt"], P["temb"]
    x, c = P["h"][:, S_txt:], P["h"][:, :S_txt]
    for i in range(cfg.num_layers):
        e = fo._lin(sd, f"transformer_blocks.{i}.norm1.linear", F.silu(temb))
        ec = fo._lin(sd, f"transformer_blocks.{i}.norm1_context.linear", F.silu(temb))
        a = fo.double_block(sd, i, cfg, x, c, temb, P["cos"], P["sin"])
        b = fo.double_block_mod(sd, i, cfg, x, c, e, ec, P["cos"], P["sin"])
        assert all(torch.equal(u, v) for u, v in zip(a, b))
    for i in range(cfg.num_single_layers):
        e = fo._lin(sd, f"single_transformer_blocks.{i}.norm.linear", F.silu(temb))
        assert torch.equal(fo.single_block(sd, i, cfg, P["h"], temb, P["cos"], P["sin"]),
                           fo.single_block_mod(sd, i, cfg, P["h"], e, P["cos"], P["sin"]))


def test_apply_rotary_emb_keeps_float64():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(1, 2, 5, 128, generator=g, dtype=torch.float64)
    cos, sin = fo.rope_tables(_ids(1, 5)[:5], (16, 56, 56))
    y = fo.apply_rotary_emb(x, cos, sin)
    xr, xi = x[..., 0::2], x[..., 1::2]
    c, s = cos[None, None, :, 0::2].double(), sin[None, None, :, 0::2].double()
    assert y.dtype == torch.float64
    torch.testing.assert_close(y[..., 0::2], xr * c - xi * s, rtol=0, atol=1e-15)
    torch.testing.assert_close(y[..., 1::2], xi * c + xr * s, rtol=0, atol=1e-15)
    # 16-bit inputs still compute in fp32 and round once
    xb = x.bfloat16()
    xrot = torch.stack([-xb[..., 1::2], xb[..., 0::2]], -1).flatten(3)
    assert torch.equal(fo.apply_rotary_emb(xb, cos, sin), (xb.float() * cos + xrot.float() * sin).bfloat16())


def _fd_check(loss, params, grads, g, n_dir=2, eps=1e-6):
    """<grad, v> against (L(p + eps v) - L(p - eps v)) / (2 eps) for `n_dir` random directions of every family.
    params: {family: [tensors perturbed together]}; grads: {family: gradient of the concatenated tensors}."""
    for fam, ts in params.items():
        for _ in range(n_dir):
            vs = [torch.randn(t.shape, generator=g, dtype=torch.float64) for t in ts]
            v = torch.cat([u.reshape(-1) for u in vs])
            an = (grads[fam].reshape(-1) * v).sum().item()
            with torch.no_grad():
                for t, u in zip(ts, vs):
                    t += eps * u
                lp = loss()
                for t, u in zip(ts, vs):
                    t -= 2 * eps * u
                lm = loss()
                for t, u in zip(ts, vs):
                    t += eps * u
            fd = (lp - lm) / (2 * eps)
            scale = grads[fam].norm().item() * v.norm().item()
            assert abs(fd - an) <= 1e-7 * scale + 1e-7 * abs(an), f"{fam}: fd {fd:.10e} autograd-ref {an:.10e}"


def _qkv(prefix):
    return [prefix + f"attn.{n}.weight" for n in ("to_q", "to_k", "to_v")], [prefix + f"attn.{n}.bias" for n in ("to_q", "to_k", "to_v")]


@pytest.mark.parametrize("blk", [0, 1])
def test_double_stage_reference_matches_finite_differences(blk):
    P = _problem(torch.float64)
    cfg, sd, S_txt, temb, h, dh = P["cfg"], P["sd"], P["S_txt"], P["temb"], P["h"], P["dh"]
    mod = _full_mod(sd, cfg, temb)
    r = TB.double_stage(sd, cfg, blk, h, dh, mod, F.silu(temb), P["cos"], P["sin"], S_txt, torch.float64)
    p = f"transformer_blocks.{blk}."

    def loss():
        c, x = fo.double_block(sd, blk, cfg, h[:, S_txt:], h[:, :S_txt], temb, P["cos"], P["sin"])
        return (torch.cat([c, x], 1) * dh).sum().item()

    qw, qb = _qkv(p)
    fams = {"dh": [h], "qkv.weight": [sd[k] for k in qw], "qkv.bias": [sd[k] for k in qb]}
    grads = {"dh": r["dh"], "qkv.weight": torch.cat([r[k] for k in qw]), "qkv.bias": torch.cat([r[k] for k in qb])}
    for k in ("attn.to_out.0.weight", "attn.to_out.0.bias", "attn.norm_q.weight", "attn.norm_k.weight",
              "norm1.linear.weight", "norm1.linear.bias"):
        fams[k], grads[k] = [sd[p + k]], r[p + k]
    _fd_check(loss, fams, grads, P["g"])


@pytest.mark.parametrize("si", [0, 1])
def test_single_stage_reference_matches_finite_differences(si):
    P = _problem(torch.float64)
    cfg, sd, temb, h, dh = P["cfg"], P["sd"], P["temb"], P["h"], P["dh"]
    mod = _full_mod(sd, cfg, temb)
    r = TB.single_stage(sd, cfg, si, h, dh, mod, F.silu(temb), P["cos"], P["sin"], torch.float64)
    p = f"single_transformer_blocks.{si}."

    def loss():
        return (fo.single_block(sd, si, cfg, h, temb, P["cos"], P["sin"]) * dh).sum().item()

    qw, qb = _qkv(p)
    fams = {"dh": [h], "qkv.weight": [sd[k] for k in qw], "qkv.bias": [sd[k] for k in qb]}
    grads = {"dh": r["dh"], "qkv.weight": torch.cat([r[k] for k in qw]), "qkv.bias": torch.cat([r[k] for k in qb])}
    for k in ("attn.norm_q.weight", "attn.norm_k.weight", "norm.linear.weight", "norm.linear.bias"):
        fams[k], grads[k] = [sd[p + k]], r[p + k]
    _fd_check(loss, fams, grads, P["g"])


def test_tail_head_and_mlp2_references_match_finite_differences():
    P = _problem(torch.float64)
    cfg, sd, S_txt, temb, h = P["cfg"], P["sd"], P["S_txt"], P["temb"], P["h"]
    B, n_out, g = P["B"], 5, P["g"]
    dout = torch.randn(B, n_out, cfg.out_channels, generator=g, dtype=torch.float64)
    r = TB.tail_stage(sd, cfg, h, dout, _full_mod(sd, cfg, temb), S_txt, n_out, torch.float64)

    def tail_loss():     # flux_forward's last lines on the image rows of the target tokens
        x = h[:, S_txt:S_txt + n_out]
        e = fo._lin(sd, "norm_out.linear", F.silu(temb))
        scale, shift = torch.chunk(e, 2, dim=1)
        return (fo._lin(sd, "proj_out", fo.layer_norm(x) * (1 + scale)[:, None, :] + shift[:, None, :]) * dout).sum().item()

    w, b = TB.adaln_grads(r["dmod"], F.silu(temb))
    _fd_check(tail_loss, {"dh": [h], "norm_out.weight": [sd["norm_out.linear.weight"]], "norm_out.bias": [sd["norm_out.linear.bias"]]},
              {"dh": r["dh"], "norm_out.weight": w, "norm_out.bias": b}, g)
    assert not r["dh"][:, :S_txt].any() and not r["dh"][:, S_txt + n_out:].any()

    # head: d_enc = dh_txt . W_ctx is the gradient of context_embedder(enc)
    enc = torch.randn(B, S_txt, cfg.joint_attention_dim, generator=g, dtype=torch.float64)
    dh = P["dh"]
    _fd_check(lambda: (fo._lin(sd, "context_embedder", enc) * dh[:, :S_txt]).sum().item(), {"d_enc": [enc]},
              {"d_enc": TB.head_stage(sd, dh, S_txt, torch.float64)}, g)

    # MLP2
    pw = {"0.weight": torch.randn(24, 16, generator=g, dtype=torch.float64) * 0.3, "0.bias": torch.randn(24, generator=g, dtype=torch.float64),
          "2.weight": torch.randn(8, 24, generator=g, dtype=torch.float64) * 0.3, "2.bias": torch.randn(8, generator=g, dtype=torch.float64)}
    x = torch.randn(B, S_txt, 16, generator=g, dtype=torch.float64)
    dv = torch.randn(B, S_txt, 8, generator=g, dtype=torch.float64)
    rm = TB.mlp2_stage(pw, x, dv, torch.float64)
    mlp = lambda: (F.linear(F.silu(F.linear(x, pw["0.weight"], pw["0.bias"])), pw["2.weight"], pw["2.bias"]) * dv).sum().item()
    _fd_check(mlp, {k: [v] for k, v in pw.items()}, rm, g)


# ------------------------------------------------------------------------------------------------ gate power
def _double_checks(stage_out, R, Y, P, blk):
    """every gate of a double-block stage, as the GPU test applies them."""
    d, S_txt = P["d"], P["S_txt"]
    p = f"transformer_blocks.{blk}."
    qw, qb = _qkv(p)
    cat = lambda r, ks: torch.cat([r[k] for k in ks])
    out = TB.dh_gates("double", stage_out["dh"], R["dh"], Y["dh"], P["dh"], P["B"], S_txt)
    out += TB.gate("double", "qkv.weight", cat(stage_out, qw), cat(R, qw), cat(Y, qw), ("rows", "cols"), TB.qkv_label(d, 128))
    out += TB.gate("double", "qkv.bias", cat(stage_out, qb), cat(R, qb), cat(Y, qb), ("elems",))
    for k, kinds in (("attn.to_out.0.weight", ("rows", "cols")), ("attn.to_out.0.bias", ("elems",)),
                     ("attn.norm_q.weight", ("elems",)), ("attn.norm_k.weight", ("elems",)), ("norm1.linear.bias", ("elems",))):
        out += TB.gate("double", k, stage_out[p + k], R[p + k], Y[p + k], kinds)
    out += TB.gate("double", "norm1.linear.weight", stage_out[p + "norm1.linear.weight"], R[p + "norm1.linear.weight"],
                   Y[p + "norm1.linear.weight"], ("chunks",), TB.chunk_label(TB.CHUNKS["double"]), n_chunks=6)
    return out


@pytest.fixture(scope="module")
def bench_proportions():
    """A double block at the train512 lengths (B 1, S_txt 288, S_img 2048, n_out 1024), d = 256: the float64 reference
    and the CPU torch-bf16 yardstick on the same bf16 inputs."""
    P = _problem(torch.bfloat16, B=1, S_txt=288, hl=32, wl=32, seed=4)
    P["n_out"] = 1024
    g = torch.Generator().manual_seed(5)
    for k, v in P["sd"].items():      # O(1) shifts, scales and gates, as trained FLUX has: the block's share of dh counts
        if "norm1" in k and k.endswith(".bias"):
            P["sd"][k] = torch.randn(v.shape, generator=g).bfloat16()
    P["dh"][:, P["S_txt"] + P["n_out"]:] = 0           # the tail leaves the context rows' gradient at zero
    P["mod"] = _full_mod(P["sd"], P["cfg"], P["temb"])
    P["stemb"] = F.silu(P["temb"])
    f = lambda dt, dh=None: TB.double_stage(P["sd"], P["cfg"], 1, P["h"], P["dh"] if dh is None else dh, P["mod"], P["stemb"],
                                            P["cos"], P["sin"], P["S_txt"], dt)
    P["stage"] = f
    P["R"], P["Y"] = f(torch.float64), f(torch.bfloat16)
    return P


def _verdicts(checks):
    tensor = {c.tensor: c.ok for c in checks if c.kind == "tensor"}
    slices = [c for c in checks if c.kind != "tensor" and not c.ok]
    return tensor, slices


def test_gates_pass_the_yardstick_itself(bench_proportions):
    """the bf16 yardstick passes its own gates (e = y): the gates leave room for an engine as good as torch-bf16."""
    P = bench_proportions
    checks = _double_checks(P["Y"], P["R"], P["Y"], P, 1)
    assert all(c.ok for c in checks), [str(c) for c in checks if not c.ok]


def _report(name, checks):
    tensor, slices = _verdicts(checks)
    print(f"\n{name}: per-tensor rule fails on {sorted(k for k, ok in tensor.items() if not ok) or 'nothing'}")
    print("\n".join(str(c) for c in checks))
    assert slices, f"{name}: the per-slice gate passed"
    return tensor, slices


def test_slice_gate_catches_a_dropped_target_token(bench_proportions):
    P = bench_proportions
    dh = P["dh"].clone()
    dh[:, P["S_txt"] + 517] = 0                        # target token 517 gets no gradient
    K = P["stage"](torch.float64, dh)
    tensor, slices = _report("dropped target token", _double_checks(K, P["R"], P["Y"], P, 1))
    assert any(c.tensor == "dh image" and c.where == "batch 0 image token 517" for c in slices)
    # measured: the per-tensor rule catches this one too at stage level (rel-L2 ~3e-2 against a bf16 yardstick of ~4e-3
    # per stage), on dh image and on every weight gradient but norm_q / norm_k
    assert not tensor["dh image"] and not tensor["qkv.weight"], tensor


def test_slice_gate_catches_one_token_with_the_text_modulation(bench_proportions, monkeypatch):
    P = bench_proportions
    d, S_txt, tok = P["d"], P["S_txt"], 1234
    e = P["mod"][:, 12 * d:18 * d].double()
    ec = P["mod"][:, 18 * d:24 * d].double()
    calls = []
    ln = fo.layer_norm

    def swapped(x, eps=1e-6):
        # the image stream's first LayerNorm: give token `tok` the text stream's (shift, scale) after modulation
        y = ln(x, eps)
        calls.append(1)
        if len(calls) == 1:
            y = y.clone()
            sh, sc, csh, csc = e[:, None, :d], e[:, None, d:2 * d], ec[:, None, :d], ec[:, None, d:2 * d]
            y[:, tok] = ((y[:, tok:tok + 1] * (1 + csc) + csh - sh) / (1 + sc))[:, 0]
        return y

    monkeypatch.setattr(fo, "layer_norm", swapped)
    K = P["stage"](torch.float64)
    monkeypatch.setattr(fo, "layer_norm", ln)
    assert len(calls) == 4
    checks = _double_checks(K, P["R"], P["Y"], P, 1)
    tensor, slices = _report("image token with text modulation", checks)
    # measured: the per-tensor rule passes everything; the slice gate fails on single elements of the AdaLN bias
    # gradient in the token's shift / scale chunks, and the worst dh row is that token's (2x the yardstick, inside beta)
    assert all(tensor.values()), tensor
    assert any(c.tensor == "norm1.linear.bias" and 0 <= int(c.where.split()[-1]) < 2 * d for c in slices)
    assert all(c.where == f"batch 0 image token {tok}" for c in checks if c.tensor.startswith("dh") and "image" in c.tensor
               and c.kind == "rows")


def test_slice_gate_catches_one_scaled_head_block(bench_proportions):
    P = bench_proportions
    K = dict(P["R"])
    key = "transformer_blocks.1.attn.to_k.weight"
    K[key] = K[key].clone()
    K[key][128:256] *= 0.9                              # k, head 1: rows 384..511 of the fused q|k|v gradient
    tensor, slices = _report("scaled head block", _double_checks(K, P["R"], P["Y"], P, 1))
    assert all(tensor.values()), tensor                  # measured: the per-tensor rule passes it
    assert any(c.tensor == "qkv.weight" and c.kind == "rows" and "k head 1" in c.where for c in slices)
