"""FP8 block linears and attention on the 1024^2 edit (S_txt 544 + S_img 8192 = 8736 tokens, d 3072, 19 + 38 blocks,
B = 1), H100.

  step    per-step ms of one transformer forward with the AdaLN modulation hoisted (as the sampling loop runs it), in four
          configurations alternating within every round: bf16, fp8 (enable_fp8: linears), fp8+attn (linears and
          attention) and attn (enable_fp8(linears=False, attention=True)), reported as the range over --rounds rounds,
          with the denoise-only images/s that implies (28 steps) and torch.cuda.max_memory_allocated of each
  attn    TFLOP/s (4 S^2 d per call) of bf16 b2f_attention_fwd and FP8 b2f_attention_fp8 at the loop shape (B 1, H 24,
          S 8736), alternating, and the ms of the b2f_attn_quant_fp8 pass that feeds the FP8 kernel; each timed window
          is ATTN_ITERS back-to-back calls (about a quarter of a second), so one round's ratio is not a 30 ms sample
  gemm    TFLOP/s of the bf16 GEMM (b2f_gemm_bf16) and the FP8 GEMM (b2f_gemm_fp8) on each loop shape, alternating
  quant   ms of the launches FP8 adds or replaces per forward: b2f_ln_modulate_fp8 against b2f_ln_modulate, and the
          b2f_quant_fp8_rows launches over cat's [0, d), [d, 5d) and [0, 5d) columns, times their count per forward
The card's name and power limit are read in the same process.

  python scripts/bench_fp8.py [--rounds 3] [--iters 5] [--what step,attn,gemm,quant] [--out-dir bench_out]
"""
import argparse
import json
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from bench_lora import card, timed  # noqa: E402

S_TXT, N_IMG, D = 544, 4096, 3072
ATTN_ITERS = 200
S = S_TXT + 2 * N_IMG


def _rng(v):
    return [min(v), max(v)]


def step_bench(args):
    from gpt_image_edit_b200.flux_transformer import B200FluxTransformer2DModel, FluxTransformerConfig
    m = B200FluxTransformer2DModel(FluxTransformerConfig()).randomize_(seed=0)
    g = torch.Generator(device="cuda").manual_seed(1)
    side = 64
    ids = torch.stack([torch.zeros(N_IMG), torch.arange(N_IMG) // side, torch.arange(N_IMG) % side], 1)
    ctx = ids.clone()
    ctx[:, 0] = 1
    inp = dict(hidden_states=torch.randn(1, 2 * N_IMG, 64, device="cuda", generator=g).bfloat16(),
               encoder_hidden_states=torch.randn(1, S_TXT, 4096, device="cuda", generator=g).bfloat16(),
               pooled_projections=torch.randn(1, 768, device="cuda", generator=g).bfloat16(),
               timestep=torch.full((1,), 0.5, device="cuda").bfloat16(),
               img_ids=torch.cat([ids, ctx]).cuda().bfloat16(), txt_ids=torch.zeros(S_TXT, 3, device="cuda").bfloat16(),
               guidance=torch.full((1,), 3.5, device="cuda"))
    m.prepare_schedule(inp["timestep"], inp["guidance"], inp["pooled_projections"])
    jak = {"_b2f_schedule_step": 0, "_b2f_out_rows": N_IMG}
    f = lambda: m(**inp, joint_attention_kwargs=jak, return_dict=False)
    confs = {"bf16": None, "fp8": dict(), "fp8+attn": dict(attention=True), "attn": dict(linears=False, attention=True)}
    per = {c: [] for c in confs}
    peak = {c: 0 for c in confs}
    outs = {}
    for rnd in range(args.rounds):
        for conf, kw in confs.items():
            if kw is not None:
                m.enable_fp8(**kw)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            for _ in range(args.warmup):
                outs[conf] = f()[0]
            per[conf].append(timed(f, args.iters))
            peak[conf] = max(peak[conf], torch.cuda.max_memory_allocated())
            m.disable_fp8()
        print(f"round {rnd}: " + ", ".join(f"{c} {per[c][-1]:.1f} ms" for c in per), flush=True)
    b = outs["bf16"].double()
    res = {c: {"step_ms": _rng(v), "denoise_img_per_s": [1000 / (28 * max(v)), 1000 / (28 * min(v))],
               "max_memory_allocated_GB": peak[c] / 1e9} for c, v in per.items()}
    for c in ("fp8", "fp8+attn", "attn"):
        a = outs[c].double()
        res[f"{c}_vs_bf16_time"] = _rng([x / y for x, y in zip(per[c], per["bf16"])])
        res[f"{c}_vs_bf16_output_rel_l2"] = ((a - b).norm() / b.norm()).item()
    del m, outs
    torch.cuda.empty_cache()
    return res


def gemm_bench(args):
    from gpt_image_edit_b200 import ops
    shapes = [("qkv img", 8192, 3 * D, D), ("single qkv+mlp", S, 7 * D, D), ("to_out", 8192, D, D),
              ("ff1", 8192, 4 * D, D), ("ff2", 8192, D, 4 * D), ("single proj_out", S, D, 5 * D)]
    g = torch.Generator(device="cuda").manual_seed(3)
    out = {}
    for name, M, N, K in shapes:
        x = torch.randn(M, K, device="cuda", generator=g).bfloat16()
        w = (torch.randn(N, K, device="cuda", generator=g) * K ** -0.5).bfloat16()
        b = torch.zeros(N, device="cuda", dtype=torch.bfloat16)
        y = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        xq, xs = ops.quant_fp8_rows(x)
        wq, ws = ops.quant_fp8_rows(w)
        bf, f8 = [], []
        for _ in range(args.rounds):
            bf.append(timed(lambda: ops.linear(x, w, b, out=y), 20))
            f8.append(timed(lambda: ops.linear_fp8(xq, xs, wq, ws, b, out=y), 20))
        fl = 2.0 * M * N * K
        row = {"bf16_tflops": [fl / max(bf) / 1e9, fl / min(bf) / 1e9],
               "fp8_tflops": [fl / max(f8) / 1e9, fl / min(f8) / 1e9],
               "fp8_time_vs_bf16": _rng([a / c for a, c in zip(f8, bf)])}
        out[f"{name} {M}x{N}x{K}"] = row
        print(name, json.dumps(row), flush=True)
        del x, w, xq, wq, y
    return out


def attn_bench(args):
    from gpt_image_edit_b200 import ops
    H = D // 128
    g = torch.Generator(device="cuda").manual_seed(5)
    # the model's layout: q, k, v as column slices of one qkv [1, S, 3d] buffer, out into cat [1, S, 5d]; q / k with
    # the spread RMSNorm + RoPE leave them (unit rms per head)
    qkv = torch.randn(1, S, 3 * D, device="cuda", generator=g).bfloat16()
    q, k, v = (qkv[:, :, i * D:(i + 1) * D].unflatten(-1, (H, 128)) for i in range(3))
    cat = torch.empty(1, S, 5 * D, device="cuda", dtype=torch.bfloat16)
    bufs = ops.attn_quant_fp8(q, k, v)
    runs = {"bf16": lambda: ops.attention(q, k, v, out=cat[:, :, :D]),
            "fp8": lambda: ops.attention_fp8(*bufs, out=cat[:, :, :D]),
            "quant": lambda: ops.attn_quant_fp8(q, k, v, q8=bufs[0], k8=bufs[1], sq=bufs[2], sk=bufs[3], v8t=bufs[4],
                                                sv=bufs[5])}
    t = {k_: [] for k_ in runs}
    for _ in range(args.rounds):
        for k_, fn in runs.items():
            fn()
            t[k_].append(timed(fn, ATTN_ITERS))
    fl = 4.0 * S * S * D
    res = {"shape": f"B1 H{H} S{S}", "bf16_tflops": [fl / max(t["bf16"]) / 1e9, fl / min(t["bf16"]) / 1e9],
           "fp8_tflops": [fl / max(t["fp8"]) / 1e9, fl / min(t["fp8"]) / 1e9],
           "bf16_ms": _rng(t["bf16"]), "fp8_ms": _rng(t["fp8"]), "quant_ms": _rng(t["quant"]),
           "fp8_speedup": _rng([a / c for a, c in zip(t["bf16"], t["fp8"])]),
           "fp8_plus_quant_speedup": _rng([a / (c + e) for a, c, e in zip(t["bf16"], t["fp8"], t["quant"])])}
    print("attn", json.dumps(res), flush=True)
    return res


def quant_bench(args):
    from gpt_image_edit_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(4)
    h = torch.randn(1, S, D, device="cuda", generator=g).bfloat16()
    mod = (torch.randn(1, 4 * D, device="cuda", generator=g) * 0.3).bfloat16()
    cat = torch.randn(1, S, 5 * D, device="cuda", generator=g).bfloat16()
    q8 = torch.empty(1, S, 5 * D, device="cuda", dtype=ops.FP8)
    qs = torch.empty(1, S, device="cuda")
    xn = torch.empty_like(h)
    sc, sh, sc_b, sh_b = mod[:, :D], mod[:, D:2 * D], mod[:, 2 * D:3 * D], mod[:, 3 * D:]
    runs = {
        "ln_modulate (bf16)": lambda: ops.ln_modulate(h, sc, sh, out=xn, split_row=S_TXT, scale_b=sc_b, shift_b=sh_b),
        "ln_modulate_fp8": lambda: ops.ln_modulate_fp8(h, sc, sh, out=q8[:, :, :D], row_scale=qs, split_row=S_TXT,
                                                       scale_b=sc_b, shift_b=sh_b),
        "quant cat[0:d]": lambda: ops.quant_fp8_rows(cat[:, :, :D], out=q8[:, :, :D], scale=qs),
        "quant cat[d:5d]": lambda: ops.quant_fp8_rows(cat[:, :, D:], out=q8[:, :, :4 * D], scale=qs),
        "quant cat[0:5d]": lambda: ops.quant_fp8_rows(cat, out=q8, scale=qs),
    }
    t = {k: [] for k in runs}
    for _ in range(args.rounds):
        for k, fn in runs.items():
            fn()
            t[k].append(timed(fn, 20))
    res = {k: {"ms": _rng(v)} for k, v in t.items()}
    # per forward: 2 LayerNorms + quant [0, d) + quant [d, 5d) per double block, 1 LayerNorm + quant [0, 5d) per single
    nd, ns = 19, 38
    added = [nd * (2 * (a - b) + c + d4) + ns * ((a - b) + e) for a, b, c, d4, e in
             zip(t["ln_modulate_fp8"], t["ln_modulate (bf16)"], t["quant cat[0:d]"], t["quant cat[d:5d]"],
                 t["quant cat[0:5d]"])]
    res["added_ms_per_forward"] = _rng(added)
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--what", default="step,attn,gemm,quant")
    ap.add_argument("--out-dir", default="bench_out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8.py measures on the GPU; no CUDA device is visible")
    res = {"card_before": card(), "time": time.strftime("%Y-%m-%d %H:%M:%S")}
    if "step" in args.what:
        res["step"] = step_bench(args)
    if "attn" in args.what:
        res["attn"] = attn_bench(args)
    if "gemm" in args.what:
        res["gemm"] = gemm_bench(args)
    if "quant" in args.what:
        res["quant"] = quant_bench(args)
    res["card_after"] = card()
    Path(args.out_dir).mkdir(parents=True, exist_ok=True)
    (Path(args.out_dir) / "bench_fp8.json").write_text(json.dumps(res, indent=1))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
