"""Batches of distinct edit instructions on the FLUX denoiser (19 + 38 blocks, d 3072): is one B = 4 call with per-item
text windows faster than four B = 1 calls?

  step    Four instructions whose Qwen2.5-VL parts are 288, 301, 330 and 395 tokens long, each followed by 256 T5 tokens
          (text lengths 544, 557, 586 and 651), at 512^2, 768^2 and 1024^2 (S_img = 2 * (side / 16)^2: target and
          context image).  "batched" is one transformer forward over the four, left-padded to 651 by
          stack_prompt_embeds with encoder_attention_mask; "separate" is four forwards of B = 1, each on its own
          unpadded text.  Both run with the AdaLN modulation hoisted as the sampling loop runs it (a schedule per
          call: the batched call's B = 4 one, one per instruction for the separate calls), so a number is the time of
          one denoising step of all four requests.  bf16, and FP8 linears + FP8 attention (enable_fp8(attention=True)).
          The two orders alternate within every round; reported as the range over --rounds rounds.
  kernel  The attention kernels at the loop shape (B 1, H 24, S_txt 544, S 8736) with the full window (0, 544) against
          the unwindowed ones, alternating: b2f_attention_fwd_window vs b2f_attention_fwd and b2f_attention_fp8_window
          vs b2f_attention_fp8; each timed window is KERNEL_ITERS back-to-back calls.
The card's name and power limit are read in the same process.

  python scripts/bench_ragged.py [--rounds 3] [--iters 2] [--what step,kernel] [--out-dir bench_out]
"""
import argparse
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from bench_lora import card, timed  # noqa: E402

QWEN_LENS = (288, 301, 330, 395)
T5_LEN = 256
SIDES = (512, 768, 1024)
KERNEL_ITERS = 200


def _rng(v):
    return [min(v), max(v)]


def _ids(side):
    n = side // 16
    ids = torch.stack([torch.zeros(n * n), torch.arange(n * n) // n, torch.arange(n * n) % n], 1)
    ctx = ids.clone()
    ctx[:, 0] = 1
    return torch.cat([ids, ctx]).cuda().bfloat16()


def step_bench(args):
    from gpt_image_edit_b200.flux_transformer import B200FluxTransformer2DModel, FluxTransformerConfig
    from gpt_image_edit_b200.pipeline import stack_prompt_embeds

    m = B200FluxTransformer2DModel(FluxTransformerConfig()).randomize_(seed=0)
    g = torch.Generator(device="cuda").manual_seed(1)
    B = len(QWEN_LENS)
    encs = [torch.randn(1, q + T5_LEN, 4096, device="cuda", generator=g).bfloat16() for q in QWEN_LENS]
    enc, mask = stack_prompt_embeds(encs)
    pooled = torch.randn(B, 768, device="cuda", generator=g).bfloat16()
    t = torch.full((1,), 0.5, device="cuda").bfloat16()
    gd = torch.full((B,), 3.5, device="cuda")
    res = {}
    for conf in ("bf16", "fp8+attn"):
        if conf != "bf16":
            m.enable_fp8(linears=True, attention=True)
        sched_b = m.prepare_schedule(t, gd, pooled)
        sched_1 = [m.prepare_schedule(t, gd[b:b + 1], pooled[b:b + 1]) for b in range(B)]
        for side in SIDES:
            n_img = (side // 16) ** 2
            img_ids = _ids(side)
            hs = torch.randn(B, 2 * n_img, 64, device="cuda", generator=g).bfloat16()
            jak = {"_b2f_schedule_step": 0, "_b2f_out_rows": n_img}

            def batched():
                m._schedule = sched_b
                return m(hidden_states=hs, encoder_hidden_states=enc, pooled_projections=pooled, timestep=t.expand(B),
                         img_ids=img_ids, txt_ids=torch.zeros(enc.shape[1], 3, device="cuda").bfloat16(), guidance=gd,
                         encoder_attention_mask=mask, joint_attention_kwargs=jak, return_dict=False)[0]

            txt_ids = [torch.zeros(e.shape[1], 3, device="cuda").bfloat16() for e in encs]

            def separate():
                outs = []
                for b in range(B):
                    m._schedule = sched_1[b]
                    outs.append(m(hidden_states=hs[b:b + 1], encoder_hidden_states=encs[b],
                                  pooled_projections=pooled[b:b + 1], timestep=t, img_ids=img_ids, txt_ids=txt_ids[b],
                                  guidance=gd[b:b + 1], joint_attention_kwargs=jak, return_dict=False)[0])
                return outs

            runs = {"batched": batched, "separate": separate}
            per = {k: [] for k in runs}
            for fn in runs.values():     # warm-up: every shape of the timed window
                fn()
            for rnd in range(args.rounds):
                order = list(runs) if rnd % 2 == 0 else list(reversed(runs))
                for k in order:
                    per[k].append(timed(runs[k], args.iters))
            a, s = batched(), separate()
            diff = max(((a[b].double() - s[b][0].double()).norm() / s[b][0].double().norm()).item() for b in range(B))
            row = {"S_img": 2 * n_img, "batched_step_ms": _rng(per["batched"]),
                   "separate_step_ms": _rng(per["separate"]),
                   "batched_speedup": _rng([x / y for x, y in zip(per["separate"], per["batched"])]),
                   "max_item_rel_l2_batched_vs_separate": diff}
            res[f"{conf} {side}^2"] = row
            print(conf, side, json.dumps(row), flush=True)
            del hs
        m._schedule = None
        m.disable_fp8()
    del m
    torch.cuda.empty_cache()
    return res


def kernel_bench(args):
    from gpt_image_edit_b200 import ops

    D, S_txt, S = 3072, 544, 544 + 8192
    H = D // 128
    g = torch.Generator(device="cuda").manual_seed(5)
    qkv = torch.randn(1, S, 3 * D, device="cuda", generator=g).bfloat16()
    q, k, v = (qkv[:, :, i * D:(i + 1) * D].unflatten(-1, (H, 128)) for i in range(3))
    cat = torch.empty(1, S, 5 * D, device="cuda", dtype=torch.bfloat16)
    win = torch.tensor([[0, S_txt]], dtype=torch.int32, device="cuda")
    bufs = ops.attn_quant_fp8(q, k, v)
    runs = {"bf16": lambda: ops.attention(q, k, v, out=cat[:, :, :D]),
            "bf16_window": lambda: ops.attention(q, k, v, out=cat[:, :, :D], win=win, S_txt=S_txt),
            "fp8": lambda: ops.attention_fp8(*bufs, out=cat[:, :, :D]),
            "fp8_window": lambda: ops.attention_fp8(*bufs, out=cat[:, :, :D], win=win, S_txt=S_txt)}
    t = {k_: [] for k_ in runs}
    for rnd in range(args.rounds):
        order = list(runs) if rnd % 2 == 0 else list(reversed(runs))
        for k_ in order:
            runs[k_]()
            t[k_].append(timed(runs[k_], KERNEL_ITERS))
    res = {"shape": f"B1 H{H} S_txt{S_txt} S{S}"}
    for k_ in ("bf16", "fp8"):
        res[f"{k_}_ms"] = _rng(t[k_])
        res[f"{k_}_window_ms"] = _rng(t[k_ + "_window"])
        res[f"{k_}_window_over_unwindowed"] = _rng([a / b for a, b in zip(t[k_ + "_window"], t[k_])])
    print("kernel", json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=2)
    ap.add_argument("--what", default="step,kernel")
    ap.add_argument("--out-dir", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_ragged.py measures on a CUDA device; none is visible")
    out = {"card": card()}
    what = args.what.split(",")
    if "kernel" in what:
        out["kernel"] = kernel_bench(args)
    if "step" in what:
        out["step"] = step_bench(args)
    out["card_after"] = card()
    print(json.dumps(out))
    if args.out_dir:
        d = Path(args.out_dir)
        d.mkdir(parents=True, exist_ok=True)
        (d / "bench_ragged.json").write_text(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
