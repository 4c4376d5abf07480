"""First-block cache on the 1024^2 edit (S_txt 544 + S_img 8192 = 8736 tokens, d 3072, 19 + 38 blocks, B = 1), H100.

  step    per-step ms of one transformer forward with the AdaLN modulation hoisted (as the sampling loop runs it), in
          three cache settings alternating within every round: off; threshold 0 (every step a miss: what the cache adds
          to a full step); threshold +inf (every step after the first a hit: the cost of a skipped step).  Each in bf16
          and with FP8 linears + attention.  Reported as the range over --rounds rounds, with torch.cuda.max_memory_allocated
          of each setting.  The timed calls of threshold 0 / +inf are checked to be all misses / all hits.
  traj    for information only: a 28-step Euler trajectory (sigma 1 -> 1/28 -> 0) of synthetic weights with the cache at
          threshold 0 (all misses, identical to the cache off) and at the median of that run's distances: the decision
          log and the final-latent rel-L2 between the two.  Synthetic-weight numbers: they say nothing about the hit
          rate or the image quality of a real checkpoint.
The card's name and power limit are read in the same process.

  python scripts/bench_cache.py [--rounds 3] [--iters 5] [--what step,traj] [--out-dir bench_out]
"""
import argparse
import json
import math
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from bench_lora import card, timed  # noqa: E402

S_TXT, N_IMG, STEPS = 544, 4096, 28


def _rng(v):
    return [min(v), max(v)]


def _model():
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
               img_ids=torch.cat([ids, ctx]).cuda().bfloat16(), txt_ids=torch.zeros(S_TXT, 3, device="cuda").bfloat16(),
               guidance=torch.full((1,), 3.5, device="cuda"))
    return m, inp


def step_bench(args, m, inp):
    from gpt_image_edit_b200 import _lib
    from gpt_image_edit_b200.flux_transformer import FirstBlockCacheConfig
    t = torch.full((1,), 0.5, device="cuda").bfloat16()
    m.prepare_schedule(t, inp["guidance"], inp["pooled_projections"])
    jak = {"_b2f_schedule_step": 0, "_b2f_out_rows": N_IMG, "_b2f_cache_branch": "cond"}
    f = lambda: m(**inp, timestep=t, joint_attention_kwargs=jak, return_dict=False)
    caches = {"off": None, "thr0": 0.0, "inf": math.inf}
    res = {}
    for mode in ("bf16", "fp8+attn"):
        if mode != "bf16":
            m.enable_fp8(linears=True, attention=True)
            m.prepare_schedule(t, inp["guidance"], inp["pooled_projections"])
        per = {c: [] for c in caches}
        peak = {c: 0 for c in caches}
        for rnd in range(args.rounds):
            for c, thr in caches.items():
                if thr is None:
                    m.disable_cache()
                else:
                    m.enable_cache(FirstBlockCacheConfig(threshold=thr))
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                for _ in range(args.warmup):
                    f()
                n0 = len(m.cache_log)
                per[c].append(timed(f, args.iters))
                peak[c] = max(peak[c], torch.cuda.max_memory_allocated())
                if thr is not None:
                    hits = [e["hit"] for e in m.cache_log[n0:]]
                    assert len(hits) == args.iters and all(hits) == (thr == math.inf) and any(hits) == all(hits), hits
            print(f"{mode} round {rnd}: " + ", ".join(f"{c} {per[c][-1]:.2f} ms" for c in per), flush=True)
        m.disable_cache()
        r = {c: {"step_ms": _rng(v), "max_memory_allocated_GB": peak[c] / 1e9} for c, v in per.items()}
        r["thr0_minus_off_ms"] = _rng([a - b for a, b in zip(per["thr0"], per["off"])])
        r["inf_over_off"] = _rng([a / b for a, b in zip(per["inf"], per["off"])])
        r["cache_state_MB"] = int(_lib.lib.b2f_flux_cache_bytes(m._h, 1, 2 * N_IMG, S_TXT, N_IMG)) / 1e6
        res[mode] = r
        print(mode, json.dumps(r), flush=True)
    m.disable_fp8()
    return res


def trajectory(m, inp, thr):
    """28 Euler steps of the cached forward at threshold thr -> (final latents, decision log)."""
    from gpt_image_edit_b200.flux_transformer import FirstBlockCacheConfig
    sig = [1.0 - i / STEPS for i in range(STEPS)] + [0.0]
    ts = torch.tensor(sig[:STEPS], device="cuda").bfloat16()
    m.prepare_schedule(ts, inp["guidance"], inp["pooled_projections"])
    m.enable_cache(FirstBlockCacheConfig(threshold=thr))
    lat = inp["hidden_states"][:, :N_IMG].clone()
    img = inp["hidden_states"][:, N_IMG:]
    kw = {k: v for k, v in inp.items() if k != "hidden_states"}
    for i in range(STEPS):
        jak = {"_b2f_schedule_step": i, "_b2f_out_rows": N_IMG, "_b2f_cache_branch": "cond"}
        v = m(hidden_states=torch.cat([lat, img], 1), timestep=ts[i:i + 1], **kw, joint_attention_kwargs=jak,
              return_dict=False)[0]
        lat = (lat.float() + (sig[i + 1] - sig[i]) * v.float()).bfloat16()
    log = list(m.cache_log)
    m.disable_cache()
    return lat, log


def traj_bench(m, inp):
    ref, log0 = trajectory(m, inp, 0.0)
    dists = sorted(e["dist"] for e in log0[1:])
    thr = dists[len(dists) // 2]
    lat, log = trajectory(m, inp, thr)
    rel = ((lat.double() - ref.double()).norm() / ref.double().norm()).item()
    res = {"note": "synthetic weights: says nothing about real checkpoints or images",
           "all_miss_dists": [e["dist"] for e in log0],
           "threshold": thr, "decisions": "".join("H" if e["hit"] else "m" for e in log),
           "hits": sum(e["hit"] for e in log), "final_latent_rel_l2_to_uncached": rel}
    print("traj", json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--what", default="step,traj")
    ap.add_argument("--out-dir", default="bench_out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_cache.py measures on the GPU; no CUDA device is visible")
    res = {"card_before": card(), "time": time.strftime("%Y-%m-%d %H:%M:%S")}
    m, inp = _model()
    if "step" in args.what:
        res["step"] = step_bench(args, m, inp)
    if "traj" in args.what:
        res["traj"] = traj_bench(m, inp)
    res["card_after"] = card()
    Path(args.out_dir).mkdir(parents=True, exist_ok=True)
    (Path(args.out_dir) / "bench_cache.json").write_text(json.dumps(res, indent=1))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
