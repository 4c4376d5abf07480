"""LoRA cost on the 1024^2 edit (S_txt 544 + S_img 8192 = 8736 tokens, d 3072, 19 + 38 blocks, B = 1), H100.

Per-step ms of one transformer forward with the AdaLN modulation hoisted (as the sampling loop runs it), and the
denoise-only images/s that implies (28 steps), for:
  none            no adapter
  unfused x1      one synthetic adapter of rank r on every block linear (to_q/k/v, add_*_proj, to_out.0, to_add_out,
                  ff*, ff_context*, proj_mlp, single proj_out), run as down projection + K-extended GEMM
  unfused x2      two such adapters (ranks concatenated: one down projection and one K-extension per linear)
  fused           the x1 adapter merged into the weights (fuse_lora)
for r = 16 and 64.  The configurations alternate within every round (none first), rounds repeat --rounds times and
each number is reported as the range over the rounds.  Then the K-extended GEMM's TFLOP/s on the loop shapes beside
the plain kernel, alternating.  The card's name and power limit are read in the same process.

  python scripts/bench_lora.py [--rounds 3] [--iters 5] [--out-dir bench_out]
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", "0"], capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable ({e})"
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q}


def block_modules(cfg):
    out = []
    for i in range(cfg.num_layers):
        p = f"transformer_blocks.{i}."
        out += [p + "attn." + n for n in ("to_q", "to_k", "to_v", "add_q_proj", "add_k_proj", "add_v_proj",
                                           "to_out.0", "to_add_out")]
        out += [p + n for n in ("ff.net.0.proj", "ff.net.2", "ff_context.net.0.proj", "ff_context.net.2")]
    for i in range(cfg.num_single_layers):
        p = f"single_transformer_blocks.{i}."
        out += [p + "attn.to_q", p + "attn.to_k", p + "attn.to_v", p + "proj_mlp", p + "proj_out"]
    return out


def synthetic_lora(cfg, rank, seed):
    from gpt_image_edit_b200 import lora as L
    parts = L.diffusers_parts(cfg)
    g = torch.Generator(device="cuda").manual_seed(seed)
    sd = {}
    for n in block_modules(cfg):
        p = parts[n]
        sd[f"transformer.{n}.lora_A.weight"] = (torch.randn(rank, p.in_features, device="cuda", generator=g)
                                                * p.in_features ** -0.5).bfloat16()
        sd[f"transformer.{n}.lora_B.weight"] = (torch.randn(p.rows, rank, device="cuda", generator=g) * 0.01).bfloat16()
        sd[f"transformer.{n}.alpha"] = torch.tensor(float(rank))
    return sd


def timed(fn, iters):
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def step_bench(args):
    from gpt_image_edit_b200.flux_transformer import B200FluxTransformer2DModel, FluxTransformerConfig
    cfg = FluxTransformerConfig()
    m = B200FluxTransformer2DModel(cfg).randomize_(seed=0)
    g = torch.Generator(device="cuda").manual_seed(1)
    S_txt, n = 544, 4096
    side = 64
    ids = torch.stack([torch.zeros(n), torch.arange(n) // side, torch.arange(n) % side], 1)
    ctx = ids.clone()
    ctx[:, 0] = 1
    inp = dict(hidden_states=torch.randn(1, 2 * n, 64, device="cuda", generator=g).bfloat16(),
               encoder_hidden_states=torch.randn(1, S_txt, 4096, device="cuda", generator=g).bfloat16(),
               pooled_projections=torch.randn(1, 768, device="cuda", generator=g).bfloat16(),
               timestep=torch.full((1,), 0.5, device="cuda").bfloat16(),
               img_ids=torch.cat([ids, ctx]).cuda().bfloat16(), txt_ids=torch.zeros(S_txt, 3, device="cuda").bfloat16(),
               guidance=torch.full((1,), 3.5, device="cuda"))

    def fwd():
        m.prepare_schedule(inp["timestep"], inp["guidance"], inp["pooled_projections"])
        jak = {"_b2f_schedule_step": 0, "_b2f_out_rows": n}
        return lambda: m(**inp, joint_attention_kwargs=jak, return_dict=False)

    results = {}
    for rank in args.ranks:
        loras = [synthetic_lora(cfg, rank, 10 + rank), synthetic_lora(cfg, rank, 20 + rank)]
        confs = ["none", "unfused x1", "unfused x2", "fused"]
        per = {c: [] for c in confs}
        for rnd in range(args.rounds):
            for conf in confs:
                m.unload_lora()
                if conf != "none":
                    m.load_lora_adapter(loras[0], adapter_name="a")
                if conf == "unfused x2":
                    m.load_lora_adapter(loras[1], adapter_name="b")
                if conf == "fused":
                    m.fuse_lora()
                f = fwd()
                for _ in range(args.warmup):
                    f()
                per[conf].append(timed(f, args.iters))
                if conf == "fused":
                    m.unfuse_lora()
                m.unload_lora()
            print(f"r={rank} round {rnd}: " + ", ".join(f"{c} {per[c][-1]:.1f} ms" for c in confs), flush=True)
        base = per["none"]
        results[f"r{rank}"] = {c: {"step_ms": [min(v), max(v)], "denoise_img_per_s": [1000 / (28 * max(v)),
                                                                                      1000 / (28 * min(v))],
                                   "vs_none": [min(a / b for a, b in zip(v, base)), max(a / b for a, b in zip(v, base))]}
                               for c, v in per.items()}
        del loras
    del m
    torch.cuda.empty_cache()
    return results


def gemm_bench(args):
    from gpt_image_edit_b200 import ops
    d = 3072
    shapes = [("qkv img", 8192, 3 * d, d), ("single qkv+mlp", 8736, 7 * d, d), ("to_out", 8192, d, d),
              ("ff1", 8192, 4 * d, d), ("ff2", 8192, d, 4 * d), ("single proj_out", 8736, d, 5 * d)]
    g = torch.Generator(device="cuda").manual_seed(3)
    out = {}
    for name, M, N, K in shapes:
        x = torch.randn(M, K, device="cuda", generator=g).bfloat16()
        w = (torch.randn(N, K, device="cuda", generator=g) * K ** -0.5).bfloat16()
        b = torch.zeros(N, device="cuda", dtype=torch.bfloat16)
        y = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        row = {}
        for r_pad in (64, 256):
            t = torch.randn(M, r_pad, device="cuda", generator=g).bfloat16()
            bc = (torch.randn(N, r_pad, device="cuda", generator=g) * 0.01).bfloat16()
            a = (torch.randn(r_pad, K, device="cuda", generator=g) * K ** -0.5).bfloat16()
            cs = torch.ones(r_pad, device="cuda")
            plain, ext, down = [], [], []
            for _ in range(args.rounds):
                plain.append(timed(lambda: ops.linear(x, w, b, out=y), 20))
                ext.append(timed(lambda: ops.linear_lora(x, w, b, t, bc, out=y), 20))
                down.append(timed(lambda: ops.lora_down(x, a, cs, out=t), 20))
            fl = 2.0 * M * N * K
            row[f"r_pad{r_pad}"] = {
                "plain_tflops": [fl / max(plain) / 1e9, fl / min(plain) / 1e9],
                "kext_tflops_incl_ext": [fl * (1 + r_pad / K) / max(ext) / 1e9, fl * (1 + r_pad / K) / min(ext) / 1e9],
                "kext_time_vs_plain": [min(e / p for e, p in zip(ext, plain)), max(e / p for e, p in zip(ext, plain))],
                "down_ms": [min(down), max(down)]}
        out[f"{name} {M}x{N}x{K}"] = row
        print(name, json.dumps(row), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ranks", type=int, nargs="+", default=[16, 64])
    ap.add_argument("--what", default="step,gemm")
    ap.add_argument("--out-dir", default="bench_out")
    args = ap.parse_args()
    res = {"card_before": card(), "time": time.strftime("%Y-%m-%d %H:%M:%S")}
    if "step" in args.what:
        res["step"] = step_bench(args)
    if "gemm" in args.what:
        res["gemm"] = gemm_bench(args)
    res["card_after"] = card()
    Path(args.out_dir).mkdir(parents=True, exist_ok=True)
    (Path(args.out_dir) / "bench_lora.json").write_text(json.dumps(res, indent=1))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
