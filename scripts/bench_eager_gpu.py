"""Whole-path GPU comparator (context, NOT the reference arm): one C1024 MMDiT forward of the bf16 oracle on the same
GPU — the reference's op sequence through the libraries it would use on a GPU (cuBLAS nn.Linear, cuDNN / flash SDPA,
ATen norm and elementwise chains) — next to this engine's `b2f_flux_forward` on identical weights and inputs.

    python scripts/bench_eager_gpu.py [--height 1024 --width 1024 --steps 5]     -> gpurun_out/eager_gpu_step.json

oracle/ is test infrastructure: this script is a measurement tool under scripts/, the product never imports it.
Timing: 3 warm-ups, K forwards bracketed by CUDA events; 23.8 GB of weights stream every forward (inputs > L2).
"""
import argparse
import json
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--height", type=int, default=1024)
    ap.add_argument("--width", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=str(ROOT / "gpurun_out" / "eager_gpu_step.json"))
    a = ap.parse_args()
    from gpt_image_edit_b200.flux_transformer import B200FluxTransformer2DModel, FluxTransformerConfig
    from oracle import flux_oracle as fo

    dev = torch.device("cuda")
    model = B200FluxTransformer2DModel(FluxTransformerConfig(), device=dev).randomize_(seed=0)
    sd = dict(model.state_dict())                      # the oracle reads the SAME storage through the diffusers names
    cfg = fo.FluxConfig()
    S_txt, n = 544, (a.height // 16) * (a.width // 16)
    g = torch.Generator(device=dev).manual_seed(1)
    hs = torch.randn(1, 2 * n, 64, device=dev, generator=g).bfloat16()
    enc = torch.randn(1, S_txt, 4096, device=dev, generator=g).bfloat16()
    pooled = torch.randn(1, 768, device=dev, generator=g).bfloat16()
    hh, ww = a.height // 16, a.width // 16
    ids = torch.zeros(hh, ww, 3)
    ids[..., 1] += torch.arange(hh)[:, None]
    ids[..., 2] += torch.arange(ww)[None, :]
    ids = ids.reshape(-1, 3)
    ctx = ids.clone()
    ctx[:, 0] = 1
    img_ids = torch.cat([ids, ctx]).to(dev, torch.bfloat16)
    txt_ids = torch.zeros(S_txt, 3, device=dev, dtype=torch.bfloat16)
    t = torch.full((1,), 0.5, device=dev).bfloat16()
    gd = torch.full((1,), 3.5, device=dev)

    def eager():
        with torch.no_grad():
            return fo.flux_forward(sd, cfg, hs, enc, pooled, t, img_ids, txt_ids, guidance=gd)

    def engine():
        return model(hidden_states=hs, encoder_hidden_states=enc, pooled_projections=pooled, timestep=t, img_ids=img_ids,
                     txt_ids=txt_ids, guidance=gd, return_dict=False)[0]

    def timeit(fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(a.steps):
            out = fn()
        e.record()
        torch.cuda.synchronize()
        return s.elapsed_time(e) / a.steps, out

    res = {"workload": f"one MMDiT forward, {a.height}x{a.width}, S = {S_txt} + {2 * n}, B = 1, bf16, 19 + 38 blocks",
           "sdpa_backends": {}}
    ms_engine, out_e = timeit(engine)
    res["engine_ms"] = ms_engine
    from torch.nn.attention import SDPBackend, sdpa_kernel
    best = None
    for name, be in (("default", None), ("cudnn", SDPBackend.CUDNN_ATTENTION), ("flash", SDPBackend.FLASH_ATTENTION)):
        try:
            if be is None:
                ms, out_o = timeit(eager)
            else:
                with sdpa_kernel(be):
                    ms, out_o = timeit(eager)
            res["sdpa_backends"][name] = ms
            if best is None or ms < best[0]:
                best = (ms, name, out_o)
        except Exception as ex:          # a backend that refuses the shape
            res["sdpa_backends"][name] = f"unavailable: {type(ex).__name__}"
    res["eager_ms"], res["eager_best_backend"] = best[0], best[1]
    res["engine_speedup_over_eager"] = best[0] / ms_engine
    res["rel_l2_engine_vs_eager"] = ((out_e.float() - best[2].float()).norm() / best[2].float().norm()).item()
    res["when"] = time.strftime("%Y-%m-%dT%H:%M:%SZ", time.gmtime())
    Path(a.out).parent.mkdir(exist_ok=True)
    Path(a.out).write_text(json.dumps(res, indent=1))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
