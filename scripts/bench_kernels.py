"""Developer micro-benchmark (not bench.py): times libb2f kernels against the library kernels the
reference reaches (cuBLAS via torch.matmul, SDPA) on the same shapes.  Run on an H100; the JSON rows also go to --out-dir."""
import argparse
import json
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from gpt_image_edit_b200 import _lib, ops  # noqa: E402


def timeit(fn, iters=20, warmup=5, flush=None):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    evs = []
    for _ in range(iters):
        if flush is not None:
            flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        evs.append((s, e))
    torch.cuda.synchronize()
    ts = sorted(s.elapsed_time(e) for s, e in evs)
    return ts[len(ts) // 2]


def sustained(fn, seconds=1.2):
    """Average ms per call over `seconds` of back-to-back launches after a 0.6 s heat-up: the power-capped
    steady state a kernel sees inside the 4 s denoising loop (clocks settle near 1.4-1.6 GHz)."""
    t0 = time.time()
    while time.time() - t0 < 0.6:
        for _ in range(20):
            fn()
        torch.cuda.synchronize()
    n = 0
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    t0 = time.time()
    while time.time() - t0 < seconds:
        for _ in range(20):
            fn()
        n += 20
        torch.cuda.synchronize()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / n


def _auto_tile(fn):
    """The tile width the automatic rule gives the launch of `fn`, read from its profiling tag (" t128" / " t256")."""
    _lib.prof_enable(True)
    try:
        _lib.prof_shapes()
        fn()
        tags = [t for t, *_ in _lib.prof_shapes()]
        _lib.prof_collect()
    finally:
        _lib.prof_enable(False)
    return [int(t.rsplit(" t", 1)[1]) for t in tags]


def cublas_kernels():
    """Names of the kernels cuBLAS (torch.nn.functional.linear) runs for the loop's plain-bias GEMM shapes, recorded with
    torch.profiler."""
    from torch.profiler import ProfilerActivity, profile

    d = 3072
    shapes = [(8192, 3 * d, d), (544, 3 * d, d), (8736, 7 * d, d), (8192, d, d), (544, d, d), (8192, 4 * d, d),
              (544, 4 * d, d), (8192, d, 4 * d), (544, d, 4 * d), (8736, d, 5 * d), (8192, 8192, 8192)]
    res = []
    for M, N, K in shapes:
        x = torch.randn(M, K, device="cuda").bfloat16()
        w = (torch.randn(N, K, device="cuda") * K ** -0.5).bfloat16()
        b = torch.randn(N, device="cuda").bfloat16()
        for _ in range(3):
            torch.nn.functional.linear(x, w, b)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            torch.nn.functional.linear(x, w, b)
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        r = dict(kind="cublas_kernels", M=M, N=N, K=K, kernels=sorted(set(names)))
        print(json.dumps(r), flush=True)
        res.append(r)
    return res


def loop_gemms(args, flush):
    """The GEMMs of the 1024^2 edit loop (image M 8192, text M 544, single blocks M 8736, d 3072) and of the text
    encoders (Qwen M 288, T5 M 256), each with the epilogue it runs with; dgrad / wgrad at train512 (S 2336).
    Each forward GEMM is timed with the automatic tile, forced onto 128 x 128 and onto 128 x 256, and beside cuBLAS
    (torch) on its plain-bias twin."""
    from gpt_image_edit_b200 import train_ops as T

    d = 3072
    cases = [
        # name, M, N, K, epilogue
        ("qkv_norm_rope img", 8192, 3 * d, d, "qkv"),
        ("qkv_norm_rope txt", 544, 3 * d, d, "qkv"),
        ("single qkv+mlp split", 8736, 7 * d, d, "qkv_split"),
        ("to_out gate_resid", 8192, d, d, ops.EPI_GATE_RESID),
        ("ff2 gate_resid", 8192, d, 4 * d, ops.EPI_GATE_RESID),
        ("single proj_out gate_resid", 8736, d, 5 * d, ops.EPI_GATE_RESID),
        ("ff1 gelu", 8192, 4 * d, d, ops.EPI_GELU_TANH),
        ("to_out txt gate_resid", 544, d, d, ops.EPI_GATE_RESID),
        ("ff1 txt gelu", 544, 4 * d, d, ops.EPI_GELU_TANH),
        ("ff2 txt gate_resid", 544, d, 4 * d, ops.EPI_GATE_RESID),
        ("adaln M28", 28, 6 * d, d, ops.EPI_BIAS),
        ("adaln single M28", 28, 3 * d, d, ops.EPI_BIAS),
        ("qwen gate_up M288", 288, 2 * 18944, 3584, ops.EPI_BIAS),
        ("qwen down M288", 288, 3584, 18944, ops.EPI_BIAS),
        ("t5 wi M256", 256, 10240, 4096, ops.EPI_BIAS),
        ("t5 wo M256", 256, 4096, 10240, ops.EPI_BIAS),
        ("context_embedder M544", 544, d, 4096, ops.EPI_BIAS),
    ]
    S = 2336
    train = [
        ("dgrad to_out", "dgrad", S, d, d, 0),
        ("dgrad ff2 dgelu", "dgrad", S, 4 * d, d, 8),
        ("dgrad qkv", "dgrad", S, d, 3 * d, 0),
        ("wgrad qkv", "wgrad", 3 * d, d, S, None),
        ("wgrad ff1", "wgrad", 4 * d, d, S, None),
        ("wgrad ff2", "wgrad", d, 4 * d, S, None),
    ]
    t_of = sustained if args.sustained else (lambda f: timeit(f, flush=flush))
    res = []
    for name, M, N, K, epi in cases:
        x = torch.randn(M, K, device="cuda").bfloat16()
        w = (torch.randn(N, K, device="cuda") * K ** -0.5).bfloat16()
        b = torch.randn(N, device="cuda").bfloat16()
        r = dict(kind="loop_gemm", name=name, M=M, N=N, K=K, epi=str(epi), lib=args.tag)
        if epi in ("qkv", "qkv_split"):
            nq = torch.ones(128, device="cuda").bfloat16()
            ang = torch.rand(M, 64, device="cuda") * 6.28
            cos, sin = (f(ang).repeat_interleave(2, 1).contiguous() for f in (torch.cos, torch.sin))
            out = torch.empty(M, 3 * d, device="cuda", dtype=torch.bfloat16)
            extra = torch.empty(M, 4 * d, device="cuda", dtype=torch.bfloat16) if epi == "qkv_split" else None
            fn = lambda: ops.linear_qkv_norm_rope(x, w, b, nq, nq, cos, sin, out=out, out_extra=extra,
                                                  epi_extra=ops.EPI_GELU_TANH)
        else:
            out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
            gate = torch.randn(1, N, device="cuda").bfloat16() if epi == ops.EPI_GATE_RESID else None
            resid = out if epi == ops.EPI_GATE_RESID else None
            fn = lambda: ops.linear(x[None], w, b, epilogue=epi, out=out[None], resid=None if resid is None else resid[None],
                                    gate=gate)
        r["b2f_ms"] = t_of(fn)
        r["b2f_tflops"] = 2.0 * M * N * K / r["b2f_ms"] / 1e9
        # the same launch forced onto each tile of the forward GEMM (b2f_ms above is the automatic choice), and cuBLAS
        # on the shape's plain-bias twin (cuBLAS has none of the fused epilogues)
        for tile in (128, 256):
            _lib.check(_lib.lib.b2f_gemm_set_tile_override(tile), "b2f_gemm_set_tile_override")
            r[f"t{tile}_ms"] = t_of(fn)
            r[f"t{tile}_tflops"] = 2.0 * M * N * K / r[f"t{tile}_ms"] / 1e9
        _lib.check(_lib.lib.b2f_gemm_set_tile_override(0), "b2f_gemm_set_tile_override")
        r["auto_tile"] = _auto_tile(fn)
        r["cublas_ms"] = t_of(lambda: torch.nn.functional.linear(x, w, b))
        r["cublas_tflops"] = 2.0 * M * N * K / r["cublas_ms"] / 1e9
        print(json.dumps(r), flush=True)
        res.append(r)
        del x, w, b, out
    for name, kind, M, N, K, epi in train:
        r = dict(kind="loop_" + kind, name=name, M=M, N=N, K=K, lib=args.tag)
        if kind == "dgrad":
            dy = torch.randn(M, K, device="cuda").bfloat16()
            w = (torch.randn(K, N, device="cuda") * K ** -0.5).bfloat16()
            aux = torch.randn(M, N, device="cuda").bfloat16() if epi else None
            out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
            fn = lambda: T.linear_dgrad(dy, w, epilogue=epi, aux=aux, out=out)
        else:
            dy = torch.randn(1, K, M, device="cuda").bfloat16()
            xx = torch.randn(1, K, N, device="cuda").bfloat16()
            out = torch.zeros(M, N, device="cuda")
            fn = lambda: T.linear_wgrad(dy, xx, out=out, accumulate=True)
        r["b2f_ms"] = t_of(fn)
        r["b2f_tflops"] = 2.0 * M * N * K / r["b2f_ms"] / 1e9
        print(json.dumps(r), flush=True)
        res.append(r)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--what", default="gemm", help="any of gemm, loop (the edit loop's and training's GEMMs), attn")
    ap.add_argument("--sustained", action="store_true")
    ap.add_argument("--cublas-kernels", action="store_true", help="record the cuBLAS kernel names of the loop's GEMM "
                    "shapes with torch.profiler (a run of its own: no timing)")
    ap.add_argument("--tag", default="", help="label of the library under test (B2F_LIB), added to rows and file name")
    ap.add_argument("--out-dir", default="bench_out", help="directory of the bench_kernels_<what>[_<tag>].json file")
    args = ap.parse_args()
    if args.cublas_kernels:
        res = cublas_kernels()
        out_dir = Path(args.out_dir)
        out_dir.mkdir(parents=True, exist_ok=True)
        with open(out_dir / "bench_kernels_cublas_kernels.json", "w") as f:
            json.dump(res, f, indent=1)
        return
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    res = []
    if "gemm" in args.what:
        shapes = [
            (8736, 3072, 3072), (8736, 9216, 3072), (8736, 12288, 3072), (8736, 21504, 3072),
            (8736, 3072, 12288), (8736, 3072, 15360), (8192, 8192, 8192), (544, 9216, 3072),
            (28, 18432, 3072),
        ]
        for M, N, K in shapes:
            x = torch.randn(M, K, device="cuda").bfloat16()
            w = (torch.randn(N, K, device="cuda") * 0.02).bfloat16()
            b = torch.randn(N, device="cuda").bfloat16()
            out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
            if args.sustained:
                t_b2f = sustained(lambda: ops.linear(x, w, b, out=out))
                t_lib = sustained(lambda: torch.nn.functional.linear(x, w, b))
            else:
                t_b2f = timeit(lambda: ops.linear(x, w, b, out=out), flush=flush)
                t_lib = timeit(lambda: torch.nn.functional.linear(x, w, b), flush=flush)
            fl = 2.0 * M * N * K
            r = dict(kind="gemm", M=M, N=N, K=K, b2f_ms=t_b2f, cublas_ms=t_lib,
                     b2f_tflops=fl / t_b2f / 1e9, cublas_tflops=fl / t_lib / 1e9)
            print(json.dumps(r), flush=True)
            res.append(r)
    if "loop" in args.what:
        res += loop_gemms(args, flush)
    if "attn" in args.what:
        from torch.nn.attention import SDPBackend, sdpa_kernel
        for (B, H, S) in [(1, 24, 8736), (1, 24, 2592), (4, 24, 8736)]:
            qkv = torch.randn(B, S, 3 * H * 128, device="cuda").bfloat16()
            q = qkv[:, :, : H * 128].unflatten(-1, (H, 128))
            k = qkv[:, :, H * 128 : 2 * H * 128].unflatten(-1, (H, 128))
            v = qkv[:, :, 2 * H * 128 :].unflatten(-1, (H, 128))
            out = torch.empty(B, S, H * 128, device="cuda", dtype=torch.bfloat16)
            t_b2f = sustained(lambda: ops.attention(q, k, v, out=out)) if args.sustained else \
                timeit(lambda: ops.attention(q, k, v, out=out), iters=10, warmup=3, flush=flush)
            fl = 4.0 * B * H * S * S * 128
            r = dict(kind="attn", B=B, H=H, S=S, b2f_ms=t_b2f, b2f_tflops=fl / t_b2f / 1e9)
            qt, kt, vt = (x.permute(0, 2, 1, 3).contiguous() for x in (q, k, v))
            for name, be in (("flash", SDPBackend.FLASH_ATTENTION), ("cudnn", SDPBackend.CUDNN_ATTENTION),
                             ("efficient", SDPBackend.EFFICIENT_ATTENTION)):
                try:
                    with sdpa_kernel(be):
                        f_ = lambda: torch.nn.functional.scaled_dot_product_attention(qt, kt, vt)
                        t = sustained(f_) if (args.sustained and name == "cudnn") else timeit(f_, iters=10, warmup=3, flush=flush)
                    r[f"sdpa_{name}_ms"] = t
                    r[f"sdpa_{name}_tflops"] = fl / t / 1e9
                except Exception as e:  # backend unavailable for this shape
                    r[f"sdpa_{name}_err"] = str(e)[:80]
            print(json.dumps(r), flush=True)
            res.append(r)
    out_dir = Path(args.out_dir)
    out_dir.mkdir(parents=True, exist_ok=True)
    with open(out_dir / f"bench_kernels_{args.what}{'_' + args.tag if args.tag else ''}.json", "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
