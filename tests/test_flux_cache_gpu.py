"""The first-block cache (b2f_flux_forward_cached, include/b2f.h) on the GPU, against the engine's own uncached stages.

Every quantity the cache computes is rebuilt in torch from intermediates of uncached block-range forwards
(`_b2f_block_range` + `debug_hidden`) and compared bit for bit: r_k = float(y0) - float(x0), the saved y0, R =
float(h_final) - float(y0) of a miss, and a hit's output = the engine's tail (block range (nblk, nblk)) on
bf16(y0 + R).  `dist` is checked against its float64 recomputation from the state's r slots.  Pipeline calls check
threshold 0 (bit-identical to the cache off, in bf16, FP8 and with unfused LoRA), the decision log against the host
policy (tests/cache_ref.py) and true CFG's two branches.  The models are the 2 + 2-block d = 3072 ones of
test_flux_blocks_gpu.py.
"""
import ctypes as C
import math

import pytest
import torch

import cache_ref as CR
from test_flux_blocks_gpu import FULL, TOYW, _setup

pytestmark = pytest.mark.gpu

f64, bf16 = torch.float64, torch.bfloat16
BOC = (64, 128, 256, 256)

# name: (width, B, S_txt, latent h, w, n_out, double, single, heavy q/k, LoRA)
CASES = {
    "c1024": (FULL, 1, 544, 64, 64, 4096, 2, 2, False, False),   # the edit's shapes: S_img 8192, n_out 4096
    "ragged": (FULL, 2, 77, 9, 10, 90, 2, 2, False, False),      # S_txt % 8 != 0
    "ragged_b3": (FULL, 3, 77, 9, 10, 90, 2, 2, False, False),   # three batch items pooled into one decision
    "toy": (TOYW, 3, 1, 8, 8, 64, 2, 2, False, False),           # d 256, one text token: the sanitizer's shape
}


def _cfg(threshold):
    from gpt_image_edit_b200.flux_transformer import FirstBlockCacheConfig
    return FirstBlockCacheConfig(threshold=threshold)


def _inputs(s, k):
    """Step k's forward inputs: the hidden states drift a little and the timestep moves, as in a sampling loop."""
    g = torch.Generator(device="cuda").manual_seed(100 + k)
    hs = (s.hs.float() + 0.05 * k * torch.randn(s.hs.shape, device="cuda", generator=g)).bfloat16()
    t = (s.t.float() * (1.0 - 0.125 * k)).bfloat16()
    return dict(hidden_states=hs, encoder_hidden_states=s.enc, pooled_projections=s.pooled, timestep=t, guidance=s.gd)


def _call(s, inp, rng=None, n_out=None):
    jak = {"_b2f_out_rows": n_out or s.n_out}
    if rng is not None:
        jak["_b2f_block_range"] = rng
    if s.scale is not None:
        jak["scale"] = s.scale
    return s.model(**inp, img_ids=s.img_ids, txt_ids=s.txt_ids, return_dict=False, joint_attention_kwargs=jak)[0]


def _img(s):
    return s.model.debug_hidden(s.B, s.S_img, s.S_txt)[:, s.S_txt:]


def _stages(s, inp):
    """Uncached: x0, y0 (image rows after the embedders / block 0), h_final[:n_out] and the output of one forward."""
    _call(s, inp, (0, 0))
    x0 = _img(s).clone()
    _call(s, inp, (0, 1))
    y0 = _img(s).clone()
    out = _call(s, inp).clone()
    hf = _img(s)[:, :s.n_out].clone()
    return x0, y0, hf, out


def _tail_on(s, inp, h_img):
    """The engine's own tail (block range (nblk, nblk)) on the image rows h_img [B, n_out, d]."""
    _call(s, inp, (0, 1))
    _img(s)[:, :s.n_out] = h_img
    return _call(s, inp, (s.nblk, s.nblk)).clone()


def _dist64(r_k, r_prev):
    return CR.residual_distance(r_k, r_prev)


@pytest.mark.parametrize("case", list(CASES))
def test_cached_forward_equals_the_engines_stages(case):
    s = _setup(*CASES[case])
    m = s.model
    A, Bi = _inputs(s, 0), _inputs(s, 1)
    x0A, y0A, hfA, outA = _stages(s, A)
    x0B, y0B, _, outB = _stages(s, Bi)
    rA = y0A.float() - x0A.float()
    rB = y0B.float() - x0B.float()
    RA = hfA.float() - y0A[:, :s.n_out].float()
    hit_out = _tail_on(s, Bi, (y0B[:, :s.n_out].float() + RA).bfloat16())

    m.enable_cache(_cfg(math.inf))
    try:
        # step 0: no state -> a miss, bit-identical to the uncached forward; the state holds r_k, R and y0
        assert torch.equal(_call(s, A), outA)
        e = m.cache_log[-1]
        assert e["hit"] is False and math.isnan(e["dist"]) and e["step"] == 0
        st = m.debug_cache("default", s.B, s.S_img, s.n_out)
        assert st.valid
        assert torch.equal(st.r, rA), "r_k != float(y0) - float(x0)"
        assert torch.equal(st.y0, y0A)
        assert torch.equal(st.R, RA), "R != float(h_final) - float(y0)"
        # step 1: a hit whose output is the engine's tail on bf16(y0 + R); the state does not move
        assert torch.equal(_call(s, Bi), hit_out)
        e = m.cache_log[-1]
        assert e["hit"] is True and e["step"] == 1
        st = m.debug_cache("default", s.B, s.S_img, s.n_out)
        assert torch.equal(st.r, rA) and torch.equal(st.R, RA)
        assert torch.equal(st.r_other, rB), "r_k of the hit"
        ref = _dist64(rB, rA)
        assert abs(e["dist"] - ref) <= 1e-5 * ref, (e["dist"], ref)
        # bit-reproducible: the same call again gives the same distance and output
        d1 = e["dist"]
        assert torch.equal(_call(s, Bi), hit_out)
        assert m.cache_log[-1]["dist"] == d1 and m.cache_log[-1]["hit"]
        # sum |r_prev| == 0: a miss (the full forward runs and becomes the state)
        st.r.zero_()
        assert torch.equal(_call(s, Bi), outB)
        assert m.cache_log[-1]["hit"] is False
        st = m.debug_cache("default", s.B, s.S_img, s.n_out)
        assert torch.equal(st.r, rB)
        # a NaN in r_prev: a miss
        st.r[0, 0, 0] = float("nan")
        assert torch.equal(_call(s, A), outA)
        assert m.cache_log[-1]["hit"] is False and math.isnan(m.cache_log[-1]["dist"])
        assert m.cache_log[-1]["step"] == 4
        # another n_out: the state is invalid (a miss with no distance), then valid for the new shape
        n2 = s.n_out - 1
        out2 = _call(s, A, n_out=n2)
        assert torch.equal(out2, outA[:, :n2])
        assert m.cache_log[-1]["hit"] is False and math.isnan(m.cache_log[-1]["dist"])
        _call(s, A, n_out=n2)
        assert m.cache_log[-1]["hit"] is True
        # one batch item fewer (when there are several): a miss as well
        if s.B > 1:
            one = {k: v[:1] for k, v in A.items()}
            _call(s, one)
            assert m.cache_log[-1]["hit"] is False and math.isnan(m.cache_log[-1]["dist"])
    finally:
        m.disable_cache()


def _pipe(model):
    from gpt_image_edit_b200.pipeline import FluxKontextPipeline
    from gpt_image_edit_b200.scheduler import FlowMatchEulerDiscreteScheduler
    from gpt_image_edit_b200.vae import B200AutoencoderKL, VaeConfig
    from oracle import vae_oracle as vo

    vae = B200AutoencoderKL(VaeConfig(block_out_channels=BOC))
    vae.load_state_dict(vo.make_synthetic_state_dict(vo.VaeConfig(block_out_channels=BOC), seed=4, dtype=bf16,
                                                     device="cuda"))
    return FluxKontextPipeline(transformer=model, vae=vae, scheduler=FlowMatchEulerDiscreteScheduler())


H, W, STEPS = 128, 160, 6


def _pipe_inputs(s, B=2, seed=7):
    g = torch.Generator().manual_seed(seed)
    n = (H // 16) * (W // 16)
    return dict(
        image=(torch.rand(B, 3, H, W, generator=g) * 2 - 1).cuda(),
        prompt_embeds=torch.randn(B, 77, s.ocfg.joint_attention_dim, generator=g).bfloat16().cuda(),
        pooled_prompt_embeds=torch.randn(B, s.ocfg.pooled_projection_dim, generator=g).bfloat16().cuda(),
        negative_prompt_embeds=torch.randn(B, 77, s.ocfg.joint_attention_dim, generator=g).bfloat16().cuda(),
        negative_pooled_prompt_embeds=torch.randn(B, s.ocfg.pooled_projection_dim, generator=g).bfloat16().cuda(),
        latents=torch.randn(B, n, 64, generator=g).bfloat16().cuda())


def _run(pipe, inp, true_cfg=1.0, tracer=None):
    kw = dict(inp)
    kw["latents"] = kw["latents"].clone()
    if true_cfg <= 1.0:
        kw.pop("negative_prompt_embeds")
        kw.pop("negative_pooled_prompt_embeds")
    return pipe(height=H, width=W, num_inference_steps=STEPS, guidance_scale=3.5, max_area=H * W, _auto_resize=False,
                output_type="latent", true_cfg_scale=true_cfg, **kw).images


@pytest.mark.parametrize("mode", ["bf16", "fp8", "lora"])
def test_threshold_zero_pipeline_is_bit_identical_to_the_cache_off(mode):
    s = _setup(*CASES["ragged"][:-1], mode == "lora")
    if mode == "fp8":
        s.model.enable_fp8(linears=True, attention=True)
    pipe = _pipe(s.model)
    inp = _pipe_inputs(s)
    for cfg_scale in (1.0, 2.0):
        off = _run(pipe, inp, cfg_scale)
        s.model.enable_cache(_cfg(0.0))
        on = _run(pipe, inp, cfg_scale)
        log = list(s.model.cache_log)
        s.model.disable_cache()
        assert torch.equal(on, off), f"{mode} true_cfg {cfg_scale}"
        assert len(log) == STEPS * (2 if cfg_scale > 1 else 1) and not any(e["hit"] for e in log)
        assert all(math.isfinite(e["dist"]) == (e["step"] > 0) for e in log)


class _Tracer:
    """Stands in for the transformer: records, after every call, the fp64 distance recomputed from the state's r slots."""

    def __init__(self, model, s):
        self.model, self.s, self.ref = model, s, []

    def __getattr__(self, k):
        return getattr(self.model, k)

    def __call__(self, **kw):
        out = self.model(**kw)
        e = self.model.cache_log[-1]
        B, S_img = kw["hidden_states"].shape[:2]
        st = self.model.debug_cache(e["branch"], B, S_img, kw["joint_attention_kwargs"]["_b2f_out_rows"])
        # a miss moved r_k into the r_prev slot; a hit left r_k in the other one
        r_k, r_prev = (st.r_other, st.r) if e["hit"] else (st.r, st.r_other)
        self.ref.append(_dist64(r_k, r_prev) if e["step"] > 0 else math.nan)
        return out


def _check_log(log, ref, thr):
    for b in {e["branch"] for e in log}:
        mine = [e for e in log if e["branch"] == b]
        assert [e["hit"] for e in mine] == CR.replay(mine, thr), b
    for e, r in zip(log, ref):
        if e["step"] > 0:
            assert abs(e["dist"] - r) <= 1e-5 * r, (e, r)


def test_decisions_follow_the_host_policy_with_true_cfg():
    s = _setup(*CASES["ragged"])
    pipe = _pipe(s.model)
    inp = _pipe_inputs(s)
    m = s.model
    tr = _Tracer(m, s)
    pipe.transformer = tr
    try:
        # +inf: each branch misses on step 0 and hits on every later step
        m.enable_cache(_cfg(math.inf))
        _run(pipe, inp, 2.0)
        for b in ("cond", "uncond"):
            assert [e["hit"] for e in m.cache_log if e["branch"] == b] == [False] + [True] * (STEPS - 1), b
        _check_log(m.cache_log, tr.ref, math.inf)
        # all misses, then a threshold at the median of their distances
        m.enable_cache(_cfg(0.0))
        tr.ref = []
        _run(pipe, inp, 2.0)
        dists = sorted(e["dist"] for e in m.cache_log if e["step"] > 0)
        _check_log(m.cache_log, tr.ref, 0.0)
        thr = dists[len(dists) // 2]
        m.enable_cache(_cfg(thr))
        runs = []
        for _ in range(2):
            tr.ref = []
            lat = _run(pipe, inp, 2.0)
            # NaN (no state yet) as None, so that two logs compare equal
            runs.append((lat, [dict(e, dist=None if math.isnan(e["dist"]) else e["dist"]) for e in m.cache_log]))
            _check_log(m.cache_log, tr.ref, thr)
        print(f"\nmedian threshold {thr:.4g}: " + " ".join(f"{e['branch'][0]}{e['step']}:{'H' if e['hit'] else 'm'}"
                                                        for e in runs[0][1]))
        # two identical calls: bit-identical latents and logs
        assert torch.equal(runs[0][0], runs[1][0])
        assert runs[0][1] == runs[1][1]
        assert any(e["hit"] for e in runs[0][1])
    finally:
        pipe.transformer = m
        m.disable_cache()


def test_what_changes_the_blocks_invalidates_the_state():
    s = _setup(*CASES["ragged"][:-1], True)   # with unfused LoRA adapters
    m = s.model
    A = _inputs(s, 0)
    m.enable_cache(_cfg(math.inf))

    def step():
        _call(s, A)
        return m.cache_log[-1]["hit"]

    def prime():
        step()
        assert step() is True

    try:
        assert step() is False and step() is True
        s.scale = 0.5                      # a new LoRA call scale
        assert step() is False and step() is True
        m.set_adapters(["a"], [1.0])
        assert step() is False
        prime()
        m.fuse_lora()
        assert step() is False
        prime()
        m.enable_fp8(linears=True)
        assert step() is False
        prime()
        m.disable_fp8()
        assert step() is False
        prime()
        m.enable_fp8(attention=True)
        assert step() is False
        prime()
        m.load_state_dict(m.state_dict())
        assert step() is False
        prime()
        m.cache_reset()
        assert m.cache_log == [] and step() is False
    finally:
        m.disable_fp8()
        m.disable_cache()


def test_refusals():
    from gpt_image_edit_b200 import _lib
    from gpt_image_edit_b200._lib import ptr, stream_ptr

    for bad in (-1e-3, float("nan")):
        with pytest.raises(ValueError):
            _cfg(bad)
    s = _setup(*CASES["toy"])
    m = s.model
    A = _inputs(s, 0)
    m.enable_cache(_cfg(0.1))
    try:
        with pytest.raises(_lib.B2FError):
            _call(s, A, (0, 1))
        _call(s, A)
        st = m._cache_states["default"]
        # the C ABI refuses a negative or NaN threshold itself
        hit, dist = C.c_int(), C.c_float()
        out = torch.empty(s.B, s.n_out, 64, device="cuda", dtype=bf16)
        ws = m._ws["fwd"]
        mod = torch.zeros(s.B, m.mod_width, device="cuda", dtype=bf16)
        enc = s.enc.contiguous()
        for bad in (-1.0, float("nan")):
            rc = _lib.lib.b2f_flux_forward_cached(m._h, st.h, bad, ptr(A["hidden_states"]), ptr(enc), ptr(mod),
                                                  mod.stride(0), ptr(out), s.B, s.S_img, s.S_txt, s.n_out, ptr(ws),
                                                  ws.numel(), C.byref(hit), C.byref(dist), stream_ptr())
            assert rc == -1
        # too little state memory
        assert int(_lib.lib.b2f_flux_cache_bytes(m._h, s.B, s.S_img, s.S_txt, s.n_out)) <= st.mem.numel()
        assert int(_lib.lib.b2f_flux_cache_bytes(m._h, s.B, s.S_img, s.S_txt, s.S_img + 1)) == 0
    finally:
        m.disable_cache()
    # a forward with the cache off ignores the branch key
    assert not m.cache_enabled


def test_cli_cache_threshold(tmp_path):
    import numpy as np
    from PIL import Image

    from univa.serve import cli

    rng = np.random.default_rng(0)
    src = tmp_path / "src.png"
    Image.fromarray(rng.integers(0, 256, size=(256, 256, 3), dtype=np.uint8)).save(src)
    out = tmp_path / "out.png"
    args = cli.build_parser().parse_args([
        "--synthetic", "--small", "--prompt", "make the sky purple", "--image", str(src), "--output", str(out),
        "--height", "256", "--width", "256", "--num_inference_steps", "3", "--max_area", str(256 * 256),
        "--cache-threshold", "inf"])
    assert args.cache_threshold == math.inf
    cli.main(args)
    assert np.asarray(Image.open(out)).std() > 0
    assert cli.build_parser().parse_args(["--synthetic"]).cache_threshold is None
