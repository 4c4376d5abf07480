"""The first-block cache policy (tests/cache_ref.py) run over the float64 oracle on the CPU: a short Euler trajectory of a
toy model, with and without true CFG."""
import math

import pytest
import torch

import cache_ref as CR
from oracle import flux_oracle as fo

f64 = torch.float64
STEPS = 5


def _ids(hl, wl, index):
    ids = torch.zeros(hl, wl, 3, dtype=f64)
    ids[..., 0] = index
    ids[..., 1] += torch.arange(hl, dtype=f64)[:, None]
    ids[..., 2] += torch.arange(wl, dtype=f64)[None, :]
    return ids.reshape(-1, 3)


def _setup(B=2, S_txt=5, hl=4, wl=4, seed=0):
    cfg = fo.FluxConfig.toy()
    sd = fo.make_synthetic_state_dict(cfg, seed=seed, dtype=f64)
    g = torch.Generator().manual_seed(seed + 1)
    n = hl * wl
    return dict(
        cfg=cfg, sd=sd, n=n, B=B,
        latents=torch.randn(B, n, cfg.in_channels, generator=g, dtype=f64),
        image=torch.randn(B, n, cfg.in_channels, generator=g, dtype=f64),
        enc=torch.randn(B, S_txt, cfg.joint_attention_dim, generator=g, dtype=f64),
        neg=torch.randn(B, S_txt, cfg.joint_attention_dim, generator=g, dtype=f64),
        pooled=torch.randn(B, cfg.pooled_projection_dim, generator=g, dtype=f64),
        neg_pooled=torch.randn(B, cfg.pooled_projection_dim, generator=g, dtype=f64),
        img_ids=torch.cat([_ids(hl, wl, 0), _ids(hl, wl, 1)]), txt_ids=torch.zeros(S_txt, 3, dtype=f64),
        guidance=torch.full((B,), 3.5, dtype=f64))


def _trajectory(s, forward, true_cfg=None):
    """Euler steps from sigma 1 to 0; forward(branch, enc, pooled, x_in, t) -> velocity of the n target tokens."""
    sig = torch.linspace(1.0, 1.0 / STEPS, STEPS, dtype=f64).tolist() + [0.0]
    lat = s["latents"].clone()
    for i in range(STEPS):
        x_in = torch.cat([lat, s["image"]], dim=1)
        t = torch.full((s["B"],), sig[i], dtype=f64)
        v = forward("cond", s["enc"], s["pooled"], x_in, t)
        if true_cfg is not None:
            vn = forward("uncond", s["neg"], s["neg_pooled"], x_in, t)
            v = vn + true_cfg * (v - vn)
        lat = lat + (sig[i + 1] - sig[i]) * v
    return lat


def _oracle_fwd(s):
    def f(branch, enc, pooled, x_in, t):
        out = fo.flux_forward(s["sd"], s["cfg"], x_in, enc, pooled, t, s["img_ids"], s["txt_ids"], guidance=s["guidance"])
        return out[:, :s["n"]]
    return f


def _cached_fwd(s, co):
    def f(branch, enc, pooled, x_in, t):
        return co.forward(branch, x_in, enc, pooled, t, s["img_ids"], s["txt_ids"], s["guidance"], s["n"])
    return f


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


@pytest.mark.parametrize("true_cfg", [None, 2.0])
def test_threshold_zero_reproduces_the_uncached_trajectory(true_cfg):
    s = _setup()
    ref = _trajectory(s, _oracle_fwd(s), true_cfg)
    co = CR.CachedOracle(s["sd"], s["cfg"], threshold=0.0)
    got = _trajectory(s, _cached_fwd(s, co), true_cfg)
    assert _rel(got, ref) < 1e-12
    assert not any(e["hit"] for e in co.log)
    assert len(co.log) == STEPS * (2 if true_cfg else 1)
    # every call after a branch's first compares with a state: its distance is finite and positive
    assert all(math.isnan(e["dist"]) == (e["step"] == 0) for e in co.log)


def test_infinite_threshold_hits_every_step_after_the_first_and_hits_never_advance_the_state():
    s = _setup()
    co = CR.CachedOracle(s["sd"], s["cfg"], threshold=math.inf)
    seen = []

    def f(branch, enc, pooled, x_in, t):
        out = co.forward(branch, x_in, enc, pooled, t, s["img_ids"], s["txt_ids"], s["guidance"], s["n"])
        st = co.states[branch]
        seen.append((st.r_prev, st.R, st.full_steps))
        return out

    _trajectory(s, f)
    assert [e["hit"] for e in co.log] == [False] + [True] * (STEPS - 1)
    assert CR.replay(co.log, math.inf) == [e["hit"] for e in co.log]
    r0, R0, n0 = seen[0]
    for r, R, n in seen[1:]:
        assert r is r0 and R is R0 and n == n0 == 1   # the state still holds the first (only full) step
    assert all(e["dist"] >= 0 for e in co.log[1:])


def test_mixed_threshold_replays_from_the_reported_distances():
    s = _setup()
    co = CR.CachedOracle(s["sd"], s["cfg"], threshold=0.0)
    _trajectory(s, _cached_fwd(s, co))
    dists = sorted(e["dist"] for e in co.log[1:])
    thr = dists[len(dists) // 2]
    co2 = CR.CachedOracle(s["sd"], s["cfg"], threshold=thr)
    _trajectory(s, _cached_fwd(s, co2))
    assert CR.replay(co2.log, thr) == [e["hit"] for e in co2.log]
    # up to the first hit both runs compare the same states
    assert co2.log[1]["dist"] == co.log[1]["dist"]
    assert not co2.log[0]["hit"]


def test_cond_and_uncond_keep_separate_states():
    s = _setup()
    co = CR.CachedOracle(s["sd"], s["cfg"], threshold=math.inf)
    _trajectory(s, _cached_fwd(s, co), true_cfg=2.0)
    for b in ("cond", "uncond"):
        hits = [e["hit"] for e in co.log if e["branch"] == b]
        assert hits == [False] + [True] * (STEPS - 1), b
        assert co.states[b].full_steps == 1
    assert not torch.equal(co.states["cond"].R, co.states["uncond"].R)
    # one shared state instead would compare the negative prompt's residual with the positive one's
    one = CR.CachedOracle(s["sd"], s["cfg"], threshold=0.0)
    fwd = _cached_fwd(s, one)
    _trajectory(s, lambda b, *a: fwd("shared", *a), true_cfg=2.0)
    sep = [e["dist"] for e in co.log if e["branch"] == "uncond"][1]
    assert one.log[1]["dist"] != sep


def test_shape_change_invalidates_the_state():
    s = _setup()
    co = CR.CachedOracle(s["sd"], s["cfg"], threshold=math.inf)
    f = _cached_fwd(s, co)
    x_in = torch.cat([s["latents"], s["image"]], dim=1)
    t = torch.full((s["B"],), 0.5, dtype=f64)
    f("cond", s["enc"], s["pooled"], x_in, t)
    f("cond", s["enc"], s["pooled"], x_in, t)
    assert [e["hit"] for e in co.log] == [False, True]
    # fewer text tokens: a miss that re-records the state; the same call again hits
    co.forward("cond", x_in, s["enc"][:, :3], s["pooled"], t, s["img_ids"], s["txt_ids"][:3], s["guidance"], s["n"])
    assert co.log[-1]["hit"] is False and co.states["cond"].shape[2] == 3
    # one batch item: a miss as well
    one = lambda a: a[:1]
    co.forward("cond", one(x_in), one(s["enc"]), one(s["pooled"]), one(t), s["img_ids"], s["txt_ids"],
               one(s["guidance"]), s["n"])
    assert co.log[-1]["hit"] is False and co.states["cond"].shape[0] == 1
    co.forward("cond", one(x_in), one(s["enc"]), one(s["pooled"]), one(t), s["img_ids"], s["txt_ids"],
               one(s["guidance"]), s["n"])
    assert co.log[-1]["hit"] is True
    co.reset()
    assert not co.states and not co.log


def test_decision_rule_edges():
    assert not CR.decide(0.0, 0.0)            # strict: threshold 0 never hits
    assert CR.decide(0.0, 1e-9)
    assert not CR.decide(math.nan, math.inf)
    assert not CR.decide(math.inf, math.inf)
    assert CR.decide(1e30, math.inf)
    assert not CR.decide(0.0, 1.0, valid=False)
    z = torch.zeros(3, 4)
    assert CR.residual_distance(torch.ones(3, 4), z) == math.inf   # sum |r_prev| == 0: no finite distance
