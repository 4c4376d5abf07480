"""GPU parity of the training step's forward/backward graph (MLP2 -> FLUX denoiser with per-block recompute)
against torch.autograd over the oracle (reference train_denoiser.py:1073-1172 reaches the same gradients through
autograd over diffusers' modules).

Every gradient the engine produces — the reference's trainable set (train_denoiser.py:71-119) plus MLP2 — is compared
with the fp32 oracle's autograd on identical bf16-rounded weights; the torch-bf16 autograd of the same oracle is
compared with the fp32 one as well, and the engine's error must stay within 2x torch-bf16's + 1e-2 (the rule
used for composed models).
"""
from types import SimpleNamespace

import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-20)).item()


def _setup(nd=2, ns=2, heads=2, B=2, L=32, hw=8, seed=0, heavy=False):
    from gpt_image_edit_b200.flux_transformer import B200FluxTransformer2DModel, FluxTransformerConfig
    from oracle import flux_oracle as fo
    from univa.models.modeling_univa_denoise_tower import DenoiseProjector

    toy = dict(num_layers=nd, num_single_layers=ns, attention_head_dim=128, num_attention_heads=heads,
               joint_attention_dim=256, pooled_projection_dim=64)
    ocfg = fo.FluxConfig(**toy)
    sd = fo.make_synthetic_state_dict(ocfg, seed=seed, dtype=torch.bfloat16, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    # non-trivial norm weights and AdaLN biases so that every gradient path carries signal
    for k in sd:
        if "norm_q" in k or "norm_k" in k or "norm_added" in k:
            sd[k] = (1.0 + 0.2 * torch.randn(sd[k].shape, device="cuda", generator=g)).bfloat16()
        if heavy and k.endswith("attn.to_q.weight"):
            sd[k] = (sd[k].float() * 6).bfloat16()          # peaked attention rows
    den = B200FluxTransformer2DModel(FluxTransformerConfig(**toy))
    den.load_state_dict(sd)
    proj = DenoiseProjector(128, 256)
    for t in proj.state_dict().values():
        t.copy_((torch.randn(t.shape, device="cuda", generator=g) * 0.05).bfloat16())
    model = SimpleNamespace(denoise_tower=SimpleNamespace(denoiser=den, denoise_projector=proj))
    n = hw * hw
    x = torch.randn(B, L, 128, device="cuda", generator=g).bfloat16()
    hs = torch.randn(B, 2 * n, 64, device="cuda", generator=g).bfloat16()
    pooled = torch.randn(B, 64, device="cuda", generator=g).bfloat16()
    ids = torch.zeros(hw, hw, 3)
    ids[..., 1] += torch.arange(hw)[:, None]
    ids[..., 2] += torch.arange(hw)[None, :]
    ids = ids.reshape(-1, 3)
    ctx = ids.clone()
    ctx[:, 0] = 1
    img_ids = torch.cat([ids, ctx]).to("cuda", torch.bfloat16)
    t = torch.tensor([0.5, 0.25][:B], device="cuda").bfloat16()      # t * 1000 exact in bf16
    gd = torch.full((B,), 1.0, device="cuda")
    target = torch.randn(B, n, 64, device="cuda", generator=g)
    return SimpleNamespace(ocfg=ocfg, sd=sd, model=model, den=den, proj=proj, x=x, hs=hs, pooled=pooled, img_ids=img_ids, t=t,
                           gd=gd, target=target, n=n, L=L, B=B)


def _oracle_grads(s, dtype):
    """loss and gradients of the oracle (autograd) with every tensor cast to `dtype`."""
    from oracle import flux_oracle as fo

    sd = {k: v.to(dtype).clone().requires_grad_(True) for k, v in s.sd.items()}
    pw = {k: v.to(dtype).clone().requires_grad_(True) for k, v in s.proj.state_dict().items()}
    x = s.x.to(dtype)
    h = torch.nn.functional.silu(torch.nn.functional.linear(x, pw["0.weight"], pw["0.bias"]))
    enc = torch.nn.functional.linear(h, pw["2.weight"], pw["2.bias"])
    txt_ids = torch.zeros(s.L, 3, device="cuda", dtype=torch.bfloat16)
    out = fo.flux_forward(sd, s.ocfg, s.hs.to(dtype), enc, s.pooled.to(dtype), s.t.to(dtype), s.img_ids, txt_ids, guidance=s.gd)
    pred = out[:, :s.n]
    loss = ((pred.float() - s.target) ** 2).mean()
    loss.backward()
    return loss.detach(), {k: v.grad for k, v in sd.items()}, {k: v.grad for k, v in pw.items()}, pred.detach()


def _ref_for(name, gsd, gpw):
    """oracle gradient for a Param of training.trainable_params (fused names -> concatenated diffusers tensors)."""
    if name.startswith("denoise_projector."):
        return gpw[name[len("denoise_projector."):]]
    if "to_q|to_k|to_v" in name:
        suffix = name.rsplit(".", 1)[1]
        base = name.split("attn.")[0] + "attn."
        return torch.cat([gsd[f"{base}{p}.{suffix}"] for p in ("to_q", "to_k", "to_v")], 0)
    return gsd[name]


@pytest.mark.parametrize("heavy", [False, True])
def test_flux_train_graph_matches_oracle_autograd(heavy):
    from gpt_image_edit_b200 import training as tr

    s = _setup(heavy=heavy)
    params = tr.trainable_params(s.model)
    opt = tr.ShardedAdamW(params, lr=1e-4)            # allocates the fp32 gradient buckets
    graph = tr.FluxTrainGraph(s.model, params)
    pred = graph.forward(s.x, s.hs, s.t, s.gd, s.pooled, s.img_ids, s.n)
    # the training forward runs the inference kernels block by block: identical to one inference call
    txt_ids = torch.zeros(s.L, 3, device="cuda", dtype=torch.bfloat16)
    enc = s.proj(s.x)
    ref_fwd = s.den(hidden_states=s.hs, encoder_hidden_states=enc, pooled_projections=s.pooled, timestep=s.t,
                    img_ids=s.img_ids, txt_ids=txt_ids, guidance=s.gd, return_dict=False)[0][:, :s.n]
    assert torch.equal(pred, ref_fwd)
    loss, dpred = tr.flow_matching_loss(pred, s.target)
    graph.backward(dpred)
    torch.cuda.synchronize()

    l32, g32, p32, pred32 = _oracle_grads(s, torch.float32)
    l16, g16, p16, _ = _oracle_grads(s, torch.bfloat16)
    assert abs(loss.item() - l32.item()) < 2e-2 * l32.item()
    worst = 0.0
    report = []
    for p in params:
        ref = _ref_for(p.name, g32, p32)
        ref16 = _ref_for(p.name, g16, p16)
        assert ref is not None, p.name
        e_k, e_t = _rel(p.grad, ref), _rel(ref16, ref)
        report.append((p.name, e_k, e_t))
        worst = max(worst, e_k - 2 * e_t)
        assert torch.isfinite(p.grad).all(), p.name
    bad = [(n, round(a, 4), round(b, 4)) for n, a, b in report if a > 2 * b + 1e-2]
    print("\n".join(f"{n:60s} kernel {a:.3e}  torch-bf16 {b:.3e}" for n, a, b in report))
    assert not bad, bad


def test_flux_train_backward_block_by_block_equals_one_call_and_accumulates():
    from gpt_image_edit_b200 import training as tr

    s = _setup(nd=1, ns=1, B=1)
    params = tr.trainable_params(s.model)
    tr.ShardedAdamW(params, lr=1e-4)
    graph = tr.FluxTrainGraph(s.model, params)
    pred = graph.forward(s.x, s.hs, s.t, s.gd, s.pooled, s.img_ids, s.n)
    _, dpred = tr.flow_matching_loss(pred, s.target)
    graph.backward(dpred)
    one = [p.grad.clone() for p in params]
    done = []
    graph2 = tr.FluxTrainGraph(s.model, params, on_block_done=done.append)
    pred2 = graph2.forward(s.x, s.hs, s.t, s.gd, s.pooled, s.img_ids, s.n)
    assert torch.equal(pred, pred2)
    graph2.backward(dpred)
    assert done == [1, 0, 2]                                   # blocks in reverse order, then the MLP2 bucket
    for p, g in zip(params, one):
        assert torch.equal(p.grad, g), p.name                  # deterministic kernels: bit-identical
    graph2.backward(dpred, accumulate=True)
    for p, g in zip(params, one):
        assert _rel(p.grad, 2 * g) < 1e-5, p.name


def test_sharded_adamw_single_rank_updates_model_storage():
    from gpt_image_edit_b200 import training as tr

    s = _setup(nd=1, ns=1, B=1)
    params = tr.trainable_params(s.model)
    before = {p.name: p.storage.clone() for p in params}
    opt = tr.ShardedAdamW(params, lr=1e-2, weight_decay=0.0, max_grad_norm=1.0)
    graph = tr.FluxTrainGraph(s.model, params)
    losses = []
    for _ in range(4):
        pred = graph.forward(s.x, s.hs, s.t, s.gd, s.pooled, s.img_ids, s.n)
        loss, dpred = tr.flow_matching_loss(pred, s.target)
        graph.backward(dpred)
        norm = opt.step()
        losses.append(loss.item())
        assert torch.isfinite(norm).all()
    assert any(not torch.equal(before[p.name], p.storage) for p in params)
    assert losses[-1] < losses[0], losses                     # four steps on one sample reduce its loss
    # the fused views still alias the trained storage (diffusers names see the update)
    sd = s.den.state_dict()
    assert sd["transformer_blocks.0.attn.to_k.weight"].data_ptr() != 0
    assert not torch.equal(sd["transformer_blocks.0.attn.to_k.weight"], s.sd["transformer_blocks.0.attn.to_k.weight"])
