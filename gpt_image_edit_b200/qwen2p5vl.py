"""Qwen2.5-VL conditioning prefill (ViT + 28-layer decoder, final norm) over libb2f kernels — the
compute behind `UnivaQwen2p5VLForConditionalGeneration.forward(output_type="denoise_embeds")`
(reference univa/models/qwen2p5vl/modeling_univa_qwen2p5vl.py:325-530; arithmetic from
transformers' Qwen2_5_VL modules, SURVEY.md Appendix B).

Every matmul is `b2f_gemm_bf16` (wgmma), every attention is `b2f_attention_fwd` (causal GQA for
the decoder; windowed / full bidirectional for the ViT, head_dim 80 zero-padded to 128 in the weight
layout so no activation is ever re-laid-out), norms / RoPE / SwiGLU / gathers are the HBM-bound
kernels of csrc/llm_kernels.cu.  Python here only sequences C-ABI calls and does integer position
bookkeeping (window order, M-RoPE ids) on the host.

State-dict keys are the transformers-4.50 names the reference checkpoint uses (`visual.*`,
`model.layers.*`, `model.embed_tokens`, `model.norm`).
"""
from __future__ import annotations

from collections import OrderedDict
from types import SimpleNamespace

import torch
import torch.nn.functional as F

from . import _lib, ops


class QwenVisionConfig(SimpleNamespace):
    def __init__(self, **kw):
        base = dict(depth=32, hidden_size=1280, num_heads=16, intermediate_size=3420, in_channels=3, patch_size=14,
                    temporal_patch_size=2, spatial_merge_size=2, window_size=112, fullatt_block_indexes=(7, 15, 23, 31),
                    out_hidden_size=3584, tokens_per_second=2)
        base.update(kw)
        super().__init__(**base)


class QwenTextConfig(SimpleNamespace):
    def __init__(self, **kw):
        base = dict(hidden_size=3584, num_hidden_layers=28, num_attention_heads=28, num_key_value_heads=4,
                    intermediate_size=18944, vocab_size=152064, rms_norm_eps=1e-6, rope_theta=1000000.0,
                    mrope_section=(16, 24, 24), image_token_id=151655, video_token_id=151656,
                    vision_start_token_id=151652)
        base.update(kw)
        super().__init__(**base)


def _pad8(n: int) -> int:
    return (n + 7) // 8 * 8


# ------------------------------------------------------------------------------------------------ host logic
def get_rope_index(input_ids: torch.Tensor, image_grid_thw: torch.Tensor | None, attention_mask=None, *,
                   spatial_merge_size=2, image_token_id=151655, vision_start_token_id=151652):
    """M-RoPE position ids [3, B, L] (t, h, w) and deltas [B, 1] for text + still images — the image
    branch of the reference's get_rope_index (modeling_univa_qwen2p5vl.py:139-318: text runs count up on
    all three axes, an image of llm grid h x w gets t = const, h = row, w = col offset by the running
    position, text resumes at max + 1; a trailing <|vision_start|> without image tokens is ignored)."""
    B, L = input_ids.shape
    ids_cpu = input_ids.cpu()
    mask = torch.ones_like(ids_cpu) if attention_mask is None else attention_mask.cpu()
    if image_grid_thw is None:
        pos = (mask.long().cumsum(-1) - 1).masked_fill(mask == 0, 1)
        pos = pos.unsqueeze(0).expand(3, -1, -1).contiguous()
        delta = pos.max(0)[0].max(-1, keepdim=True)[0] + 1 - L
        return pos.to(input_ids.device), delta.to(input_ids.device)
    grids = image_grid_thw.cpu().tolist() if torch.is_tensor(image_grid_thw) else [list(g) for g in image_grid_thw]
    pos = torch.ones(3, B, L, dtype=torch.long)
    deltas = []
    img_i = 0
    for b in range(B):
        toks = ids_cpu[b][mask[b] == 1].tolist()
        starts = [i for i, t in enumerate(toks) if t == vision_start_token_id and i + 1 < len(toks)]
        n_images = sum(1 for i in starts if toks[i + 1] == image_token_id)
        chunks = []
        st = 0
        nxt = 0
        for _ in range(n_images):
            ed = toks.index(image_token_id, st)
            t, h, w = grids[img_i]
            img_i += 1
            gh, gw = h // spatial_merge_size, w // spatial_merge_size
            text_len = ed - st
            chunks.append(torch.arange(text_len).view(1, -1).expand(3, -1) + nxt)
            base = nxt + text_len
            t_idx = torch.zeros(t * gh * gw, dtype=torch.long)                 # still images: temporal id 0
            h_idx = torch.arange(gh).view(1, -1, 1).expand(t, -1, gw).flatten()
            w_idx = torch.arange(gw).view(1, 1, -1).expand(t, gh, -1).flatten()
            chunks.append(torch.stack([t_idx, h_idx, w_idx]) + base)
            nxt = int(chunks[-1].max()) + 1
            st = ed + t * gh * gw
        if st < len(toks):
            chunks.append(torch.arange(len(toks) - st).view(1, -1).expand(3, -1) + nxt)
        llm = torch.cat(chunks, dim=1)
        pos[:, b, mask[b] == 1] = llm
        deltas.append(int(llm.max()) + 1 - L)
    return pos.to(input_ids.device), torch.tensor(deltas).unsqueeze(1).to(input_ids.device)


def vision_window_index(grid_thw, *, window_size=112, spatial_merge_size=2, patch_size=14):
    """Window permutation of the merged-token grid and the cumulative window lengths (in patches) —
    transformers get_window_index."""
    window_index, cu = [], [0]
    offset = 0
    vw = window_size // spatial_merge_size // patch_size
    unit = spatial_merge_size * spatial_merge_size
    for t, h, w in grid_thw:
        gh, gw = h // spatial_merge_size, w // spatial_merge_size
        idx = torch.arange(t * gh * gw).reshape(t, gh, gw)
        ph, pw = vw - gh % vw, vw - gw % vw
        nh, nw = (gh + ph) // vw, (gw + pw) // vw
        padded = F.pad(idx, (0, pw, 0, ph), "constant", -100).reshape(t, nh, vw, nw, vw)
        padded = padded.permute(0, 1, 3, 2, 4).reshape(t, nh * nw, vw, vw)
        seqlens = (padded != -100).sum([2, 3]).reshape(-1)
        flat = padded.reshape(-1)
        window_index.append(flat[flat != -100] + offset)
        cu.extend((seqlens.cumsum(0) * unit + cu[-1]).tolist())
        offset += t * gh * gw
    cu_t = torch.unique_consecutive(torch.tensor(cu))
    return torch.cat(window_index), cu_t.tolist()


def vision_rot_pos_ids(grid_thw, spatial_merge_size=2):
    """(h, w) position of every patch in the processor's 2x2-merge order — transformers rot_pos_emb."""
    out = []
    m = spatial_merge_size
    for t, h, w in grid_thw:
        hp = torch.arange(h).unsqueeze(1).expand(-1, w).reshape(h // m, m, w // m, m).permute(0, 2, 1, 3).flatten()
        wp = torch.arange(w).unsqueeze(0).expand(h, -1).reshape(h // m, m, w // m, m).permute(0, 2, 1, 3).flatten()
        out.append(torch.stack([hp, wp], dim=-1).repeat(t, 1))
    return torch.cat(out, dim=0)


# ------------------------------------------------------------------------------------------------ model
def padding_spans(attention_mask):
    """[(lo, hi)] per batch row: the run of ones of a 2-D attention mask (right- or left-padded prompts, as the
    processor's `padding=True` produces them).  Holes inside a prompt are not a padding pattern and are refused."""
    am = attention_mask.detach().to("cpu") != 0
    if am.dim() != 2:
        raise _lib.B2FError(f"attention_mask: expected [B, L], got {tuple(am.shape)}")
    spans = []
    for b in range(am.shape[0]):
        idx = am[b].nonzero().squeeze(1)
        if idx.numel() == 0:
            raise _lib.B2FError(f"attention_mask row {b} is empty")
        lo, hi = int(idx[0]), int(idx[-1]) + 1
        if hi - lo != idx.numel():
            raise _lib.B2FError(f"attention_mask row {b} is not one contiguous run of ones (left or right padding)")
        spans.append((lo, hi))
    return spans


class B200Qwen2p5VL(torch.nn.Module):
    """Weights in kernel layout + the prefill forward.  `denoise_projector` (MLP2) is owned by the
    denoise tower (univa.models.modeling_univa_denoise_tower)."""

    HP = 128  # head slot pitch (vision head_dim 80 is zero-padded to 128)

    def __init__(self, text: QwenTextConfig | None = None, vision: QwenVisionConfig | None = None, device="cuda"):
        super().__init__()
        self.tc, self.vc = text or QwenTextConfig(), vision or QwenVisionConfig()
        dev = torch.device(device)
        if dev.type != "cuda":
            raise _lib.B2FError("B200Qwen2p5VL lives on a CUDA device; there is no CPU path")
        self._dev = dev
        tc, vc = self.tc, self.vc
        self.vhd = vc.hidden_size // vc.num_heads           # 80
        self.vi = _pad8(vc.intermediate_size)                # 3424
        self.thd = tc.hidden_size // tc.num_attention_heads
        W = self.W = self.alloc_weights(tc, vc, dev)
        for k, t in W.items():
            self.register_buffer("w__" + k.replace(".", "__"), t, persistent=False)

    @classmethod
    def alloc_weights(cls, tc, vc, dev) -> "OrderedDict[str, torch.Tensor]":
        """Zeroed weight storage in kernel layout (fused q|k|v and gate|up, vision heads padded 80 -> 128, padded MLP width)."""
        z = lambda *s: torch.zeros(s, device=dev, dtype=torch.bfloat16)
        o = lambda *s: torch.ones(s, device=dev, dtype=torch.bfloat16)
        vi = _pad8(vc.intermediate_size)
        HPv = vc.num_heads * cls.HP
        pe_in = vc.in_channels * vc.temporal_patch_size * vc.patch_size ** 2
        W = OrderedDict()
        W["visual.patch_embed"] = z(vc.hidden_size, pe_in)
        for i in range(vc.depth):
            p = f"visual.blocks.{i}."
            W[p + "norm1"], W[p + "norm2"] = o(vc.hidden_size), o(vc.hidden_size)
            W[p + "qkv.w"], W[p + "qkv.b"] = z(3 * HPv, vc.hidden_size), z(3 * HPv)
            W[p + "proj.w"], W[p + "proj.b"] = z(vc.hidden_size, HPv), z(vc.hidden_size)
            W[p + "gu.w"], W[p + "gu.b"] = z(2 * vi, vc.hidden_size), z(2 * vi)
            W[p + "down.w"], W[p + "down.b"] = z(vc.hidden_size, vi), z(vc.hidden_size)
        mh = vc.hidden_size * vc.spatial_merge_size ** 2
        W["visual.merger.ln_q"] = o(vc.hidden_size)
        W["visual.merger.0.w"], W["visual.merger.0.b"] = z(mh, mh), z(mh)
        W["visual.merger.2.w"], W["visual.merger.2.b"] = z(vc.out_hidden_size, mh), z(vc.out_hidden_size)
        d = tc.hidden_size
        thd = d // tc.num_attention_heads
        nq, nkv = tc.num_attention_heads * thd, tc.num_key_value_heads * thd
        W["model.embed_tokens"] = z(tc.vocab_size, d)
        for i in range(tc.num_hidden_layers):
            p = f"model.layers.{i}."
            W[p + "ln1"], W[p + "ln2"] = o(d), o(d)
            W[p + "qkv.w"], W[p + "qkv.b"] = z(nq + 2 * nkv, d), z(nq + 2 * nkv)
            W[p + "o.w"] = z(d, nq)
            W[p + "gu.w"] = z(2 * tc.intermediate_size, d)
            W[p + "down.w"] = z(d, tc.intermediate_size)
        W["model.norm"] = o(d)
        W["lm_head"] = z(tc.vocab_size, d)                    # text-reply branch (generate)
        return W

    @property
    def dtype(self):
        return torch.bfloat16

    @property
    def device(self):
        return self._dev

    def storage(self):
        return list(self.W.values())

    # ------------------------------------------------------------------ weights (HF names <-> kernel layout)
    @torch.no_grad()
    def load_state_dict(self, sd, strict: bool = True, assign: bool = False):
        tc, vc, W, HP, hd = self.tc, self.vc, self.W, self.HP, self.vhd
        g = lambda k: sd[k].to(self._dev, torch.bfloat16)
        W["visual.patch_embed"].copy_(g("visual.patch_embed.proj.weight").reshape(vc.hidden_size, -1))
        nh = vc.num_heads
        for i in range(vc.depth):
            p, s = f"visual.blocks.{i}.", f"visual.blocks.{i}."
            W[p + "norm1"].copy_(g(s + "norm1.weight"))
            W[p + "norm2"].copy_(g(s + "norm2.weight"))
            qw = g(s + "attn.qkv.weight").view(3, nh, hd, vc.hidden_size)
            W[p + "qkv.w"].view(3, nh, HP, vc.hidden_size)[:, :, :hd].copy_(qw)
            W[p + "qkv.b"].view(3, nh, HP)[:, :, :hd].copy_(g(s + "attn.qkv.bias").view(3, nh, hd))
            W[p + "proj.w"].view(vc.hidden_size, nh, HP)[:, :, :hd].copy_(g(s + "attn.proj.weight").view(vc.hidden_size, nh, hd))
            W[p + "proj.b"].copy_(g(s + "attn.proj.bias"))
            I, Ip = vc.intermediate_size, self.vi
            W[p + "gu.w"][:I].copy_(g(s + "mlp.gate_proj.weight"))
            W[p + "gu.w"][Ip:Ip + I].copy_(g(s + "mlp.up_proj.weight"))
            W[p + "gu.b"][:I].copy_(g(s + "mlp.gate_proj.bias"))
            W[p + "gu.b"][Ip:Ip + I].copy_(g(s + "mlp.up_proj.bias"))
            W[p + "down.w"][:, :I].copy_(g(s + "mlp.down_proj.weight"))
            W[p + "down.b"].copy_(g(s + "mlp.down_proj.bias"))
        W["visual.merger.ln_q"].copy_(g("visual.merger.ln_q.weight"))
        for j in ("0", "2"):
            W[f"visual.merger.{j}.w"].copy_(g(f"visual.merger.mlp.{j}.weight"))
            W[f"visual.merger.{j}.b"].copy_(g(f"visual.merger.mlp.{j}.bias"))
        W["model.embed_tokens"].copy_(g("model.embed_tokens.weight"))
        nq = tc.num_attention_heads * self.thd
        nkv = tc.num_key_value_heads * self.thd
        for i in range(tc.num_hidden_layers):
            p = s = f"model.layers.{i}."
            W[p + "ln1"].copy_(g(s + "input_layernorm.weight"))
            W[p + "ln2"].copy_(g(s + "post_attention_layernorm.weight"))
            for name, lo, n in (("q_proj", 0, nq), ("k_proj", nq, nkv), ("v_proj", nq + nkv, nkv)):
                W[p + "qkv.w"][lo:lo + n].copy_(g(s + f"self_attn.{name}.weight"))
                W[p + "qkv.b"][lo:lo + n].copy_(g(s + f"self_attn.{name}.bias"))
            W[p + "o.w"].copy_(g(s + "self_attn.o_proj.weight"))
            I = tc.intermediate_size
            W[p + "gu.w"][:I].copy_(g(s + "mlp.gate_proj.weight"))
            W[p + "gu.w"][I:].copy_(g(s + "mlp.up_proj.weight"))
            W[p + "down.w"].copy_(g(s + "mlp.down_proj.weight"))
        W["model.norm"].copy_(g("model.norm.weight"))
        missing = []
        if "lm_head.weight" in sd:
            W["lm_head"].copy_(g("lm_head.weight"))
        else:
            missing.append("lm_head.weight")                 # only the text-reply branch needs it
        return SimpleNamespace(missing_keys=missing, unexpected_keys=[])

    def state_dict(self, *a, **k):
        """transformers-4.50 key names <- kernel layout: the inverse of `load_state_dict` (fused tensors split, padding slots
        dropped), so `save_pretrained` writes what `from_pretrained` — here and in the reference — reads."""
        tc, vc, W, HP, hd = self.tc, self.vc, self.W, self.HP, self.vhd
        sd = OrderedDict()
        sd["visual.patch_embed.proj.weight"] = W["visual.patch_embed"].reshape(vc.hidden_size, vc.in_channels, vc.temporal_patch_size,
                                                                               vc.patch_size, vc.patch_size)
        nh, H = vc.num_heads, vc.hidden_size
        I, Ip = vc.intermediate_size, self.vi
        for i in range(vc.depth):
            p = f"visual.blocks.{i}."
            sd[p + "norm1.weight"], sd[p + "norm2.weight"] = W[p + "norm1"], W[p + "norm2"]
            sd[p + "attn.qkv.weight"] = W[p + "qkv.w"].view(3, nh, HP, H)[:, :, :hd].reshape(3 * nh * hd, H)
            sd[p + "attn.qkv.bias"] = W[p + "qkv.b"].view(3, nh, HP)[:, :, :hd].reshape(3 * nh * hd)
            sd[p + "attn.proj.weight"] = W[p + "proj.w"].view(H, nh, HP)[:, :, :hd].reshape(H, nh * hd)
            sd[p + "attn.proj.bias"] = W[p + "proj.b"]
            sd[p + "mlp.gate_proj.weight"], sd[p + "mlp.up_proj.weight"] = W[p + "gu.w"][:I], W[p + "gu.w"][Ip:Ip + I]
            sd[p + "mlp.gate_proj.bias"], sd[p + "mlp.up_proj.bias"] = W[p + "gu.b"][:I], W[p + "gu.b"][Ip:Ip + I]
            sd[p + "mlp.down_proj.weight"], sd[p + "mlp.down_proj.bias"] = W[p + "down.w"][:, :I], W[p + "down.b"]
        sd["visual.merger.ln_q.weight"] = W["visual.merger.ln_q"]
        for j in ("0", "2"):
            sd[f"visual.merger.mlp.{j}.weight"], sd[f"visual.merger.mlp.{j}.bias"] = W[f"visual.merger.{j}.w"], W[f"visual.merger.{j}.b"]
        sd["model.embed_tokens.weight"] = W["model.embed_tokens"]
        nq, nkv = tc.num_attention_heads * self.thd, tc.num_key_value_heads * self.thd
        It = tc.intermediate_size
        for i in range(tc.num_hidden_layers):
            p = f"model.layers.{i}."
            sd[p + "input_layernorm.weight"], sd[p + "post_attention_layernorm.weight"] = W[p + "ln1"], W[p + "ln2"]
            for name, lo, n in (("q_proj", 0, nq), ("k_proj", nq, nkv), ("v_proj", nq + nkv, nkv)):
                sd[p + f"self_attn.{name}.weight"], sd[p + f"self_attn.{name}.bias"] = W[p + "qkv.w"][lo:lo + n], W[p + "qkv.b"][lo:lo + n]
            sd[p + "self_attn.o_proj.weight"] = W[p + "o.w"]
            sd[p + "mlp.gate_proj.weight"], sd[p + "mlp.up_proj.weight"] = W[p + "gu.w"][:It], W[p + "gu.w"][It:]
            sd[p + "mlp.down_proj.weight"] = W[p + "down.w"]
        sd["model.norm.weight"] = W["model.norm"]
        sd["lm_head.weight"] = W["lm_head"]
        return sd

    @torch.no_grad()
    def randomize_(self, seed: int = 0, std: float = 0.02):
        """Synthetic weights directly in kernel layout (padded slots stay zero)."""
        g = torch.Generator(device=self._dev).manual_seed(seed)
        vc, HP, hd = self.vc, self.HP, self.vhd
        rnd = lambda t, s=std: t.copy_((torch.randn(t.shape, device=self._dev, generator=g) * s).to(torch.bfloat16))
        for k, t in self.W.items():
            if t.dim() == 1 and ("norm" in k or "ln" in k):
                t.fill_(1.0)
            elif k.endswith("qkv.w") and k.startswith("visual"):
                rnd(t.view(3, vc.num_heads, HP, -1)[:, :, :hd])
            elif k.endswith("qkv.b") and k.startswith("visual"):
                rnd(t.view(3, vc.num_heads, HP)[:, :, :hd])
            elif k.endswith("proj.w") and k.startswith("visual"):
                rnd(t.view(vc.hidden_size, vc.num_heads, HP)[:, :, :hd])
            elif k.endswith("gu.w") and k.startswith("visual"):
                rnd(t[: vc.intermediate_size]); rnd(t[self.vi: self.vi + vc.intermediate_size])
            elif k.endswith("gu.b") and k.startswith("visual"):
                rnd(t[: vc.intermediate_size]); rnd(t[self.vi: self.vi + vc.intermediate_size])
            elif k.endswith("down.w") and k.startswith("visual"):
                rnd(t[:, : vc.intermediate_size])
            else:
                step = 1 << 26
                flat = t.view(-1)
                for o_ in range(0, flat.numel(), step):
                    n = min(step, flat.numel() - o_)
                    flat[o_:o_ + n] = (torch.randn(n, device=self._dev, generator=g) * std).to(torch.bfloat16)
        return self

    # ------------------------------------------------------------------ vision tower
    @torch.no_grad()
    def forward_visual(self, pixel_values: torch.Tensor, grid_thw) -> torch.Tensor:
        """pixel_values [T, C*2*14*14] (processor order), grid_thw [[t,h,w]] -> merged image embeds
        [T/4, out_hidden] in the original (un-windowed) token order."""
        vc, W, HP = self.vc, self.W, self.HP
        grid = [tuple(int(v) for v in g) for g in (grid_thw.tolist() if torch.is_tensor(grid_thw) else grid_thw)]
        T = pixel_values.shape[0]
        unit = vc.spatial_merge_size ** 2
        x = ops.linear(pixel_values.to(self._dev, torch.bfloat16).contiguous(), W["visual.patch_embed"])
        # 2-D rope table (fp32), reordered with the windows
        pos = vision_rot_pos_ids(grid, vc.spatial_merge_size)
        dim = self.vhd // 2
        inv = 1.0 / (10000.0 ** (torch.arange(0, dim, 2, dtype=torch.float) / dim))
        freqs = torch.outer(torch.arange(max(max(g[1], g[2]) for g in grid), dtype=torch.float), inv)
        rope = freqs[pos].flatten(1)                                          # [T, 40]
        widx, cu_win = vision_window_index(grid, window_size=vc.window_size, spatial_merge_size=vc.spatial_merge_size,
                                           patch_size=vc.patch_size)
        rope = rope.reshape(T // unit, unit, -1)[widx].reshape(T, -1)
        emb = torch.cat((rope, rope), dim=-1)
        cos, sin = emb.cos().to(self._dev).contiguous(), emb.sin().to(self._dev).contiguous()
        widx_d = widx.to(self._dev)
        x = ops.gather_rows(x.view(T // unit, unit * vc.hidden_size), widx_d).view(T, vc.hidden_size)
        cu_full = [0]
        for t, h, w in grid:
            for _ in range(t):
                cu_full.append(cu_full[-1] + h * w)
        nh = vc.num_heads
        HPv = nh * HP
        scale = self.vhd ** -0.5
        attn_out = torch.empty((T, HPv), device=self._dev, dtype=torch.bfloat16)
        for i in range(vc.depth):
            p = f"visual.blocks.{i}."
            xn = ops.rmsnorm(x, W[p + "norm1"])
            qkv = ops.linear(xn, W[p + "qkv.w"], W[p + "qkv.b"])
            ops.rope_half_(qkv, 2 * nh, HP, cos, sin, fp32_math=True)         # q heads then k heads
            cu = cu_full if i in vc.fullatt_block_indexes else cu_win
            self._segment_attention(qkv, attn_out, cu, nh, nh, HPv, HPv, scale, causal=False)
            ops.linear(attn_out, W[p + "proj.w"], W[p + "proj.b"], epilogue=ops.EPI_RESID, resid=x, out=x)
            xn = ops.rmsnorm(x, W[p + "norm2"])
            gu = ops.linear(xn, W[p + "gu.w"], W[p + "gu.b"])
            a = ops.swiglu(gu, self.vi)
            ops.linear(a, W[p + "down.w"], W[p + "down.b"], epilogue=ops.EPI_RESID, resid=x, out=x)
        xn = ops.rmsnorm(x, W["visual.merger.ln_q"]).view(T // unit, unit * vc.hidden_size)
        h = ops.linear(xn, W["visual.merger.0.w"], W["visual.merger.0.b"], epilogue=ops.EPI_GELU_ERF)
        merged = ops.linear(h, W["visual.merger.2.w"], W["visual.merger.2.b"])
        return ops.gather_rows(merged, torch.argsort(widx).to(self._dev))

    def _segment_attention(self, qkv, out, cu, H, Hkv, k_off, v_off_rel, scale, causal):
        """Block-diagonal attention over contiguous token segments cu[i]:cu[i+1]; runs of equal-length
        segments go out as ONE batched launch (windows of a 448x448 image: 16 x 64 tokens)."""
        HP = self.HP
        i = 0
        n = len(cu) - 1
        while i < n:
            L = cu[i + 1] - cu[i]
            j = i + 1
            while j < n and cu[j + 1] - cu[j] == L:
                j += 1
            rows = qkv[cu[i]:cu[j]]
            Bn = j - i
            q = rows[:, : H * HP].unflatten(1, (H, HP)).unflatten(0, (Bn, L))
            k = rows[:, k_off: k_off + Hkv * HP].unflatten(1, (Hkv, HP)).unflatten(0, (Bn, L))
            v = rows[:, k_off + v_off_rel: k_off + v_off_rel + Hkv * HP].unflatten(1, (Hkv, HP)).unflatten(0, (Bn, L))
            ops.attention(q, k, v, out=out[cu[i]:cu[j]].unflatten(0, (Bn, L)), causal=causal, scale=scale)
            i = j

    # ------------------------------------------------------------------ decoder prefill
    @torch.no_grad()
    def _rope_tables(self, pos):
        """M-RoPE cos/sin for position ids [3, B, L]: fp32 angles, values rounded to bf16 (transformers casts the
        tables to the model dtype), flattened to [B*L, head_dim] fp32 on the device."""
        tc, hd = self.tc, self.thd
        inv = 1.0 / (tc.rope_theta ** (torch.arange(0, hd, 2, dtype=torch.int64).float() / hd))
        freqs = pos.cpu()[:, :, :, None].float() * inv[None, None, None, :]           # [3,B,L,hd/2]
        emb = torch.cat((freqs, freqs), dim=-1)
        sec = list(tc.mrope_section) * 2
        pick = lambda t: torch.cat([m[i % 3] for i, m in enumerate(t.split(sec, dim=-1))], dim=-1)
        n = pos.shape[1] * pos.shape[2]
        cos = pick(emb.cos()).bfloat16().float().reshape(n, hd).to(self._dev).contiguous()
        sin = pick(emb.sin()).bfloat16().float().reshape(n, hd).to(self._dev).contiguous()
        return cos, sin

    def _decoder(self, x, cos, sin, B, L, kv_cache=None, past: int = 0, spans=None):
        """The 28 decoder layers + final norm on x [B*L, hidden] (updated in place).  With `kv_cache`
        ([layers, 2, B, Lmax, Hkv, head_dim]) the post-RoPE K and V of these L tokens are stored at
        [past, past+L) and attention runs over the cached prefix as well (L == 1: decode step).
        `spans` [(lo, hi)] * B marks the real tokens of a padded batch: attention then runs per sequence over its
        own tokens only and the padding rows get a zero attention output — what transformers' flash_attention_2
        path does (unpad -> varlen attention -> pad_input), the backend the reference selects (cli.py:40,
        train_denoiser.py:1633)."""
        tc, W, hd = self.tc, self.W, self.thd
        nq, nkv = tc.num_attention_heads, tc.num_key_value_heads
        # padded prefill: the rows no launch writes must read as zeros in every layer
        o = (torch.zeros if (spans is not None and not past) else torch.empty)((B * L, nq * hd), device=self._dev, dtype=torch.bfloat16)
        if past and L != 1:
            raise _lib.B2FError("chunked prefill is not implemented: use past == 0 (prefill) or one new token (decode)")
        for i in range(tc.num_hidden_layers):
            p = f"model.layers.{i}."
            xn = ops.rmsnorm(x, W[p + "ln1"], eps=tc.rms_norm_eps)
            qkv = ops.linear(xn, W[p + "qkv.w"], W[p + "qkv.b"])
            ops.rope_half_(qkv, nq + nkv, hd, cos, sin, fp32_math=False)
            q = qkv[:, : nq * hd].unflatten(1, (nq, hd)).unflatten(0, (B, L))
            k = qkv[:, nq * hd: (nq + nkv) * hd].unflatten(1, (nkv, hd)).unflatten(0, (B, L))
            v = qkv[:, (nq + nkv) * hd:].unflatten(1, (nkv, hd)).unflatten(0, (B, L))
            if kv_cache is not None:
                kv_cache[i, 0, :, past:past + L].copy_(k)
                kv_cache[i, 1, :, past:past + L].copy_(v)
            if past:
                # decode: the new token attends to every cached position of its own sequence (no mask needed: a left-padded
                # prompt's padding slots lie before `lo`); one launch per sequence because the cache's batch pitch (Lmax
                # rows) differs from the attended length
                for b in range(B):
                    lo = spans[b][0] if spans is not None else 0
                    ops.attention(q[b:b + 1], kv_cache[i, 0, b:b + 1, lo:past + 1], kv_cache[i, 1, b:b + 1, lo:past + 1],
                                  out=o.unflatten(0, (B, L))[b:b + 1])
            elif spans is not None:                      # padded prefill
                o3 = o.unflatten(0, (B, L))
                for b, (lo, hi) in enumerate(spans):
                    ops.attention(q[b:b + 1, lo:hi], k[b:b + 1, lo:hi], v[b:b + 1, lo:hi], out=o3[b:b + 1, lo:hi], causal=True)
            else:
                ops.attention(q, k, v, out=o.unflatten(0, (B, L)), causal=True)
            ops.linear(o, W[p + "o.w"], None, epilogue=ops.EPI_RESID, resid=x, out=x)
            xn = ops.rmsnorm(x, W[p + "ln2"], eps=tc.rms_norm_eps)
            gu = ops.linear(xn, W[p + "gu.w"])
            a = ops.swiglu(gu, tc.intermediate_size)
            ops.linear(a, W[p + "down.w"], None, epilogue=ops.EPI_RESID, resid=x, out=x)
        return ops.rmsnorm(x, W["model.norm"], eps=tc.rms_norm_eps)

    def lm_logits(self, hidden):
        """lm_head on [n, hidden] -> [n, vocab] bf16 (wgmma GEMM; vocab rows stream once from HBM)."""
        return ops.linear(hidden.reshape(-1, self.tc.hidden_size), self.W["lm_head"])

    @torch.no_grad()
    def generate(self, input_ids: torch.Tensor, pixel_values=None, attention_mask=None, image_grid_thw=None,
                 max_new_tokens: int = 128, eos_token_id=(151645, 151643), pad_token_id: int = 151643,
                 repetition_penalty: float = 1.0, forced_tokens=None, output_scores: bool = False, **kw):
        """Greedy text reply with a KV cache (the `model.generate(**inputs, max_new_tokens=128)` call of the
        reference's understanding branch, univa/serve/cli.py:256-267): prefill through the same kernels as
        the conditioning path, then one token per step — M = B GEMMs (weight-streaming, HBM-bound), single-query
        attention over the cache, lm_head, argmax.  Returns ids [B, L + new] (prompt included, as transformers
        does); with `output_scores` also the per-step fp32 logits.  `forced_tokens` [B, T] replaces the argmax
        (teacher forcing for tests).  Sampling is not implemented: Qwen2.5-VL's generation_config asks for
        temperature 1e-6, i.e. greedy up to ties; `repetition_penalty` follows transformers' processor."""
        tc = self.tc
        B, L = input_ids.shape
        ids = input_ids.to(self._dev)
        steps = int(forced_tokens.shape[1]) if forced_tokens is not None else int(max_new_tokens)
        cache = torch.empty((tc.num_hidden_layers, 2, B, L + steps, tc.num_key_value_heads, self.thd), device=self._dev,
                            dtype=torch.bfloat16)
        hidden, deltas, spans = self.forward(ids, pixel_values=pixel_values, attention_mask=attention_mask,
                                             image_grid_thw=image_grid_thw, kv_cache=cache, return_rope_deltas=True)
        last = hidden[:, -1]                                            # [B, hidden]
        eos = torch.tensor(list(eos_token_id) if not isinstance(eos_token_id, int) else [eos_token_id], device=self._dev)
        out = [ids]
        scores = []
        done = torch.zeros(B, dtype=torch.bool, device=self._dev)
        seen = ids.clone()
        for t in range(steps):
            logits = self.lm_logits(last).float()                         # [B, vocab]
            if repetition_penalty != 1.0:
                g = logits.gather(1, seen)
                logits.scatter_(1, seen, torch.where(g < 0, g * repetition_penalty, g / repetition_penalty))
            if output_scores:
                scores.append(logits)
            nxt = logits.argmax(dim=-1) if forced_tokens is None else forced_tokens[:, t].to(self._dev)
            nxt = torch.where(done, torch.full_like(nxt, pad_token_id), nxt)
            out.append(nxt[:, None])
            seen = torch.cat([seen, nxt[:, None]], dim=1)
            done = done | torch.isin(nxt, eos)
            if forced_tokens is None and bool(done.all()):
                break
            if t == steps - 1:
                break
            # text continues on all three M-RoPE axes at (past length + delta)
            pos = (torch.full((B, 1), L + t, dtype=torch.long) + deltas.cpu().view(B, 1))[None].expand(3, B, 1)
            cos, sin = self._rope_tables(pos)
            x = ops.gather_rows(self.W["model.embed_tokens"], nxt.contiguous())
            last = self._decoder(x, cos, sin, B, 1, cache, past=L + t, spans=spans)
        seq = torch.cat(out, dim=1)
        return (seq, scores) if output_scores else seq

    @torch.no_grad()
    def forward(self, input_ids: torch.Tensor, pixel_values=None, attention_mask=None, image_grid_thw=None,
                return_image_embeds: bool = False, kv_cache=None, return_rope_deltas: bool = False):
        """-> last hidden state after model.norm, [B, L, hidden] (what the reference feeds to MLP2)."""
        tc, W = self.tc, self.W
        B, L = input_ids.shape
        spans = None
        if attention_mask is not None and not bool((attention_mask == 1).all()):
            spans = padding_spans(attention_mask)
            if kv_cache is not None and any(hi != L for _, hi in spans):
                raise _lib.B2FError("generate() takes left-padded prompt batches (every prompt ends at the last column, as the "
                                    "processor pads for generation); this batch is padded on the right")
        ids = input_ids.to(self._dev)
        x = ops.gather_rows(W["model.embed_tokens"], ids.reshape(-1).contiguous())
        image_embeds = None
        if pixel_values is not None:
            image_embeds = self.forward_visual(pixel_values, image_grid_thw)
            where = (ids.reshape(-1) == tc.image_token_id).nonzero().squeeze(1).contiguous()
            if where.numel() != image_embeds.shape[0]:
                raise ValueError(f"Image features and image tokens do not match: tokens: {where.numel()}, "
                                 f"features {image_embeds.shape[0]}")
            ops.scatter_rows_(x, where, image_embeds)
        pos, deltas = get_rope_index(ids, image_grid_thw if pixel_values is not None else None, attention_mask,
                                spatial_merge_size=self.vc.spatial_merge_size, image_token_id=tc.image_token_id,
                                vision_start_token_id=tc.vision_start_token_id)
        cos, sin = self._rope_tables(pos)
        h = self._decoder(x, cos, sin, B, L, kv_cache, spans=spans).view(B, L, tc.hidden_size)
        if return_rope_deltas:
            return h, deltas, spans
        return (h, image_embeds) if return_image_embeds else h
