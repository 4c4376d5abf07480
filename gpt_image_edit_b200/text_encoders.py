"""T5-XXL encoder and CLIP-L text encoder on libb2f kernels (SURVEY.md §8 row a11).

Replaces `pipe.text_encoder_2` (transformers `T5EncoderModel`) and `pipe.text_encoder`
(`CLIPTextModel`) as the reference drives them from `encode_prompt`
(univa/utils/denoiser_prompt_embedding_flux.py:44 `text_encoder(text_input_ids)[0]`, :91-98
`text_encoder(ids, output_hidden_states=False).pooler_output`; called from univa/serve/cli.py:221):

  T5 v1.1 encoder   pre-RMSNorm blocks; q/k/v/o without bias, NO 1/sqrt(d) score scale, additive
                    bucketed relative-position bias shared by all layers (block 0 owns the table),
                    NO padding mask (the reference passes ids only); FF = wo(gelu_new(wi_0 x) * wi_1 x)
  CLIP text         token + learned position embeddings; pre-LayerNorm blocks with biases, causal
                    attention scaled by d_h^-0.5, quick-GELU MLP; final LayerNorm; pooled = the
                    hidden state at argmax(input_ids) (config eos_token_id == 2 legacy rule, which
                    is what FLUX.1's text_encoder/config.json carries)

Every matmul is the wgmma GEMM (`b2f_gemm_bf16`, residual adds and quick-GELU fused into the
epilogue), attention is the FA-style wgmma kernel with head_dim 64 zero-padded to the 128-wide
head slot in the WEIGHT layout (so no activation is ever re-laid out) — `b2f_attention_bias_fwd`
for T5, causal `b2f_attention_fwd` for CLIP; norms / gated-GELU / embeddings are the HBM-bound
kernels in csrc/llm_kernels.cu.  There is no CPU path.
"""
from __future__ import annotations

import math
from collections import OrderedDict
from types import SimpleNamespace

import torch

from . import _lib, ops

HP = 128  # head slot pitch of the attention kernel


class T5EncoderConfig(SimpleNamespace):
    """google/t5-v1_1-xxl encoder (FLUX.1 `text_encoder_2/config.json`)."""

    def __init__(self, **kw):
        d = dict(vocab_size=32128, d_model=4096, d_kv=64, num_heads=64, d_ff=10240, num_layers=24,
                 relative_attention_num_buckets=32, relative_attention_max_distance=128, layer_norm_epsilon=1e-6)
        d.update(kw)
        super().__init__(**d)


class CLIPTextConfig(SimpleNamespace):
    """openai/clip-vit-large-patch14 text tower (FLUX.1 `text_encoder/config.json`)."""

    def __init__(self, **kw):
        d = dict(vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=12, num_attention_heads=12,
                 max_position_embeddings=77, layer_norm_eps=1e-5, eos_token_id=2)
        d.update(kw)
        super().__init__(**d)


class EncoderOutput:
    """Minimal stand-in for transformers' ModelOutput: `out[0]`, `.last_hidden_state`, `.pooler_output`."""

    def __init__(self, last_hidden_state, pooler_output=None):
        self.last_hidden_state = last_hidden_state
        self.pooler_output = pooler_output

    def __getitem__(self, i):
        return (self.last_hidden_state, self.pooler_output)[i] if self.pooler_output is not None else \
            (self.last_hidden_state,)[i]


def t5_relative_position_bucket(L: int, num_buckets: int = 32, max_distance: int = 128) -> torch.Tensor:
    """Bidirectional T5 bucket index of (memory - query) for an L x L grid, int64 [L, L]
    (transformers T5Attention._relative_position_bucket; integer work, bit-exact)."""
    ctx = torch.arange(L, dtype=torch.long)[:, None]
    mem = torch.arange(L, dtype=torch.long)[None, :]
    rel = mem - ctx
    nb = num_buckets // 2
    buckets = (rel > 0).to(torch.long) * nb
    rel = rel.abs()
    max_exact = nb // 2
    is_small = rel < max_exact
    large = max_exact + (torch.log(rel.float() / max_exact) / math.log(max_distance / max_exact) * (nb - max_exact)).to(torch.long)
    large = torch.min(large, torch.full_like(large, nb - 1))
    return buckets + torch.where(is_small, rel, large)


def _randn_into(t, g, std):
    step = 1 << 26
    flat = t.view(-1)
    for o in range(0, flat.numel(), step):
        n = min(step, flat.numel() - o)
        flat[o:o + n] = (torch.randn(n, device=t.device, generator=g) * std).to(torch.bfloat16)


class _Base(torch.nn.Module):
    def __init__(self, device):
        super().__init__()
        dev = torch.device(device)
        if dev.type != "cuda":
            raise _lib.B2FError(f"{type(self).__name__} lives on a CUDA device; there is no CPU path")
        self._dev = dev
        self.W = OrderedDict()

    def _register(self):
        for k, t in self.W.items():
            self.register_buffer("w__" + k.replace(".", "__"), t, persistent=False)

    @property
    def dtype(self):
        return torch.bfloat16

    @property
    def device(self):
        return self._dev

    def storage(self):
        return list(self.W.values())


# ------------------------------------------------------------------------------------------------ T5
class B200T5Encoder(_Base):
    def __init__(self, config: T5EncoderConfig | None = None, device="cuda"):
        super().__init__(device)
        c = self.config = config or T5EncoderConfig()
        if c.d_kv > HP or c.d_model % 256:
            raise _lib.B2FError("T5 config outside the kernel envelope (d_kv <= 128, d_model % 256 == 0)")
        dev, d, H = self._dev, c.d_model, c.num_heads
        z = lambda *s: torch.zeros(s, device=dev, dtype=torch.bfloat16)
        o = lambda *s: torch.ones(s, device=dev, dtype=torch.bfloat16)
        W = self.W
        W["shared"] = z(c.vocab_size, d)
        W["rel_bias"] = z(c.relative_attention_num_buckets, H)
        for i in range(c.num_layers):
            p = f"block.{i}."
            W[p + "ln1"], W[p + "ln2"] = o(d), o(d)
            W[p + "qkv.w"] = z(3 * H * HP, d)            # heads in 128-wide slots, rows [d_kv, 128) zero
            W[p + "o.w"] = z(d, H * HP)
            W[p + "wi.w"] = z(2 * c.d_ff, d)             # [wi_0 ; wi_1]
            W[p + "wo.w"] = z(d, c.d_ff)
        W["final_ln"] = o(d)
        self._register()
        self._bias_cache: dict[int, torch.Tensor] = {}

    @torch.no_grad()
    def load_state_dict(self, sd, strict: bool = True, assign: bool = False):
        """transformers T5EncoderModel names -> kernel layout."""
        c, W = self.config, self.W
        H, dk, d = c.num_heads, c.d_kv, c.d_model
        g = lambda k: sd[k].to(self._dev, torch.bfloat16)
        W["shared"].copy_(g("shared.weight") if "shared.weight" in sd else g("encoder.embed_tokens.weight"))
        W["rel_bias"].copy_(g("encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"))
        for i in range(c.num_layers):
            p, s = f"block.{i}.", f"encoder.block.{i}.layer."
            W[p + "ln1"].copy_(g(s + "0.layer_norm.weight"))
            W[p + "ln2"].copy_(g(s + "1.layer_norm.weight"))
            qkv = W[p + "qkv.w"].view(3, H, HP, d)
            for j, n in enumerate("qkv"):
                qkv[j, :, :dk].copy_(g(s + f"0.SelfAttention.{n}.weight").view(H, dk, d))
            W[p + "o.w"].view(d, H, HP)[:, :, :dk].copy_(g(s + "0.SelfAttention.o.weight").view(d, H, dk))
            W[p + "wi.w"][: c.d_ff].copy_(g(s + "1.DenseReluDense.wi_0.weight"))
            W[p + "wi.w"][c.d_ff:].copy_(g(s + "1.DenseReluDense.wi_1.weight"))
            W[p + "wo.w"].copy_(g(s + "1.DenseReluDense.wo.weight"))
        W["final_ln"].copy_(g("encoder.final_layer_norm.weight"))
        self._bias_cache.clear()
        return SimpleNamespace(missing_keys=[], unexpected_keys=[])

    @torch.no_grad()
    def state_dict(self, *a, **kw):
        """Kernel layout -> transformers names (padding stripped)."""
        c, W = self.config, self.W
        H, dk, d = c.num_heads, c.d_kv, c.d_model
        sd = OrderedDict()
        sd["shared.weight"] = W["shared"]
        sd["encoder.embed_tokens.weight"] = W["shared"]
        sd["encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"] = W["rel_bias"]
        for i in range(c.num_layers):
            p, s = f"block.{i}.", f"encoder.block.{i}.layer."
            qkv = W[p + "qkv.w"].view(3, H, HP, d)
            for j, n in enumerate("qkv"):
                sd[s + f"0.SelfAttention.{n}.weight"] = qkv[j, :, :dk].reshape(H * dk, d)
            sd[s + "0.SelfAttention.o.weight"] = W[p + "o.w"].view(d, H, HP)[:, :, :dk].reshape(d, H * dk)
            sd[s + "0.layer_norm.weight"] = W[p + "ln1"]
            sd[s + "1.DenseReluDense.wi_0.weight"] = W[p + "wi.w"][: c.d_ff]
            sd[s + "1.DenseReluDense.wi_1.weight"] = W[p + "wi.w"][c.d_ff:]
            sd[s + "1.DenseReluDense.wo.weight"] = W[p + "wo.w"]
            sd[s + "1.layer_norm.weight"] = W[p + "ln2"]
        sd["encoder.final_layer_norm.weight"] = W["final_ln"]
        return sd

    @torch.no_grad()
    def randomize_(self, seed: int = 0, std: float = 0.02):
        """Synthetic weights directly in kernel layout (padded slots stay zero)."""
        c = self.config
        g = torch.Generator(device=self._dev).manual_seed(seed)
        for k, t in self.W.items():
            if t.dim() == 1:
                t.fill_(1.0)
            elif k.endswith("qkv.w"):
                v = t.view(3, c.num_heads, HP, c.d_model)
                v[:, :, : c.d_kv] = (torch.randn(3, c.num_heads, c.d_kv, c.d_model, device=self._dev, generator=g) * std).to(torch.bfloat16)
            elif k.endswith(".o.w"):
                v = t.view(c.d_model, c.num_heads, HP)
                v[:, :, : c.d_kv] = (torch.randn(c.d_model, c.num_heads, c.d_kv, device=self._dev, generator=g) * std).to(torch.bfloat16)
            elif k == "rel_bias":
                _randn_into(t, g, 0.5)
            else:
                _randn_into(t, g, std)
        self._bias_cache.clear()
        return self

    def position_bias(self, L: int) -> torch.Tensor:
        """[H, L, L] bf16: rel_bias[bucket(mem - ctx)] (T5Attention.compute_bias), cached per length."""
        b = self._bias_cache.get(L)
        if b is None:
            c = self.config
            idx = t5_relative_position_bucket(L, c.relative_attention_num_buckets, c.relative_attention_max_distance)
            # one-time table build per sequence length (like the RoPE tables), not on the per-call path
            b = self.W["rel_bias"][idx.to(self._dev)].permute(2, 0, 1).contiguous()
            self._bias_cache[L] = b
        return b

    @torch.no_grad()
    def forward(self, input_ids: torch.Tensor, attention_mask=None, **kw) -> EncoderOutput:
        if attention_mask is not None and not bool(attention_mask.all()):
            raise _lib.B2FError("T5 padding masks are not implemented (the reference never passes one: "
                                "denoiser_prompt_embedding_flux.py:44)")
        c, W = self.config, self.W
        B, L = input_ids.shape
        H, d = c.num_heads, c.d_model
        ids = input_ids.to(self._dev, torch.int64).reshape(-1).contiguous()
        x = ops.embed(W["shared"], ids)                                     # [B*L, d]
        bias = self.position_bias(L)
        attn = torch.empty((B, L, H * HP), device=self._dev, dtype=torch.bfloat16)
        for i in range(c.num_layers):
            p = f"block.{i}."
            xn = ops.rmsnorm(x, W[p + "ln1"], eps=c.layer_norm_epsilon)
            qkv = ops.linear(xn, W[p + "qkv.w"]).view(B, L, 3, H, HP)
            ops.attention(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], out=attn, scale=1.0, bias=bias)
            x = ops.linear(attn.view(B * L, H * HP), W[p + "o.w"], epilogue=ops.EPI_RESID, resid=x)
            xn = ops.rmsnorm(x, W[p + "ln2"], eps=c.layer_norm_epsilon)
            h = ops.geglu(ops.linear(xn, W[p + "wi.w"]), c.d_ff)
            x = ops.linear(h, W[p + "wo.w"], epilogue=ops.EPI_RESID, resid=x)
        out = ops.rmsnorm(x, W["final_ln"], eps=c.layer_norm_epsilon)
        return EncoderOutput(out.view(B, L, d))


# ------------------------------------------------------------------------------------------------ CLIP
class B200CLIPTextModel(_Base):
    def __init__(self, config: CLIPTextConfig | None = None, device="cuda"):
        super().__init__(device)
        c = self.config = config or CLIPTextConfig()
        d, H = c.hidden_size, c.num_attention_heads
        self.hd = d // H
        if self.hd > HP or d % 256:
            raise _lib.B2FError("CLIP config outside the kernel envelope (head_dim <= 128, hidden_size % 256 == 0)")
        dev = self._dev
        z = lambda *s: torch.zeros(s, device=dev, dtype=torch.bfloat16)
        o = lambda *s: torch.ones(s, device=dev, dtype=torch.bfloat16)
        W = self.W
        W["tok"], W["pos"] = z(c.vocab_size, d), z(c.max_position_embeddings, d)
        for i in range(c.num_hidden_layers):
            p = f"layers.{i}."
            W[p + "ln1.w"], W[p + "ln1.b"], W[p + "ln2.w"], W[p + "ln2.b"] = o(d), z(d), o(d), z(d)
            W[p + "qkv.w"], W[p + "qkv.b"] = z(3 * H * HP, d), z(3 * H * HP)
            W[p + "o.w"], W[p + "o.b"] = z(d, H * HP), z(d)
            W[p + "fc1.w"], W[p + "fc1.b"] = z(c.intermediate_size, d), z(c.intermediate_size)
            W[p + "fc2.w"], W[p + "fc2.b"] = z(d, c.intermediate_size), z(d)
        W["final.w"], W["final.b"] = o(d), z(d)
        self._register()

    _PAIRS = (("ln1", "layer_norm1"), ("ln2", "layer_norm2"), ("fc1", "mlp.fc1"), ("fc2", "mlp.fc2"))

    @torch.no_grad()
    def load_state_dict(self, sd, strict: bool = True, assign: bool = False):
        c, W, hd = self.config, self.W, self.hd
        d, H = c.hidden_size, c.num_attention_heads
        g = lambda k: sd[k].to(self._dev, torch.bfloat16)
        W["tok"].copy_(g("text_model.embeddings.token_embedding.weight"))
        W["pos"].copy_(g("text_model.embeddings.position_embedding.weight"))
        for i in range(c.num_hidden_layers):
            p, s = f"layers.{i}.", f"text_model.encoder.layers.{i}."
            for mine, theirs in self._PAIRS:
                W[p + mine + ".w"].copy_(g(s + theirs + ".weight"))
                W[p + mine + ".b"].copy_(g(s + theirs + ".bias"))
            qw, qb = W[p + "qkv.w"].view(3, H, HP, d), W[p + "qkv.b"].view(3, H, HP)
            for j, n in enumerate(("q_proj", "k_proj", "v_proj")):
                qw[j, :, :hd].copy_(g(s + f"self_attn.{n}.weight").view(H, hd, d))
                qb[j, :, :hd].copy_(g(s + f"self_attn.{n}.bias").view(H, hd))
            W[p + "o.w"].view(d, H, HP)[:, :, :hd].copy_(g(s + "self_attn.out_proj.weight").view(d, H, hd))
            W[p + "o.b"].copy_(g(s + "self_attn.out_proj.bias"))
        W["final.w"].copy_(g("text_model.final_layer_norm.weight"))
        W["final.b"].copy_(g("text_model.final_layer_norm.bias"))
        return SimpleNamespace(missing_keys=[], unexpected_keys=[])

    @torch.no_grad()
    def state_dict(self, *a, **kw):
        c, W, hd = self.config, self.W, self.hd
        d, H = c.hidden_size, c.num_attention_heads
        sd = OrderedDict()
        sd["text_model.embeddings.token_embedding.weight"] = W["tok"]
        sd["text_model.embeddings.position_embedding.weight"] = W["pos"]
        for i in range(c.num_hidden_layers):
            p, s = f"layers.{i}.", f"text_model.encoder.layers.{i}."
            qw, qb = W[p + "qkv.w"].view(3, H, HP, d), W[p + "qkv.b"].view(3, H, HP)
            for j, n in enumerate(("q_proj", "k_proj", "v_proj")):
                sd[s + f"self_attn.{n}.weight"] = qw[j, :, :hd].reshape(H * hd, d)
                sd[s + f"self_attn.{n}.bias"] = qb[j, :, :hd].reshape(H * hd)
            sd[s + "self_attn.out_proj.weight"] = W[p + "o.w"].view(d, H, HP)[:, :, :hd].reshape(d, H * hd)
            sd[s + "self_attn.out_proj.bias"] = W[p + "o.b"]
            for mine, theirs in self._PAIRS:
                sd[s + theirs + ".weight"] = W[p + mine + ".w"]
                sd[s + theirs + ".bias"] = W[p + mine + ".b"]
        sd["text_model.final_layer_norm.weight"] = W["final.w"]
        sd["text_model.final_layer_norm.bias"] = W["final.b"]
        return sd

    @torch.no_grad()
    def randomize_(self, seed: int = 0, std: float = 0.02):
        c, hd = self.config, self.hd
        d, H = c.hidden_size, c.num_attention_heads
        g = torch.Generator(device=self._dev).manual_seed(seed)
        rnd = lambda shape, s=std: (torch.randn(shape, device=self._dev, generator=g) * s).to(torch.bfloat16)
        for k, t in self.W.items():
            if k.endswith("qkv.w"):
                t.view(3, H, HP, d)[:, :, :hd] = rnd((3, H, hd, d))
            elif k.endswith("qkv.b"):
                t.view(3, H, HP)[:, :, :hd] = rnd((3, H, hd))
            elif k.endswith(".o.w"):
                t.view(d, H, HP)[:, :, :hd] = rnd((d, H, hd))
            elif t.dim() == 1 and k.endswith(".w"):
                t.fill_(1.0)
            elif t.dim() == 1:
                t.copy_(rnd(t.shape))
            else:
                _randn_into(t, g, std)
        return self

    @torch.no_grad()
    def forward(self, input_ids: torch.Tensor, attention_mask=None, output_hidden_states: bool = False, **kw) -> EncoderOutput:
        if attention_mask is not None and not bool(attention_mask.all()):
            raise _lib.B2FError("CLIP padding masks are not implemented (the reference never passes one: "
                                "denoiser_prompt_embedding_flux.py:91)")
        c, W = self.config, self.W
        B, L = input_ids.shape
        if L > c.max_position_embeddings:
            raise ValueError(f"Sequence length must be less than max_position_embeddings (got {L} > {c.max_position_embeddings})")
        d, H = c.hidden_size, c.num_attention_heads
        ids2 = input_ids.to(self._dev, torch.int64)
        x = ops.embed(W["tok"], ids2.reshape(-1).contiguous(), W["pos"], period=L)
        attn = torch.empty((B, L, H * HP), device=self._dev, dtype=torch.bfloat16)
        scale = self.hd ** -0.5
        for i in range(c.num_hidden_layers):
            p = f"layers.{i}."
            xn = ops.layernorm(x, W[p + "ln1.w"], W[p + "ln1.b"], eps=c.layer_norm_eps)
            qkv = ops.linear(xn, W[p + "qkv.w"], W[p + "qkv.b"]).view(B, L, 3, H, HP)
            ops.attention(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], out=attn, scale=scale, causal=True)
            x = ops.linear(attn.view(B * L, H * HP), W[p + "o.w"], W[p + "o.b"], epilogue=ops.EPI_RESID, resid=x)
            xn = ops.layernorm(x, W[p + "ln2.w"], W[p + "ln2.b"], eps=c.layer_norm_eps)
            h = ops.linear(xn, W[p + "fc1.w"], W[p + "fc1.b"], epilogue=ops.EPI_QUICK_GELU)
            x = ops.linear(h, W[p + "fc2.w"], W[p + "fc2.b"], epilogue=ops.EPI_RESID, resid=x)
        last = ops.layernorm(x, W["final.w"], W["final.b"], eps=c.layer_norm_eps)
        # pooled = hidden state at the EOS token: argmax(ids) under the eos_token_id == 2 legacy rule,
        # else the first occurrence of eos_token_id (transformers CLIPTextTransformer.forward)
        if c.eos_token_id == 2:
            pos = ids2.argmax(dim=-1)
        else:
            pos = (ids2 == c.eos_token_id).to(torch.int32).argmax(dim=-1)
        rows = (torch.arange(B, device=self._dev) * L + pos).to(torch.int64)
        pooled = ops.gather_rows(last, rows)
        return EncoderOutput(last.view(B, L, d), pooled)


# ------------------------------------------------------------------------------------------------ encode_prompt
def tokenize_prompt(tokenizer, prompt, max_sequence_length):
    """ids [B, max_sequence_length], padded / truncated (reference denoiser_prompt_embedding_flux.py:1-12)."""
    return tokenizer(prompt, padding="max_length", max_length=max_sequence_length, truncation=True, return_length=False,
                     return_overflowing_tokens=False, return_tensors="pt").input_ids


def _ids_or_raise(tokenizer, prompt, max_len, text_input_ids):
    if tokenizer is not None:
        return tokenize_prompt(tokenizer, prompt, max_len)
    if text_input_ids is None:
        raise ValueError("text_input_ids must be provided when the tokenizer is not specified")
    return text_input_ids


def _tile(t, batch, n):
    """the reference's duplication: repeat along dim 1, then fold into the batch (copies of a prompt adjacent)."""
    if t.dim() == 2:                                   # pooled [B, d] -> [B, n*d] -> [B*n, d]
        return t.repeat(1, n).view(batch * n, -1)
    L = t.shape[1]                                     # hidden [B, L, d] -> [B, n*L, d] -> [B*n, L, d]
    return t.repeat(1, n, 1).view(batch * n, L, -1)


def _encode_prompt_with_t5(text_encoder, tokenizer, max_sequence_length=512, prompt=None, num_images_per_prompt=1,
                           device=None, text_input_ids=None):
    """[B*n, L, d] last hidden state of the T5 encoder (reference :15-58; ids only, no padding mask)."""
    prompt = [prompt] if isinstance(prompt, str) else prompt
    ids = _ids_or_raise(tokenizer, prompt, max_sequence_length, text_input_ids)
    enc = getattr(text_encoder, "module", text_encoder)
    embeds = text_encoder(ids.to(device))[0].to(dtype=enc.dtype, device=device)
    return _tile(embeds, len(prompt), num_images_per_prompt)


def _encode_prompt_with_clip(text_encoder, tokenizer, prompt, device=None, text_input_ids=None, num_images_per_prompt: int = 1):
    """[B*n, d] pooled CLIP output (reference :61-104; fixed 77-token window)."""
    prompt = [prompt] if isinstance(prompt, str) else prompt
    ids = _ids_or_raise(tokenizer, prompt, 77, text_input_ids)
    enc = getattr(text_encoder, "module", text_encoder)
    pooled = text_encoder(ids.to(device), output_hidden_states=False).pooler_output.to(dtype=enc.dtype, device=device)
    # The reference duplicates the 2-D pooled tensor with `repeat(1, n, 1)` (:100-101): torch treats it as [1, B, d], so
    # for B > 1 and n > 1 the copies come out INTERLEAVED (b0, b1, b0, b1, ...) while the T5 embeddings above are
    # grouped (b0, b0, ..., b1, ...).  Reproduced as is (pinned by tests/golden/host_ref.pt, generated by the
    # reference's own function); the pipeline's own encode_prompt (flux_pipeline.py:354-355) groups them.
    return pooled.repeat(1, num_images_per_prompt, 1).view(len(prompt) * num_images_per_prompt, -1)


def encode_prompt(text_encoders, tokenizers, prompt, max_sequence_length, device=None, num_images_per_prompt: int = 1,
                  text_input_ids_list=None):
    """Same contract as the reference's `encode_prompt` (univa/utils/denoiser_prompt_embedding_flux.py:107-144):
    `text_encoders = [clip, t5]`, `tokenizers = [clip_tok, t5_tok]`; an encoder runs only when BOTH it and its
    tokenizer are present (otherwise its output is None); returns (t5 prompt_embeds, clip pooled)."""
    prompt = [prompt] if isinstance(prompt, str) else prompt
    device = device if device is not None else text_encoders[1].device
    ids = text_input_ids_list or [None, None]
    pooled = embeds = None
    if text_encoders[0] is not None and tokenizers[0] is not None:
        pooled = _encode_prompt_with_clip(text_encoders[0], tokenizers[0], prompt, device=device, text_input_ids=ids[0],
                                          num_images_per_prompt=num_images_per_prompt)
    if text_encoders[1] is not None and tokenizers[1] is not None:
        embeds = _encode_prompt_with_t5(text_encoders[1], tokenizers[1], max_sequence_length, prompt,
                                        num_images_per_prompt, device, ids[1])
    return embeds, pooled


class SyntheticTokenizer:
    """Deterministic stand-in for the CLIP / T5 tokenizers when no vocabulary files exist (this image has no
    network): same call signature and output field (`.input_ids`, [B, max_length] int64, padded / truncated);
    ids are a byte-pair hash of the text — NOT a real vocabulary, only for synthetic-weight runs."""

    def __init__(self, vocab_size: int, bos: int | None, eos: int, pad: int):
        self.vocab_size, self.bos, self.eos, self.pad = vocab_size, bos, eos, pad

    @classmethod
    def clip(cls, vocab_size=49408):
        return cls(vocab_size, vocab_size - 2, vocab_size - 1, vocab_size - 1)     # <|startoftext|>, <|endoftext|> (= pad)

    @classmethod
    def t5(cls, vocab_size=32128):
        return cls(vocab_size, None, 1, 0)                                        # </s> = 1, <pad> = 0

    def __call__(self, prompt, padding="max_length", max_length=77, truncation=True, return_tensors="pt", **kw):
        prompt = [prompt] if isinstance(prompt, str) else prompt
        lo = 2 if self.bos is None else 1
        hi = self.vocab_size - (1 if self.bos is None else 3)
        rows = []
        for text in prompt:
            words = text.encode("utf-8").split()
            body = [lo + (int.from_bytes(w[:8], "little") * 2654435761 + len(w)) % (hi - lo) for w in words]
            head = [] if self.bos is None else [self.bos]
            body = body[: max_length - len(head) - 1]
            row = head + body + [self.eos]
            rows.append(row + [self.pad] * (max_length - len(row)))
        return SimpleNamespace(input_ids=torch.tensor(rows, dtype=torch.int64))
