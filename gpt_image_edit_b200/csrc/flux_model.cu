// FLUX-Kontext MMDiT forward composed from the libb2f kernels (no torch, no allocation, no host
// sync inside b2f_flux_forward — CUDA-graph capturable).
//
// Restates diffusers 0.32.2 FluxTransformer2DModel.forward (SURVEY.md Appendix A.1) as the sequence
//   x_embedder / context_embedder -> 19 x double block -> 38 x single block -> norm_out -> proj_out
// over ONE joint activation buffer h[B, S_txt + S_img, d] (text rows first), so the torch.cat calls
// of the reference ([txt;img] Q/K/V, [c;x] before the single blocks, [attn|mlp] before proj_out)
// become pointer offsets:
//   * Q/K/V of both streams are written by the QKV GEMMs straight into qkv[B, S, 3d];
//   * attention reads them through strided TMA maps and writes into cat[B, S, 5d][:, :, 0:d];
//   * the MLP up-projection (GELU fused) writes into cat[:, :, d:5d]; the single-block proj_out
//     GEMM reads cat with K = 5d.
// Reference call sites of this path: univa/utils/flux_pipeline.py:1067-1077,
// univa/models/modeling_univa_denoise_tower.py:103-110.
#include <algorithm>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "flux_ctx.h"
#include "host_common.h"

namespace b2f {

static int64_t mod_width_of(const b2f_flux_cfg& c) {
  const int64_t d = (int64_t)c.num_heads * c.head_dim;
  return (int64_t)c.num_double * 12 * d + (int64_t)c.num_single * 3 * d + 2 * d;
}

static int expect(FluxCtx* c, const std::string& key, int64_t numel, const bf16_t** dst) {
  auto it = c->bound.find(key);
  if (it == c->bound.end()) {
    fprintf(stderr, "[b2f] flux_finalize: weight '%s' was never bound\n", key.c_str());
    return B2F_ERR_INVALID;
  }
  if (it->second.second != numel) {
    fprintf(stderr, "[b2f] flux_finalize: weight '%s' has %lld elements, expected %lld\n",
            key.c_str(), (long long)it->second.second, (long long)numel);
    return B2F_ERR_INVALID;
  }
  *dst = static_cast<const bf16_t*>(it->second.first);
  return B2F_OK;
}
static int expect_lin(FluxCtx* c, const std::string& name, int64_t out_f, int64_t in_f, Lin* l) {
  int rc = expect(c, name + ".weight", out_f * in_f, &l->w);
  if (rc) return rc;
  return expect(c, name + ".bias", out_f, &l->b);
}

// The model's linears: every one a LoRA can target, by its bound name (the fused ones: attn.qkv, attn.add_qkv,
// qkv_mlp) or, for the AdaLN linears, by its diffusers name (rows of the fused adaln weight, which is not a target).
// f(name, lin or nullptr, row0, out, in); the lin is const when the context is.
template <class Ctx, class F>
static void for_each_linear(Ctx* c, F&& f) {
  const b2f_flux_cfg& g = c->cfg;
  const int64_t d = c->d;
  f(std::string("x_embedder"), &c->x_embedder, 0, d, (int64_t)g.in_channels);
  f(std::string("context_embedder"), &c->context_embedder, 0, d, (int64_t)g.joint_dim);
  f(std::string("time_text_embed.timestep_embedder.linear_1"), &c->t1, 0, d, 256);
  f(std::string("time_text_embed.timestep_embedder.linear_2"), &c->t2, 0, d, d);
  if (g.guidance_embeds) {
    f(std::string("time_text_embed.guidance_embedder.linear_1"), &c->g1, 0, d, 256);
    f(std::string("time_text_embed.guidance_embedder.linear_2"), &c->g2, 0, d, d);
  }
  f(std::string("time_text_embed.text_embedder.linear_1"), &c->p1, 0, d, (int64_t)g.pooled_dim);
  f(std::string("time_text_embed.text_embedder.linear_2"), &c->p2, 0, d, d);
  f(std::string("proj_out"), &c->proj_out, 0, (int64_t)g.out_channels, d);
  for (int i = 0; i < g.num_double; ++i) {
    const std::string p = "transformer_blocks." + std::to_string(i) + ".";
    auto& w = c->dbl[i];
    f(p + "attn.qkv", &w.qkv, 0, 3 * d, d);
    f(p + "attn.add_qkv", &w.add_qkv, 0, 3 * d, d);
    f(p + "attn.to_out.0", &w.to_out, 0, d, d);
    f(p + "attn.to_add_out", &w.to_add_out, 0, d, d);
    f(p + "ff.net.0.proj", &w.ff1, 0, 4 * d, d);
    f(p + "ff.net.2", &w.ff2, 0, d, 4 * d);
    f(p + "ff_context.net.0.proj", &w.ffc1, 0, 4 * d, d);
    f(p + "ff_context.net.2", &w.ffc2, 0, d, 4 * d);
    f(p + "norm1.linear", nullptr, (int64_t)i * 12 * d, 6 * d, d);
    f(p + "norm1_context.linear", nullptr, (int64_t)i * 12 * d + 6 * d, 6 * d, d);
  }
  for (int i = 0; i < g.num_single; ++i) {
    const std::string p = "single_transformer_blocks." + std::to_string(i) + ".";
    auto& w = c->sgl[i];
    f(p + "qkv_mlp", &w.qkv_mlp, 0, 7 * d, d);
    f(p + "proj_out", &w.proj_out, 0, d, 5 * d);
    f(p + "norm.linear", nullptr, (int64_t)g.num_double * 12 * d + (int64_t)i * 3 * d, 3 * d, d);
  }
  f(std::string("norm_out.linear"), nullptr, (int64_t)g.num_double * 12 * d + (int64_t)g.num_single * 3 * d, 2 * d, d);
}

static int adaln_rmax(const FluxCtx* c) {
  int r = 0;
  for (const auto& kv : c->adaln_lora) r = std::max(r, kv.second.l.r_pad);
  return r;
}

// The e4m3 rows and per-token scales standing in for a block linear's bf16 input A while FP8 is on (b2f_flux_set_fp8).
struct Q8 {
  const uint8_t* a;
  int64_t lda, a_bs;
  const float* s;
  int64_t s_bs;
};

// A linear layer of the forward with its unfused LoRA, if one is bound:
//   T = bf16(colscale * cs_mul * (A Acat^T))  into tb [batch, M, r_pad]    (gemm_colscale)
//   out = epi(A W^T + T Bcat^T + bias)                                      (gemm_bf16_lora: r_pad / 64 more k-blocks)
// Without one it is exactly the plain gemm_bf16 launch.  With q8 (FP8 on) it is the FP8 launch on (q8, w8); an adapter
// (FP8 mode 2) then runs its down projection on the bf16 input A and extends the FP8 launch (gemm_fp8_lora).
static int lin_fwd(const Lin& l, bf16_t* tb, float cs_mul, const void* A, int64_t lda, int64_t a_bs, int64_t ldw,
                   void* out, int64_t ldc, int64_t out_bs, int batch, int M, int N, int K, int epi, const void* resid,
                   int64_t ldr, int64_t resid_bs, const void* gate, int64_t gate_ld, cudaStream_t st,
                   const Q8* q8 = nullptr) {
  if (q8 && !l.lora.A)
    return b2f_gemm_fp8(q8->a, q8->lda, q8->a_bs, q8->s, q8->s_bs, l.w8, K, l.ws, l.b, out, ldc, out_bs, batch, M, N, K,
                        epi, resid, ldr, resid_bs, gate, gate_ld, st);
  if (!l.lora.A)
    return b2f_gemm_bf16(A, lda, a_bs, l.w, ldw, l.b, out, ldc, out_bs, batch, M, N, K, epi, resid, ldr, resid_bs, gate,
                         gate_ld, st);
  const int r = l.lora.r_pad;
  const int64_t t_bs = (int64_t)M * r;
  int rc = b2f_gemm_colscale(A, lda, a_bs, l.lora.A, K, tb, r, t_bs, batch, M, r, K, l.lora.cs, cs_mul, st);
  if (rc) return rc;
  if (q8)
    return b2f_gemm_fp8_lora(q8->a, q8->lda, q8->a_bs, q8->s, q8->s_bs, l.w8, K, l.ws, l.b, out, ldc, out_bs, batch, M,
                             N, K, epi, resid, ldr, resid_bs, gate, gate_ld, tb, r, t_bs, l.lora.Bc, r, r, st);
  return b2f_gemm_bf16_lora(A, lda, a_bs, l.w, ldw, l.b, out, ldc, out_bs, batch, M, N, K, epi, resid, ldr, resid_bs,
                            gate, gate_ld, tb, r, t_bs, l.lora.Bc, r, r, st);
}
static int qkv_fwd(const Lin& l, bf16_t* tb, float cs_mul, const void* A, int64_t lda, int64_t a_bs, int64_t ldw,
                   void* out, int64_t ldc, int64_t out_bs, int batch, int M, int d_model, int K, const void* nw_q,
                   const void* nw_k, const float* cos, const float* sin, int rope_row0, float eps, int n_extra,
                   void* out_extra, int64_t ld_extra, int64_t bs_extra, int epi_extra, cudaStream_t st,
                   const Q8* q8 = nullptr) {
  if (q8 && !l.lora.A)
    return b2f_gemm_qkv_norm_rope_fp8(q8->a, q8->lda, q8->a_bs, q8->s, q8->s_bs, l.w8, K, l.ws, l.b, out, ldc, out_bs,
                                      batch, M, d_model, K, nw_q, nw_k, cos, sin, rope_row0, eps, n_extra, out_extra,
                                      ld_extra, bs_extra, epi_extra, st);
  if (!l.lora.A)
    return b2f_gemm_qkv_norm_rope(A, lda, a_bs, l.w, ldw, l.b, out, ldc, out_bs, batch, M, d_model, K, nw_q, nw_k, cos,
                                  sin, rope_row0, eps, n_extra, out_extra, ld_extra, bs_extra, epi_extra, st);
  const int r = l.lora.r_pad;
  const int64_t t_bs = (int64_t)M * r;
  int rc = b2f_gemm_colscale(A, lda, a_bs, l.lora.A, K, tb, r, t_bs, batch, M, r, K, l.lora.cs, cs_mul, st);
  if (rc) return rc;
  if (q8)
    return b2f_gemm_qkv_norm_rope_fp8_lora(q8->a, q8->lda, q8->a_bs, q8->s, q8->s_bs, l.w8, K, l.ws, l.b, out, ldc,
                                           out_bs, batch, M, d_model, K, nw_q, nw_k, cos, sin, rope_row0, eps, n_extra,
                                           out_extra, ld_extra, bs_extra, epi_extra, tb, r, t_bs, l.lora.Bc, r, r, st);
  return b2f_gemm_qkv_norm_rope_lora(A, lda, a_bs, l.w, ldw, l.b, out, ldc, out_bs, batch, M, d_model, K, nw_q, nw_k, cos,
                                     sin, rope_row0, eps, n_extra, out_extra, ld_extra, bs_extra, epi_extra, tb, r, t_bs,
                                     l.lora.Bc, r, r, st);
}

// The ten FP8-capable linears of each block (b2f_flux_bind_fp8): every linear of for_each_linear inside a block that is
// not an AdaLN linear.
template <class F>
static void for_each_block_linear(FluxCtx* c, F&& f) {
  for_each_linear(c, [&](const std::string& name, Lin* l, int64_t, int64_t out_f, int64_t in_f) {
    if (l && (name.rfind("transformer_blocks.", 0) == 0 || name.rfind("single_transformer_blocks.", 0) == 0))
      f(name, l, out_f, in_f);
  });
}

int FluxCtx::lora_rmax() const {
  int r = adaln_rmax(this);
  for_each_linear(this, [&](const std::string&, const Lin* l, int64_t, int64_t, int64_t) {
    if (l) r = std::max(r, l->lora.r_pad);
  });
  return r;
}

namespace {
// Regions of a caller's workspace, each starting at the next 256-byte boundary and counted with 256 bytes of room for
// that, so `bytes` suffices wherever the workspace starts.
struct Regions {
  uintptr_t end;   // the workspace, then the end of the last region
  size_t bytes = 0;
  template <class T>
  T* take(size_t n) {
    const uintptr_t p = al256(end);
    end = p + n;
    bytes += n + 256;
    return reinterpret_cast<T*>(p);
  }
};

// b2f_flux_temb's workspace, one region: 2 sinusoid tables [rows,256] + 6 activations [rows,d] (+ LoRA T [rows, r_pad]
// with adapters bound)
struct TembWs {
  bf16_t *sin_t, *sin_g, *a1, *et, *eg, *ep, *tb;
  size_t bytes;
};
TembWs temb_ws(const FluxCtx* c, void* ws, int rows) {
  const size_t n = rows, d = c->d;
  Regions r{reinterpret_cast<uintptr_t>(ws)};
  TembWs w;
  w.sin_t = r.take<bf16_t>((n * 256 * 2 + n * d * 6 + n * c->lora_rmax()) * 2);
  w.sin_g = w.sin_t + n * 256;
  w.a1 = w.sin_g + n * 256;   // hidden
  w.et = w.a1 + n * d;
  w.eg = w.et + n * d;
  w.ep = w.eg + n * d;
  w.tb = w.ep + n * d;
  w.bytes = r.bytes;
  return w;
}
}  // namespace

FwdWs fwd_ws(const FluxCtx* c, void* ws, int B, int S_img, int S_txt) {
  const size_t d = c->d, S = (size_t)S_img + S_txt, BS = (size_t)B * S, H = c->cfg.num_heads;
  const size_t S_pad = (S + 127) / 128 * 128;
  Regions r{reinterpret_cast<uintptr_t>(ws)};
  FwdWs w{};
  w.h = r.take<bf16_t>(BS * (10 * d + c->lora_rmax()) * 2);
  w.xn = w.h + BS * d;
  w.qkv = w.xn + BS * d;
  w.cat = w.qkv + BS * 3 * d;
  w.tb = w.cat + BS * 5 * d;
  if (c->fp8) {
    w.q8 = r.take<uint8_t>(BS * (5 * d + 4));
    w.qs = reinterpret_cast<float*>(w.q8 + BS * 5 * d);
  }
  if (c->fp8_attn) {
    w.aq8 = r.take<uint8_t>(B * d * (2 * S + S_pad) + B * (2 * H + d) * 4);
    w.ak8 = w.aq8 + BS * d;
    w.av8 = w.ak8 + BS * d;
    w.asq = reinterpret_cast<float*>(w.av8 + B * d * S_pad);
    w.ask = w.asq + B * H;
    w.asv = w.ask + B * H;
  }
  w.bytes = r.bytes;
  return w;
}

}  // namespace b2f

using namespace b2f;

extern "C" {

int b2f_flux_create(b2f_flux** out, const b2f_flux_cfg* cfg) {
  if (!out || !cfg) return B2F_ERR_INVALID;
  if (cfg->head_dim != 128) return B2F_ERR_UNSUPPORTED;
  const int64_t d = (int64_t)cfg->num_heads * cfg->head_dim;
  if (d % 256 || cfg->in_channels % 8 || cfg->out_channels % 8 || cfg->joint_dim % 8 ||
      cfg->pooled_dim % 8 || cfg->num_double < 0 || cfg->num_single < 0 || cfg->mlp_ratio != 4)
    return B2F_ERR_UNSUPPORTED;
  FluxCtx* c = new (std::nothrow) FluxCtx();
  if (!c) return B2F_ERR_INVALID;
  c->cfg = *cfg;
  c->d = (int)d;
  c->mod_width = mod_width_of(*cfg);
  *out = reinterpret_cast<b2f_flux*>(c);
  return B2F_OK;
}

void b2f_flux_destroy(b2f_flux* h) { delete reinterpret_cast<FluxCtx*>(h); }

int b2f_flux_bind_weight(b2f_flux* h, const char* key, const void* dptr, int64_t numel) {
  FluxCtx* c = reinterpret_cast<FluxCtx*>(h);
  if (!c || !key || !dptr || numel <= 0) return B2F_ERR_INVALID;
  if (reinterpret_cast<uintptr_t>(dptr) & 15) return B2F_ERR_ALIGN;
  c->bound[key] = {dptr, numel};
  c->finalized = false;
  return B2F_OK;
}

int64_t b2f_flux_mod_width(const b2f_flux* h) {
  const FluxCtx* c = reinterpret_cast<const FluxCtx*>(h);
  return c ? c->mod_width : 0;
}

int b2f_flux_finalize(b2f_flux* h) {
  FluxCtx* c = reinterpret_cast<FluxCtx*>(h);
  if (!c) return B2F_ERR_INVALID;
  const b2f_flux_cfg& g = c->cfg;
  c->dbl.assign(g.num_double, DoubleW());
  c->sgl.assign(g.num_single, SingleW());
  // the fused AdaLN weight, every other linear of the inventory, the blocks' per-head RMSNorm weights
  int rc = expect_lin(c, "adaln", c->mod_width, c->d, &c->adaln);
  for_each_linear(c, [&](const std::string& name, Lin* l, int64_t, int64_t out_f, int64_t in_f) {
    if (!rc && l) rc = expect_lin(c, name, out_f, in_f, l);
  });
  auto norm = [&](const std::string& name, const bf16_t** dst) {
    if (!rc) rc = expect(c, name, g.head_dim, dst);
  };
  for (int i = 0; i < g.num_double; ++i) {
    const std::string p = "transformer_blocks." + std::to_string(i) + ".attn.norm_";
    DoubleW& w = c->dbl[i];
    norm(p + "q.weight", &w.norm_q);
    norm(p + "k.weight", &w.norm_k);
    norm(p + "added_q.weight", &w.norm_added_q);
    norm(p + "added_k.weight", &w.norm_added_k);
  }
  for (int i = 0; i < g.num_single; ++i) {
    const std::string p = "single_transformer_blocks." + std::to_string(i) + ".attn.norm_";
    norm(p + "q.weight", &c->sgl[i].norm_q);
    norm(p + "k.weight", &c->sgl[i].norm_k);
  }
  if (rc) return rc;
  // (re)binding weights drops every LoRA binding (the FP8 ones went with the reassigned block weights)
  for_each_linear(c, [](const std::string&, Lin* l, int64_t, int64_t, int64_t) {
    if (l) l->lora = LoraBind();
  });
  c->adaln_lora.clear();
  c->fp8 = false;
  c->fp8_lora = false;
  c->fp8_attn = false;
  c->text_win = nullptr;
  c->text_win_B = 0;
  c->finalized = true;
  return B2F_OK;
}

int b2f_flux_set_rope(b2f_flux* h, const float* cos, const float* sin, int S) {
  FluxCtx* c = reinterpret_cast<FluxCtx*>(h);
  if (!c || !cos || !sin || S <= 0) return B2F_ERR_INVALID;
  if ((reinterpret_cast<uintptr_t>(cos) | reinterpret_cast<uintptr_t>(sin)) & 15) return B2F_ERR_ALIGN;
  c->rope_cos = cos;
  c->rope_sin = sin;
  c->rope_S = S;
  return B2F_OK;
}

size_t b2f_flux_workspace_bytes(const b2f_flux* h, int B, int S_img, int S_txt) {
  const FluxCtx* c = reinterpret_cast<const FluxCtx*>(h);
  if (!c || B <= 0 || S_img <= 0 || S_txt < 0) return 0;
  return fwd_ws(c, nullptr, B, S_img, S_txt).bytes;
}

size_t b2f_flux_temb_workspace_bytes(const b2f_flux* h, int rows) {
  const FluxCtx* c = reinterpret_cast<const FluxCtx*>(h);
  if (!c || rows <= 0) return 0;
  return temb_ws(c, nullptr, rows).bytes;
}

int b2f_flux_temb(b2f_flux* h, const float* timestep, const float* guidance, const void* pooled,
                  int64_t pooled_ld, int rows, void* temb, void* silu_temb, void* ws,
                  size_t ws_bytes, b2f_stream_t stream_) {
  FluxCtx* c = reinterpret_cast<FluxCtx*>(h);
  if (!c || !c->finalized || !timestep || !pooled || !temb || !silu_temb || rows <= 0 || !ws)
    return B2F_ERR_INVALID;
  if (c->cfg.guidance_embeds && !guidance) return B2F_ERR_INVALID;
  const TembWs w = temb_ws(c, ws, rows);
  if (ws_bytes < w.bytes) return B2F_ERR_WORKSPACE;
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  const int d = c->d;
  bf16_t *sin_t = w.sin_t, *sin_g = w.sin_g, *a1 = w.a1, *et = w.et, *eg = w.eg, *ep = w.ep, *tb = w.tb;
  const float ls = c->lora_scale;
  int rc;
  if ((rc = b2f_temb_sinusoid(timestep, sin_t, rows, st))) return rc;
  if ((rc = lin_fwd(c->t1, tb, ls, sin_t, 256, 0, 256, a1, d, 0, 1, rows, d, 256, B2F_EPI_SILU,
                      nullptr, 0, 0, nullptr, 0, st)))
    return rc;
  if ((rc = lin_fwd(c->t2, tb, ls, a1, d, 0, d, et, d, 0, 1, rows, d, d, B2F_EPI_BIAS, nullptr,
                      0, 0, nullptr, 0, st)))
    return rc;
  const bf16_t* eg_ptr = nullptr;
  if (c->cfg.guidance_embeds) {
    if ((rc = b2f_temb_sinusoid(guidance, sin_g, rows, st))) return rc;
    if ((rc = lin_fwd(c->g1, tb, ls, sin_g, 256, 0, 256, a1, d, 0, 1, rows, d, 256,
                        B2F_EPI_SILU, nullptr, 0, 0, nullptr, 0, st)))
      return rc;
    if ((rc = lin_fwd(c->g2, tb, ls, a1, d, 0, d, eg, d, 0, 1, rows, d, d, B2F_EPI_BIAS,
                        nullptr, 0, 0, nullptr, 0, st)))
      return rc;
    eg_ptr = eg;
  }
  if ((rc = lin_fwd(c->p1, tb, ls, pooled, pooled_ld, 0, c->cfg.pooled_dim, a1, d, 0, 1, rows, d,
                      c->cfg.pooled_dim, B2F_EPI_SILU, nullptr, 0, 0, nullptr, 0, st)))
    return rc;
  if ((rc = lin_fwd(c->p2, tb, ls, a1, d, 0, d, ep, d, 0, 1, rows, d, d, B2F_EPI_BIAS, nullptr,
                      0, 0, nullptr, 0, st)))
    return rc;
  return b2f_temb_combine(et, eg_ptr, ep, temb, silu_temb, (int64_t)rows * d, st);
}

int b2f_flux_modulation(b2f_flux* h, const void* silu_temb, int rows, void* mod, b2f_stream_t stream_) {
  FluxCtx* c = reinterpret_cast<FluxCtx*>(h);
  if (!c || !c->finalized || !silu_temb || !mod || rows <= 0) return B2F_ERR_INVALID;
  if (!c->adaln_lora.empty()) {
    fprintf(stderr, "[b2f] flux_modulation: AdaLN LoRA adapters are bound; use b2f_flux_modulation_ws\n");
    return B2F_ERR_WORKSPACE;
  }
  return b2f_gemm_bf16(silu_temb, c->d, 0, c->adaln.w, c->d, c->adaln.b, mod, c->mod_width, 0, 1, rows,
                       (int)c->mod_width, c->d, B2F_EPI_BIAS, nullptr, 0, 0, nullptr, 0,
                       static_cast<cudaStream_t>(stream_));
}

size_t b2f_flux_modulation_workspace_bytes(const b2f_flux* h, int rows) {
  const FluxCtx* c = reinterpret_cast<const FluxCtx*>(h);
  if (!c || rows <= 0) return 0;
  return (size_t)rows * adaln_rmax(c) * 2 + 256;
}

int b2f_flux_modulation_ws(b2f_flux* h, const void* silu_temb, int rows, void* mod, void* ws, size_t ws_bytes,
                           b2f_stream_t stream_) {
  FluxCtx* c = reinterpret_cast<FluxCtx*>(h);
  if (!c || !c->finalized || !silu_temb || !mod || rows <= 0 || !ws) return B2F_ERR_INVALID;
  if (ws_bytes < b2f_flux_modulation_workspace_bytes(h, rows)) return B2F_ERR_WORKSPACE;
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  const int64_t d = c->d;
  int rc = b2f_gemm_bf16(silu_temb, d, 0, c->adaln.w, d, c->adaln.b, mod, c->mod_width, 0, 1, rows, (int)c->mod_width,
                         (int)d, B2F_EPI_BIAS, nullptr, 0, 0, nullptr, 0, st);
  if (rc) return rc;
  // each AdaLN linear with an adapter: its own K-extended launch over its rows of adaln, overwriting its columns of mod
  bf16_t* tb = al256<bf16_t>(ws);
  bf16_t* m = static_cast<bf16_t*>(mod);
  for (const auto& kv : c->adaln_lora) {
    const AdalnLora& a = kv.second;
    Lin l;
    l.w = c->adaln.w + a.row0 * d;
    l.b = c->adaln.b + a.row0;
    l.lora = a.l;
    if ((rc = lin_fwd(l, tb, c->lora_scale, silu_temb, d, 0, d, m + a.row0, c->mod_width, 0, 1, rows, (int)a.rows,
                      (int)d, B2F_EPI_BIAS, nullptr, 0, 0, nullptr, 0, st)))
      return rc;
  }
  return B2F_OK;
}

int b2f_flux_bind_lora(b2f_flux* h, const char* target, const void* Acat, const void* Bcat, const float* colscale,
                       int r_pad) {
  FluxCtx* c = reinterpret_cast<FluxCtx*>(h);
  if (!c || !c->finalized || !target) return B2F_ERR_INVALID;
  const bool unbind = Acat == nullptr;
  if (!unbind && c->fp8 && !c->fp8_lora) {
    fprintf(stderr, "[b2f] flux_bind_lora: FP8 is on; fuse the adapter or switch FP8 off first\n");
    return B2F_ERR_UNSUPPORTED;
  }
  if (!unbind) {
    if (!Bcat || !colscale || r_pad <= 0 || r_pad % 64) return B2F_ERR_INVALID;
    if ((reinterpret_cast<uintptr_t>(Acat) | reinterpret_cast<uintptr_t>(Bcat) |
         reinterpret_cast<uintptr_t>(colscale)) & 15)
      return B2F_ERR_ALIGN;
  }
  LoraBind lb;
  if (!unbind) {
    lb.A = static_cast<const bf16_t*>(Acat);
    lb.Bc = static_cast<const bf16_t*>(Bcat);
    lb.cs = colscale;
    lb.r_pad = r_pad;
  }
  const std::string key(target);
  bool found = false;
  for_each_linear(c, [&](const std::string& name, Lin* l, int64_t row0, int64_t out_f, int64_t) {
    if (found || name != key) return;
    found = true;
    if (l) {
      l->lora = lb;
    } else if (unbind) {
      c->adaln_lora.erase(key);
    } else {
      AdalnLora a;
      a.row0 = row0;
      a.rows = out_f;
      a.l = lb;
      c->adaln_lora[key] = a;
    }
  });
  if (!found) {
    fprintf(stderr, "[b2f] flux_bind_lora: no linear named '%s'\n", target);
    return B2F_ERR_INVALID;
  }
  return B2F_OK;
}

int b2f_flux_clear_lora(b2f_flux* h) {
  FluxCtx* c = reinterpret_cast<FluxCtx*>(h);
  if (!c || !c->finalized) return B2F_ERR_INVALID;
  for_each_linear(c, [](const std::string&, Lin* l, int64_t, int64_t, int64_t) {
    if (l) l->lora = LoraBind();
  });
  c->adaln_lora.clear();
  return B2F_OK;
}

int b2f_flux_set_lora_scale(b2f_flux* h, float scale) {
  FluxCtx* c = reinterpret_cast<FluxCtx*>(h);
  if (!c) return B2F_ERR_INVALID;
  c->lora_scale = scale;
  return B2F_OK;
}

int b2f_flux_bind_fp8(b2f_flux* h, const char* name, const void* w8, const float* w_scale, int64_t numel) {
  FluxCtx* c = reinterpret_cast<FluxCtx*>(h);
  if (!c || !c->finalized || !name) return B2F_ERR_INVALID;
  if (w8 && !w_scale) return B2F_ERR_INVALID;
  if ((reinterpret_cast<uintptr_t>(w8) | reinterpret_cast<uintptr_t>(w_scale)) & 15) return B2F_ERR_ALIGN;
  if (!w8 && c->fp8) {
    fprintf(stderr, "[b2f] flux_bind_fp8: cannot unbind '%s' while FP8 is on\n", name);
    return B2F_ERR_INVALID;
  }
  const std::string key(name);
  int rc = B2F_ERR_INVALID;
  bool found = false;
  for_each_block_linear(c, [&](const std::string& n, Lin* l, int64_t out_f, int64_t in_f) {
    if (found || n != key) return;
    found = true;
    if (w8 && numel != out_f * in_f) {
      fprintf(stderr, "[b2f] flux_bind_fp8: '%s' has %lld elements, expected %lld\n", name, (long long)numel,
              (long long)(out_f * in_f));
      return;
    }
    l->w8 = static_cast<const uint8_t*>(w8);
    l->ws = w8 ? w_scale : nullptr;
    rc = B2F_OK;
  });
  if (!found) fprintf(stderr, "[b2f] flux_bind_fp8: no block linear named '%s'\n", name);
  return rc;
}

int b2f_flux_set_fp8(b2f_flux* h, int mode) {
  FluxCtx* c = reinterpret_cast<FluxCtx*>(h);
  if (!c || !c->finalized) return B2F_ERR_INVALID;
  if (!mode) {
    c->fp8 = false;
    c->fp8_lora = false;
    return B2F_OK;
  }
  const bool with_lora = mode == 2;
  if (!with_lora && c->lora_rmax() > 0) {
    fprintf(stderr, "[b2f] flux_set_fp8: unfused LoRA adapters are bound; fuse or unbind them first\n");
    return B2F_ERR_UNSUPPORTED;
  }
  int rc = B2F_OK;
  for_each_block_linear(c, [&](const std::string& n, Lin* l, int64_t, int64_t) {
    if (!rc && !l->w8) {
      fprintf(stderr, "[b2f] flux_set_fp8: no FP8 weight bound for '%s'\n", n.c_str());
      rc = B2F_ERR_INVALID;
    }
  });
  if (rc) return rc;
  c->fp8 = true;
  c->fp8_lora = with_lora;
  return B2F_OK;
}

int b2f_flux_set_fp8_attention(b2f_flux* h, int on) {
  FluxCtx* c = reinterpret_cast<FluxCtx*>(h);
  if (!c || !c->finalized) return B2F_ERR_INVALID;
  if (on && c->cfg.head_dim != 128) return B2F_ERR_UNSUPPORTED;
  c->fp8_attn = on != 0;
  return B2F_OK;
}

int b2f_flux_set_text_window(b2f_flux* h, const int32_t* win_dev, int B) {
  FluxCtx* c = reinterpret_cast<FluxCtx*>(h);
  if (!c || !c->finalized) return B2F_ERR_INVALID;
  if (win_dev && B <= 0) return B2F_ERR_INVALID;
  if (win_dev && (reinterpret_cast<uintptr_t>(win_dev) & 7)) return B2F_ERR_ALIGN;
  c->text_win = win_dev;
  c->text_win_B = win_dev ? B : 0;
  return B2F_OK;
}

int b2f_flux_lora_rank(const b2f_flux* h) {
  const FluxCtx* c = reinterpret_cast<const FluxCtx*>(h);
  return c && c->finalized ? c->lora_rmax() : 0;
}

int b2f_flux_forward(b2f_flux* h, const void* hidden, const void* enc, const void* mod,
                     int64_t mod_ld, void* out, int B, int S_img, int S_txt, int n_out_rows,
                     void* ws, size_t ws_bytes, int first_block, int last_block,
                     b2f_stream_t stream_) {
  return flux_forward(reinterpret_cast<FluxCtx*>(h), hidden, enc, mod, mod_ld, out, B, S_img, S_txt, n_out_rows, ws,
                      ws_bytes, first_block, last_block, nullptr, static_cast<cudaStream_t>(stream_));
}

}  // extern "C"

namespace b2f {

int flux_forward(FluxCtx* c, const void* hidden, const void* enc, const void* mod, int64_t mod_ld, void* out, int B,
                 int S_img, int S_txt, int n_out_rows, void* ws, size_t ws_bytes, int first_block, int last_block,
                 bf16_t* x0, cudaStream_t st) {
  if (!c || !c->finalized) return B2F_ERR_INVALID;
  if (!hidden || !enc || !mod || !out || !ws || B <= 0 || S_img <= 0 || S_txt <= 0)
    return B2F_ERR_INVALID;
  if (n_out_rows <= 0 || n_out_rows > S_img) return B2F_ERR_INVALID;
  const int S = S_img + S_txt;
  if (!c->rope_cos || c->rope_S != S) {
    fprintf(stderr, "[b2f] flux_forward: RoPE tables not set for S=%d (have %d)\n", S, c->rope_S);
    return B2F_ERR_INVALID;
  }
  const FwdWs L = fwd_ws(c, ws, B, S_img, S_txt);
  if (ws_bytes < L.bytes) return B2F_ERR_WORKSPACE;
  if (c->text_win && c->text_win_B != B) {
    fprintf(stderr, "[b2f] flux_forward: text windows set for B=%d, forward has B=%d\n", c->text_win_B, B);
    return B2F_ERR_INVALID;
  }
  const b2f_flux_cfg& g = c->cfg;
  const int64_t d = c->d;
  const int H = g.num_heads;
  const float eps = 1e-6f;
  const float scale = 1.0f / sqrtf((float)g.head_dim);

  bf16_t *hb = L.h, *xn = L.xn, *qkv = L.qkv, *cat = L.cat, *tb = L.tb;
  // FP8 on: e4m3 rows q8 [B,S,5d] (pitch 5d bytes) and their scales qs [B,S], rewritten before each block linear
  uint8_t* q8 = L.q8;
  float* qs = L.qs;
  const bool f8 = c->fp8;
  const int64_t q8_bs = (int64_t)S * 5 * d;
  const Q8 q_txt{q8, 5 * d, q8_bs, qs, S};
  const Q8 q_img{q8 + (int64_t)S_txt * 5 * d, 5 * d, q8_bs, qs + S_txt, S};
  const Q8* qt = f8 ? &q_txt : nullptr;   // the text rows (a single block: all rows) of q8
  const Q8* qi = f8 ? &q_img : nullptr;
  // (K columns of cat from column c0) -> q8 over all S rows
  auto quant_cat = [&](int64_t c0, int K) {
    return b2f_quant_fp8_rows(cat + c0, 5 * d, (int64_t)S * 5 * d, q8, 5 * d, q8_bs, qs, S, B, S, K, st);
  };
  // FP8 attention on: q8 / k8 [B,S,d], v8t [B,H,128,S_pad] e4m3 and their scales sq / sk [B,H], sv [B,d] fp32
  uint8_t *aq8 = L.aq8, *ak8 = L.ak8, *av8 = L.av8;
  float *asq = L.asq, *ask = L.ask, *asv = L.asv;
  // joint attention of the qkv buffer into cat[:, :, :d]
  // (with text windows set: the window entry points over the text rows [0, S_txt))
  const int32_t* tw = c->text_win;
  auto attention = [&]() {
    if (!c->fp8_attn) {
      if (tw)
        return b2f_attention_fwd_window(qkv, 3 * d, qkv + d, 3 * d, qkv + 2 * d, 3 * d, cat, 5 * d, B, H, H, S, S,
                                        g.head_dim, scale, tw, S_txt, st);
      return b2f_attention_fwd(qkv, 3 * d, qkv + d, 3 * d, qkv + 2 * d, 3 * d, cat, 5 * d, B, H, H, S, S, g.head_dim,
                               scale, 0, st);
    }
    const int r = tw ? b2f_attn_quant_fp8_window(qkv, 3 * d, qkv + d, 3 * d, qkv + 2 * d, 3 * d, aq8, ak8, asq, ask, av8,
                                                 asv, B, H, S, g.head_dim, tw, S_txt, st)
                     : b2f_attn_quant_fp8(qkv, 3 * d, qkv + d, 3 * d, qkv + 2 * d, 3 * d, aq8, ak8, asq, ask, av8, asv,
                                          B, H, S, g.head_dim, st);
    if (r) return r;
    if (tw)
      return b2f_attention_fp8_window(aq8, ak8, asq, ask, av8, asv, cat, 5 * d, B, H, S, g.head_dim, scale, tw, S_txt,
                                      st);
    return b2f_attention_fp8(aq8, ak8, asq, ask, av8, asv, cat, 5 * d, B, H, S, g.head_dim, scale, 0, st);
  };
  const float ls = c->lora_scale;
  const int64_t h_bs = (int64_t)S * d, qkv_bs = (int64_t)S * 3 * d, cat_bs = (int64_t)S * 5 * d;
  bf16_t* h_img = hb + (int64_t)S_txt * d;
  bf16_t* h_txt = hb;
  bf16_t* xn_img = xn + (int64_t)S_txt * d;
  bf16_t* xn_txt = xn;
  bf16_t* qkv_img = qkv + (int64_t)S_txt * 3 * d;
  bf16_t* qkv_txt = qkv;
  bf16_t* cat_img = cat + (int64_t)S_txt * 5 * d;
  bf16_t* cat_txt = cat;
  const bf16_t* modp = static_cast<const bf16_t*>(mod);
  // the modulated LayerNorm of h before a step's linears (the first split_row rows of each item take scale / shift,
  // the others scale_b / shift_b): e4m3 rows into q8 while FP8 is on, bf16 rows into xn when FP8 is off or an adapter
  // on one of those linears reads them (FP8 mode 2)
  auto ln_modulate = [&](const bf16_t* scale, const bf16_t* shift, int split_row, const bf16_t* scale_b,
                         const bf16_t* shift_b, bool adapted) {
    if (f8) {
      const int r = b2f_ln_modulate_fp8(hb, d, h_bs, scale, shift, mod_ld, q8, 5 * d, q8_bs, qs, S, B, S, (int)d, eps,
                                        split_row, scale_b, shift_b, st);
      if (r || !adapted) return r;
    }
    return b2f_ln_modulate(hb, d, h_bs, scale, shift, mod_ld, xn, d, h_bs, B, S, (int)d, eps, split_row, scale_b,
                           shift_b, st);
  };
  int rc;
#define RUN(expr) \
  if ((rc = (expr)) != 0) return rc
  const int total_blocks = g.num_double + g.num_single;
  if (first_block < 0) first_block = 0;
  if (last_block < 0 || last_block > total_blocks) last_block = total_blocks;

  if (first_block == 0) {
    // x = x_embedder(hidden) -> h[:, S_txt:],  c = context_embedder(enc) -> h[:, :S_txt]
    RUN(lin_fwd(c->x_embedder, tb, ls, hidden, g.in_channels, (int64_t)S_img * g.in_channels, g.in_channels, h_img,
                d, h_bs, B, S_img, (int)d, g.in_channels, B2F_EPI_BIAS, nullptr, 0, 0, nullptr, 0, st));
    RUN(lin_fwd(c->context_embedder, tb, ls, enc, g.joint_dim, (int64_t)S_txt * g.joint_dim, g.joint_dim, h_txt, d,
                h_bs, B, S_txt, (int)d, g.joint_dim, B2F_EPI_BIAS, nullptr, 0, 0, nullptr, 0, st));
    if (x0)   // the first-block cache's x0: the image rows of h before block 0, [B, S_img, d] contiguous
      RUN(cuda_err(cudaMemcpy2DAsync(x0, (size_t)S_img * d * 2, h_img, (size_t)h_bs * 2, (size_t)S_img * d * 2, B,
                                     cudaMemcpyDeviceToDevice, st),
                   "flux_forward: x0 copy"));
  }

  for (int blk = first_block; blk < last_block; ++blk) {
    if (blk < g.num_double) {
      const DoubleW& w = c->dbl[blk];
      // mod columns: [img: shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp | txt: same]
      const bf16_t* mi = modp + (int64_t)blk * 12 * d;
      const bf16_t* mt = mi + 6 * d;
      // both streams in one launch over the joint buffer: text rows use the context modulation
      RUN(ln_modulate(mt + d, mt, S_txt, mi + d, mi, w.qkv.lora.A || w.add_qkv.lora.A));
      // QKV projections with per-head RMSNorm + RoPE fused into the GEMM epilogue; both streams write
      // straight into the joint [txt; img] qkv buffer
      RUN(qkv_fwd(w.qkv, tb, ls, xn_img, d, h_bs, d, qkv_img, 3 * d, qkv_bs, B, S_img, (int)d,
                             (int)d, w.norm_q, w.norm_k, c->rope_cos, c->rope_sin, S_txt, eps, 0, nullptr, 0, 0, 0, st,
                             qi));
      RUN(qkv_fwd(w.add_qkv, tb, ls, xn_txt, d, h_bs, d, qkv_txt, 3 * d, qkv_bs, B, S_txt,
                             (int)d, (int)d, w.norm_added_q, w.norm_added_k, c->rope_cos, c->rope_sin, 0, eps, 0,
                             nullptr, 0, 0, 0, st, qt));
      RUN(attention());
      if (f8) RUN(quant_cat(0, (int)d));
      RUN(lin_fwd(w.to_out, tb, ls, cat_img, 5 * d, cat_bs, d, h_img, d, h_bs, B, S_img,
                    (int)d, (int)d, B2F_EPI_GATE_RESID, h_img, d, h_bs, mi + 2 * d, mod_ld, st, qi));
      RUN(lin_fwd(w.to_add_out, tb, ls, cat_txt, 5 * d, cat_bs, d, h_txt, d, h_bs, B,
                    S_txt, (int)d, (int)d, B2F_EPI_GATE_RESID, h_txt, d, h_bs, mt + 2 * d, mod_ld, st, qt));
      RUN(ln_modulate(mt + 4 * d, mt + 3 * d, S_txt, mi + 4 * d, mi + 3 * d, w.ff1.lora.A || w.ffc1.lora.A));
      RUN(lin_fwd(w.ff1, tb, ls, xn_img, d, h_bs, d, cat_img + d, 5 * d, cat_bs, B, S_img,
                    (int)(4 * d), (int)d, B2F_EPI_GELU_TANH, nullptr, 0, 0, nullptr, 0, st, qi));
      RUN(lin_fwd(w.ffc1, tb, ls, xn_txt, d, h_bs, d, cat_txt + d, 5 * d, cat_bs, B, S_txt,
                    (int)(4 * d), (int)d, B2F_EPI_GELU_TANH, nullptr, 0, 0, nullptr, 0, st, qt));
      if (f8) RUN(quant_cat(d, (int)(4 * d)));
      RUN(lin_fwd(w.ff2, tb, ls, cat_img + d, 5 * d, cat_bs, 4 * d, h_img, d, h_bs, B, S_img,
                    (int)d, (int)(4 * d), B2F_EPI_GATE_RESID, h_img, d, h_bs, mi + 5 * d, mod_ld, st, qi));
      RUN(lin_fwd(w.ffc2, tb, ls, cat_txt + d, 5 * d, cat_bs, 4 * d, h_txt, d, h_bs, B, S_txt,
                    (int)d, (int)(4 * d), B2F_EPI_GATE_RESID, h_txt, d, h_bs, mt + 5 * d, mod_ld, st, qt));
    } else {
      const int si = blk - g.num_double;
      const SingleW& w = c->sgl[si];
      // mod columns: [shift, scale, gate]
      const bf16_t* ms = modp + (int64_t)g.num_double * 12 * d + (int64_t)si * 3 * d;
      RUN(ln_modulate(ms + d, ms, 0, nullptr, nullptr, w.qkv_mlp.lora.A));
      // ONE launch for [to_q;to_k;to_v;proj_mlp] (N = 7d): Q/K get RMSNorm+RoPE, V passes through into
      // qkv, the MLP columns are GELU'd straight into cat[:, :, d:5d]
      RUN(qkv_fwd(w.qkv_mlp, tb, ls, xn, d, h_bs, d, qkv, 3 * d, qkv_bs, B, S, (int)d, (int)d,
                             w.norm_q, w.norm_k, c->rope_cos, c->rope_sin, 0, eps, (int)(4 * d), cat + d, 5 * d,
                             cat_bs, B2F_EPI_GELU_TANH, st, qt));
      RUN(attention());
      if (f8) RUN(quant_cat(0, (int)(5 * d)));
      RUN(lin_fwd(w.proj_out, tb, ls, cat, 5 * d, cat_bs, 5 * d, hb, d, h_bs, B, S, (int)d,
                    (int)(5 * d), B2F_EPI_GATE_RESID, hb, d, h_bs, ms + 2 * d, mod_ld, st, qt));
    }
  }

  if (last_block == total_blocks) {
    // norm_out (AdaLayerNormContinuous: chunk order scale, shift) + proj_out on the image rows
    const bf16_t* mo = modp + (int64_t)g.num_double * 12 * d + (int64_t)g.num_single * 3 * d;
    RUN(b2f_ln_modulate(h_img, d, h_bs, mo, mo + d, mod_ld, xn_img, d, h_bs, B, n_out_rows, (int)d, eps, 0, nullptr,
                        nullptr, st));
    RUN(lin_fwd(c->proj_out, tb, ls, xn_img, d, h_bs, d, out, g.out_channels,
                  (int64_t)n_out_rows * g.out_channels, B, n_out_rows, g.out_channels, (int)d,
                  B2F_EPI_BIAS, nullptr, 0, 0, nullptr, 0, st));
  }
#undef RUN
  return B2F_OK;
}

}  // namespace b2f
