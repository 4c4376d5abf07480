// FLUX VAE (diffusers AutoencoderKL, SURVEY.md A.4) encode / decode composed from libb2f kernels.
// Activations are NHWC bf16 inside; the ABI takes and returns the NCHW tensors the reference passes
// (univa/utils/flux_pipeline.py:600-613 encode -> latent_dist, :1127-1129 decode).
//   3x3 convs            wgmma implicit GEMM (conv.cu), residual add fused into conv2's epilogue
//   1x1 shortcut convs   plain wgmma GEMM over [pixels, C]
//   GroupNorm+SiLU       two HBM-bound passes (vae_kernels.cu)
//   mid-block attention  single head, dh = C: QK^T (fp32 scores, through the weight-gradient GEMM) and PV as wgmma
//                        GEMMs around a row softmax, over the P = h*w latent pixels padded to P8 = round_up(P, 8)
// b2f_vae_set_stop_stage ends a run after one stage of the numbering in b2f.h (tests read each stage's activation).
#include <map>
#include <string>
#include <vector>

#include "host_common.h"

namespace b2f {

typedef uint16_t bf16_t;

struct VaeCtx {
  b2f_vae_cfg cfg;
  std::map<std::string, std::pair<const void*, int64_t>> bound;
  bool finalized = false;
  int max_c = 0;
  int stop_stage = 0;  // b2f_vae_set_stop_stage: 0 runs to the end
};

struct VaeRun {
  VaeCtx* c;
  cudaStream_t st;
  bf16_t *X, *A, *B;   // three activation buffers (NHWC)
  bf16_t* attn_ws;     // mid-attention scratch
  double* stats;       // [N,32,2]
  bf16_t* ws0;         // start of the 256-aligned workspace
  int N;
  int rc = 0;
  int stage = 0;       // stages finished so far

  // Ends a stage whose activation X is [N, h, w, ch]; true when the run stops here (or has failed): the activation is
  // then at the start of the workspace.
  bool stage_done(int h, int w, int ch) {
    if (rc) return true;
    if (++stage != c->stop_stage) return false;
    if (X != ws0) run(cuda_err(cudaMemcpyAsync(ws0, X, (size_t)N * h * w * ch * sizeof(bf16_t), cudaMemcpyDeviceToDevice,
                                               st), "vae stage copy"));
    return true;
  }

  const bf16_t* w(const std::string& k) {
    auto it = c->bound.find(k);
    if (it == c->bound.end()) {
      if (!rc) fprintf(stderr, "[b2f] vae: weight '%s' not bound\n", k.c_str());
      rc = B2F_ERR_INVALID;
      return nullptr;
    }
    return static_cast<const bf16_t*>(it->second.first);
  }
  void run(int r) {
    if (!rc && r) rc = r;
  }
  void gn(const std::string& name, const bf16_t* x, bf16_t* y, long long P, int C, int silu) {
    if (rc) return;
    run(b2f_groupnorm_silu(x, w(name + ".weight"), w(name + ".bias"), y, stats, N, P, C, 1e-6f, silu, st));
  }
  void conv(const std::string& name, const bf16_t* in, bf16_t* out, const bf16_t* resid, int H, int W,
            int Cin, int Cout, int stride = 1, int nchw = 0) {
    if (rc) return;
    run(b2f_conv3x3(in, w(name + ".weight"), w(name + ".bias"), out, resid, N, H, W, Cin, Cout, stride, nchw, st));
  }
  // ResnetBlock2D in place on X: X[N,H,W,Cin] -> X[N,H,W,Cout]
  void resnet(const std::string& name, int H, int W, int Cin, int Cout) {
    const long long P = (long long)H * W;
    gn(name + ".norm1", X, A, P, Cin, 1);
    conv(name + ".conv1", A, B, nullptr, H, W, Cin, Cout);
    gn(name + ".norm2", B, A, P, Cout, 1);
    if (Cin != Cout) {
      if (rc) return;
      run(b2f_gemm_bf16(X, Cin, 0, w(name + ".conv_shortcut.weight"), Cin, w(name + ".conv_shortcut.bias"), B,
                        Cout, 0, 1, (int)(N * P), Cout, Cin, B2F_EPI_BIAS, nullptr, 0, 0, nullptr, 0, st));
      conv(name + ".conv2", A, X, B, H, W, Cout, Cout);
    } else {
      conv(name + ".conv2", A, X, X, H, W, Cout, Cout);
    }
  }
  // Attention(heads=1, residual) over the H*W tokens of each image, in place on X[N,P,C]
  void attention(const std::string& name, long long P, int C) {
    gn(name + ".group_norm", X, A, P, C, 0);
    if (rc) return;
    const bf16_t* wqkv = w(name + ".qkv.weight");
    const bf16_t* bqkv = w(name + ".qkv.bias");
    const bf16_t* wo = w(name + ".to_out.0.weight");
    const bf16_t* bo = w(name + ".to_out.0.bias");
    if (rc) return;
    // The scores stay in fp32 (diffusers' SDPA keeps them so; bf16 logits err by |s| 2^-9 in every exponent): S = Q K^T
    // is the weight-gradient GEMM of Q^T and K^T.  Queries, keys and values are padded to P8 pixels with zeros: the
    // softmax normalises [0, P) and zeroes [P, P8), and P V contracts over P8 against zero columns of V^T.
    const long long P8 = (P + 7) / 8 * 8;
    bf16_t* qkv = attn_ws;                          // [P, 3C]
    bf16_t* qT = qkv + P * 3 * C;                   // [C, P8] x 3: Q^T, K^T, V^T, columns [P, P8) zero
    bf16_t* kT = qT + (long long)C * P8;
    bf16_t* vT = kT + (long long)C * P8;
    bf16_t* S = vT + (long long)C * P8;             // [P, P8] bf16 probabilities
    float* Sf = reinterpret_cast<float*>(S + P * P8);  // [P8, P8] fp32 scores
    const float scale = 1.0f / sqrtf((float)C);
    if (P8 != P) run(cuda_err(cudaMemsetAsync(qT, 0, (size_t)3 * C * P8 * sizeof(bf16_t), st), "vae attn pad"));
    for (int n = 0; n < N && !rc; ++n) {
      bf16_t* xa = A + (long long)n * P * C;
      bf16_t* xx = X + (long long)n * P * C;
      run(b2f_gemm_bf16(xa, C, 0, wqkv, C, bqkv, qkv, 3 * C, 0, 1, (int)P, 3 * C, C, B2F_EPI_BIAS, nullptr, 0, 0,
                        nullptr, 0, st));
      run(b2f_transpose_bf16(qkv, 3 * C, qT, P8, (int)P, C, st));
      run(b2f_transpose_bf16(qkv + C, 3 * C, kT, P8, (int)P, C, st));
      run(b2f_transpose_bf16(qkv + 2 * C, 3 * C, vT, P8, (int)P, C, st));
      run(b2f_gemm_wgrad(qT, P8, 0, kT, P8, 0, Sf, P8, 1, C, (int)P8, (int)P8, 0, st));
      run(b2f_softmax_rows_f32(Sf, P8, S, P8, (int)P, (int)P, scale, st));
      run(b2f_gemm_bf16(S, P8, 0, vT, P8, nullptr, xa, C, 0, 1, (int)P, C, (int)P8, B2F_EPI_BIAS, nullptr, 0, 0,
                        nullptr, 0, st));
      run(b2f_gemm_bf16(xa, C, 0, wo, C, bo, xx, C, 0, 1, (int)P, C, C, B2F_EPI_RESID, xx, C, 0, nullptr, 0, st));
    }
  }
  // the mid block's three stages; true when the run stops inside it
  bool mid(const std::string& name, int H, int W, int C) {
    resnet(name + ".resnets.0", H, W, C, C);
    if (stage_done(H, W, C)) return true;
    attention(name + ".attentions.0", (long long)H * W, C);
    if (stage_done(H, W, C)) return true;
    resnet(name + ".resnets.1", H, W, C, C);
    return stage_done(H, W, C);
  }
  void swapXA() {
    bf16_t* t = X;
    X = A;
    A = t;
  }
};

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// bytes: 3 activation buffers of `act` elements + attention scratch + stats
static void ws_layout(const b2f_vae_cfg& g, int N, int H, int W, size_t* act_elems, size_t* attn_elems) {
  // largest NHWC activation: full resolution x block_out[0] channels, or (decoder) the upsampled
  // tensor entering the last upsample conv: full resolution x block_out[1]
  const size_t full = (size_t)N * H * W;
  size_t m = full * (size_t)(g.block_out[1] > g.block_out[0] ? g.block_out[1] : g.block_out[0]);
  if (m < full * 64) m = full * 64;
  *act_elems = m;
  const size_t P = (size_t)(H / 8) * (W / 8), P8 = (P + 7) / 8 * 8;
  const size_t C = g.block_out[3];
  // qkv, Q^T / K^T / V^T, bf16 probabilities and fp32 scores (two bf16 elements each)
  *attn_elems = P * 3 * C + 3 * C * P8 + P * P8 + 2 * P8 * P8;
}

}  // namespace b2f

using namespace b2f;

extern "C" {

int b2f_vae_create(b2f_vae** out, const b2f_vae_cfg* cfg) {
  if (!out || !cfg) return B2F_ERR_INVALID;
  for (int i = 0; i < 4; ++i)
    if (cfg->block_out[i] <= 0 || cfg->block_out[i] % 32) return B2F_ERR_UNSUPPORTED;
  if (cfg->block_out[0] % 64 && cfg->block_out[0] != 32) return B2F_ERR_UNSUPPORTED;
  if (cfg->latent_channels <= 0 || cfg->latent_channels > 64 || cfg->layers_per_block <= 0)
    return B2F_ERR_UNSUPPORTED;
  VaeCtx* c = new (std::nothrow) VaeCtx();
  if (!c) return B2F_ERR_INVALID;
  c->cfg = *cfg;
  *out = reinterpret_cast<b2f_vae*>(c);
  return B2F_OK;
}
void b2f_vae_destroy(b2f_vae* h) { delete reinterpret_cast<VaeCtx*>(h); }

int b2f_vae_bind_weight(b2f_vae* h, const char* key, const void* dptr, int64_t numel) {
  VaeCtx* c = reinterpret_cast<VaeCtx*>(h);
  if (!c || !key || !dptr || numel <= 0) return B2F_ERR_INVALID;
  if (reinterpret_cast<uintptr_t>(dptr) & 15) return B2F_ERR_ALIGN;
  c->bound[key] = {dptr, numel};
  return B2F_OK;
}

int b2f_vae_set_stop_stage(b2f_vae* h, int stage) {
  VaeCtx* c = reinterpret_cast<VaeCtx*>(h);
  if (!c || stage < 0) return B2F_ERR_INVALID;
  c->stop_stage = stage;
  return B2F_OK;
}

size_t b2f_vae_workspace_bytes(const b2f_vae* h, int N, int H, int W) {
  const VaeCtx* c = reinterpret_cast<const VaeCtx*>(h);
  if (!c || N <= 0 || H <= 0 || W <= 0) return 0;
  size_t act, attn;
  ws_layout(c->cfg, N, H, W, &act, &attn);
  return 3 * align_up(act * 2, 256) + align_up(attn * 2, 256) + align_up(sizeof(double) * 64 * N, 256) + 1024;
}

static int vae_setup(VaeCtx* c, VaeRun* r, int N, int H, int W, void* ws, size_t ws_bytes, cudaStream_t st) {
  if (ws_bytes < b2f_vae_workspace_bytes(reinterpret_cast<b2f_vae*>(c), N, H, W)) return B2F_ERR_WORKSPACE;
  size_t act, attn;
  ws_layout(c->cfg, N, H, W, &act, &attn);
  uint8_t* p = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~uintptr_t(255));
  const size_t ab = align_up(act * 2, 256);
  r->c = c;
  r->st = st;
  r->N = N;
  r->ws0 = reinterpret_cast<bf16_t*>(p);
  r->X = reinterpret_cast<bf16_t*>(p);
  r->A = reinterpret_cast<bf16_t*>(p + ab);
  r->B = reinterpret_cast<bf16_t*>(p + 2 * ab);
  r->attn_ws = reinterpret_cast<bf16_t*>(p + 3 * ab);
  r->stats = reinterpret_cast<double*>(p + 3 * ab + align_up(attn * 2, 256));
  return B2F_OK;
}

int b2f_vae_encode(b2f_vae* h, const void* image_nchw, int image_is_f32, int N, int H, int W,
                   void* moments_nchw, void* ws, size_t ws_bytes, b2f_stream_t stream_) {
  VaeCtx* c = reinterpret_cast<VaeCtx*>(h);
  if (!c || !image_nchw || !moments_nchw || !ws || N <= 0) return B2F_ERR_INVALID;
  if (H % 8 || W % 8 || H <= 0 || W <= 0) return B2F_ERR_UNSUPPORTED;
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  VaeRun r;
  int rc = vae_setup(c, &r, N, H, W, ws, ws_bytes, st);
  if (rc) return rc;
  const b2f_vae_cfg& g = c->cfg;
  r.run(b2f_nchw_to_nhwc_pad(image_nchw, image_is_f32, r.A, N, g.in_channels, H, W, 64, st));
  r.conv("encoder.conv_in", r.A, r.X, nullptr, H, W, 64, g.block_out[0]);
  int ch = g.block_out[0], hh = H, ww = W;
  if (r.stage_done(hh, ww, ch)) return r.rc;
  for (int i = 0; i < 4; ++i) {
    for (int j = 0; j < g.layers_per_block; ++j) {
      r.resnet("encoder.down_blocks." + std::to_string(i) + ".resnets." + std::to_string(j), hh, ww, ch,
               g.block_out[i]);
      ch = g.block_out[i];
      if (r.stage_done(hh, ww, ch)) return r.rc;
    }
    if (i != 3) {
      r.conv("encoder.down_blocks." + std::to_string(i) + ".downsamplers.0.conv", r.X, r.A, nullptr, hh, ww,
             ch, ch, 2);
      r.swapXA();
      hh /= 2;
      ww /= 2;
      if (r.stage_done(hh, ww, ch)) return r.rc;
    }
  }
  if (r.mid("encoder.mid_block", hh, ww, ch)) return r.rc;
  r.gn("encoder.conv_norm_out", r.X, r.A, (long long)hh * ww, ch, 1);
  r.conv("encoder.conv_out", r.A, static_cast<bf16_t*>(moments_nchw), nullptr, hh, ww, ch,
         2 * g.latent_channels, 1, 1);
  return r.rc;
}

static int vae_decode_impl(b2f_vae* h, const void* z_nchw, int N, int h_lat, int w_lat, void* image_nchw, int out_mode,
                           void* ws, size_t ws_bytes, b2f_stream_t stream_) {
  VaeCtx* c = reinterpret_cast<VaeCtx*>(h);
  if (!c || !z_nchw || !image_nchw || !ws || N <= 0 || h_lat <= 0 || w_lat <= 0) return B2F_ERR_INVALID;
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  const int H = h_lat * 8, W = w_lat * 8;
  VaeRun r;
  int rc = vae_setup(c, &r, N, H, W, ws, ws_bytes, st);
  if (rc) return rc;
  const b2f_vae_cfg& g = c->cfg;
  r.run(b2f_nchw_to_nhwc_pad(z_nchw, 0, r.A, N, g.latent_channels, h_lat, w_lat, 64, st));
  int ch = g.block_out[3], hh = h_lat, ww = w_lat;
  r.conv("decoder.conv_in", r.A, r.X, nullptr, hh, ww, 64, ch);
  if (r.stage_done(hh, ww, ch)) return r.rc;
  if (r.mid("decoder.mid_block", hh, ww, ch)) return r.rc;
  for (int i = 0; i < 4; ++i) {
    const int co = g.block_out[3 - i];
    for (int j = 0; j < g.layers_per_block + 1; ++j) {
      r.resnet("decoder.up_blocks." + std::to_string(i) + ".resnets." + std::to_string(j), hh, ww, ch, co);
      ch = co;
      if (r.stage_done(hh, ww, ch)) return r.rc;
    }
    if (i != 3) {
      r.run(b2f_upsample2x(r.X, r.A, N, hh, ww, ch, st));
      hh *= 2;
      ww *= 2;
      r.conv("decoder.up_blocks." + std::to_string(i) + ".upsamplers.0.conv", r.A, r.X, nullptr, hh, ww, ch, ch);
      if (r.stage_done(hh, ww, ch)) return r.rc;
    }
  }
  r.gn("decoder.conv_norm_out", r.X, r.A, (long long)hh * ww, ch, 1);
  r.conv("decoder.conv_out", r.A, static_cast<bf16_t*>(image_nchw), nullptr, hh, ww, ch, g.out_channels, 1, out_mode);
  return r.rc;
}

int b2f_vae_decode(b2f_vae* h, const void* z_nchw, int N, int h_lat, int w_lat, void* image_nchw,
                   void* ws, size_t ws_bytes, b2f_stream_t stream_) {
  return vae_decode_impl(h, z_nchw, N, h_lat, w_lat, image_nchw, 1, ws, ws_bytes, stream_);
}

int b2f_vae_decode_u8(b2f_vae* h, const void* z_nchw, int N, int h_lat, int w_lat, void* image_u8_nhwc,
                      void* ws, size_t ws_bytes, b2f_stream_t stream_) {
  return vae_decode_impl(h, z_nchw, N, h_lat, w_lat, image_u8_nhwc, 2, ws, ws_bytes, stream_);
}

}  // extern "C"
