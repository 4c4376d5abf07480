// First-block cache of the FLUX forward (b2f_flux_forward_cached; semantics and rounding points in include/b2f.h).
//
// One cached step:
//   flux_forward(0, 1) with the x0 copy-out   embedders + block 0; x0 = image rows of h before block 0
//   cache_residual_kernel                       r_k = y0 - x0 (fp32), y0 -> scratch, per-CTA partial sums
//   cache_dist_kernel                           dist = sum|r_k - r_prev| / sum|r_prev| in fixed order, decision
//   one 8-byte device -> host read of (dist, hit)
//   hit:  cache_apply_kernel (h' = bf16(y0 + R) in place) + flux_forward(nblk, nblk)    (the engine's own tail)
//   miss: flux_forward(1, nblk) + cache_capture_kernel (R = h_final - y0)
#include <cuda_bf16.h>

#include <cmath>
#include <new>

#include "flux_ctx.h"
#include "host_common.h"
#include "ptx.cuh"

namespace b2f {

namespace {

constexpr int kThreads = 256;
constexpr int kRowsPerCta = 8;   // rows of d elements per CTA of the residual pass: fixes the partials' order

// Fixed-shape tree over kThreads doubles in shared memory; the result lands in s[0].
__device__ __forceinline__ void tree_sum(double* s) {
#pragma unroll
  for (int w = kThreads / 2; w > 0; w >>= 1) {
    __syncthreads();
    if ((int)threadIdx.x < w) s[threadIdx.x] += s[threadIdx.x + w];
  }
  __syncthreads();
}

// rows = B * S_img image rows; row i = (b, s) lives at h + b * h_bs + s * d.  xy: [rows, d] bf16, x0 in, y0 out.
// r_prev may be null (no state): it reads as 0.
__global__ void __launch_bounds__(kThreads) cache_residual_kernel(const __nv_bfloat16* __restrict__ h, int64_t h_bs,
                                                                  int S_img, int rows, int d, __nv_bfloat16* xy,
                                                                  const float* __restrict__ r_prev,
                                                                  float* __restrict__ r_out,
                                                                  double* __restrict__ partials) {
  __shared__ double s_num[kThreads], s_den[kThreads];
  const int row0 = blockIdx.x * kRowsPerCta;
  const int nrow = min(kRowsPerCta, rows - row0);
  const int c8 = d >> 3;
  float num = 0.f, den = 0.f;
  for (int j = threadIdx.x; j < nrow * c8; j += kThreads) {
    const int i = row0 + j / c8, col = (j % c8) * 8;
    const int b = i / S_img, s = i % S_img;
    const int64_t o = (int64_t)i * d + col;
    const uint4 yu = *reinterpret_cast<const uint4*>(h + b * h_bs + (int64_t)s * d + col);
    const uint4 xu = *reinterpret_cast<const uint4*>(xy + o);
    float x[8], y[8], r[8], p[8];
    unpack8(xu, x);
    unpack8(yu, y);
    if (r_prev) {
      const float4 a = *reinterpret_cast<const float4*>(r_prev + o);
      const float4 c = *reinterpret_cast<const float4*>(r_prev + o + 4);
      p[0] = a.x, p[1] = a.y, p[2] = a.z, p[3] = a.w, p[4] = c.x, p[5] = c.y, p[6] = c.z, p[7] = c.w;
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) p[k] = 0.f;
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      r[k] = __fsub_rn(y[k], x[k]);
      num = __fadd_rn(num, fabsf(__fsub_rn(r[k], p[k])));
      den = __fadd_rn(den, fabsf(p[k]));
    }
    *reinterpret_cast<float4*>(r_out + o) = make_float4(r[0], r[1], r[2], r[3]);
    *reinterpret_cast<float4*>(r_out + o + 4) = make_float4(r[4], r[5], r[6], r[7]);
    *reinterpret_cast<uint4*>(xy + o) = yu;
  }
  s_num[threadIdx.x] = num;
  s_den[threadIdx.x] = den;
  tree_sum(s_num);
  tree_sum(s_den);
  if (threadIdx.x == 0) {
    partials[2 * blockIdx.x] = s_num[0];
    partials[2 * blockIdx.x + 1] = s_den[0];
  }
}

struct Decision {
  float dist;
  int hit;
};

// One CTA: thread t sums partials t, t + 256, ... in index order (fp64), then the fixed tree.
__global__ void __launch_bounds__(kThreads) cache_dist_kernel(const double* __restrict__ partials, int n,
                                                              float threshold, Decision* __restrict__ dec) {
  __shared__ double s_num[kThreads], s_den[kThreads];
  double num = 0.0, den = 0.0;
  for (int c = threadIdx.x; c < n; c += kThreads) {
    num += partials[2 * c];
    den += partials[2 * c + 1];
  }
  s_num[threadIdx.x] = num;
  s_den[threadIdx.x] = den;
  tree_sum(s_num);
  tree_sum(s_den);
  if (threadIdx.x == 0) {
    const double q = s_num[0] / s_den[0];
    const float dist = (float)q;
    dec->dist = dist;
    // strict: threshold 0 never hits; NaN / inf dist and sum|r_prev| == 0 are misses
    dec->hit = (s_den[0] > 0.0 && isfinite(dist) && dist < threshold) ? 1 : 0;
  }
}

// h'[b, s] = bf16(float(h[b, s]) + R[b, s]) for the first n_out image rows of every batch item, in place.
__global__ void __launch_bounds__(kThreads) cache_apply_kernel(__nv_bfloat16* h, int64_t h_bs, int n_out, int d,
                                                               const float* __restrict__ R, int64_t n8) {
  const int c8 = d >> 3;
  for (int64_t j = blockIdx.x * (int64_t)kThreads + threadIdx.x; j < n8; j += (int64_t)gridDim.x * kThreads) {
    const int64_t i = j / c8;
    const int col = (int)(j % c8) * 8;
    const int64_t b = i / n_out, s = i % n_out;
    uint4* hp = reinterpret_cast<uint4*>(h + b * h_bs + s * d + col);
    float y[8];
    unpack8(*hp, y);
    const float4 a = *reinterpret_cast<const float4*>(R + i * d + col);
    const float4 c = *reinterpret_cast<const float4*>(R + i * d + col + 4);
    const float r[8] = {a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w};
    uint4 o;
    __nv_bfloat162* op = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
    for (int k = 0; k < 4; ++k)
      op[k] = __floats2bfloat162_rn(__fadd_rn(y[2 * k], r[2 * k]), __fadd_rn(y[2 * k + 1], r[2 * k + 1]));
    *hp = o;
  }
}

// R[b, s] = float(h[b, s]) - float(y0[b, s]) for the first n_out image rows; y0: [B, S_img, d].
__global__ void __launch_bounds__(kThreads) cache_capture_kernel(const __nv_bfloat16* __restrict__ h, int64_t h_bs,
                                                                 const __nv_bfloat16* __restrict__ y0, int S_img,
                                                                 int n_out, int d, float* __restrict__ R, int64_t n8) {
  const int c8 = d >> 3;
  for (int64_t j = blockIdx.x * (int64_t)kThreads + threadIdx.x; j < n8; j += (int64_t)gridDim.x * kThreads) {
    const int64_t i = j / c8;
    const int col = (int)(j % c8) * 8;
    const int64_t b = i / n_out, s = i % n_out;
    float f[8], y[8];
    unpack8(*reinterpret_cast<const uint4*>(h + b * h_bs + s * d + col), f);
    unpack8(*reinterpret_cast<const uint4*>(y0 + (b * S_img + s) * d + col), y);
    float r[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) r[k] = __fsub_rn(f[k], y[k]);
    *reinterpret_cast<float4*>(R + i * d + col) = make_float4(r[0], r[1], r[2], r[3]);
    *reinterpret_cast<float4*>(R + i * d + col + 4) = make_float4(r[4], r[5], r[6], r[7]);
  }
}

// The regions of a cache's memory for one shape, in the order include/b2f.h documents.
struct Layout {
  size_t r[2], R, partials, dec, xy, end;
  int ctas;
};
Layout layout_of(int64_t d, int B, int S_img, int n_out) {
  Layout L;
  const size_t N = (size_t)B * S_img * d;
  L.ctas = (int)(((int64_t)B * S_img + kRowsPerCta - 1) / kRowsPerCta);
  L.r[0] = 0;
  L.r[1] = al256(N * 4);
  L.R = L.r[1] + al256(N * 4);
  L.partials = L.R + al256((size_t)B * n_out * d * 4);
  L.dec = L.partials + al256((size_t)L.ctas * 16);
  L.xy = L.dec + 256;
  L.end = L.xy + al256(N * 2);
  return L;
}

int grid_for(int64_t n8) { return (int)std::min<int64_t>((n8 + kThreads - 1) / kThreads, 132 * 16); }

}  // namespace

struct FluxCache {
  char* mem = nullptr;   // 256-aligned start of the caller's memory
  size_t bytes = 0;      // usable bytes from mem
  Decision* host = nullptr;
  const FluxCtx* ctx = nullptr;
  bool valid = false;
  int B = 0, S_img = 0, S_txt = 0, n_out = 0;
  int slot = 0;          // slot of r holding r_prev
};

}  // namespace b2f

using namespace b2f;

extern "C" {

size_t b2f_flux_cache_bytes(const b2f_flux* h, int B, int S_img, int S_txt, int n_out_rows) {
  const FluxCtx* c = reinterpret_cast<const FluxCtx*>(h);
  if (!c || B <= 0 || S_img <= 0 || S_txt <= 0 || n_out_rows <= 0 || n_out_rows > S_img) return 0;
  return layout_of(c->d, B, S_img, n_out_rows).end + 256;
}

int b2f_flux_cache_create(b2f_flux_cache** out, void* mem, size_t bytes) {
  if (!out || !mem) return B2F_ERR_INVALID;
  const uintptr_t p = reinterpret_cast<uintptr_t>(mem), a = al256(p);
  if (bytes < a - p + 256) return B2F_ERR_WORKSPACE;
  FluxCache* c = new (std::nothrow) FluxCache();
  if (!c) return B2F_ERR_INVALID;
  int rc = cuda_err(cudaMallocHost(&c->host, sizeof(Decision)), "flux_cache_create: cudaMallocHost");
  if (rc) {
    delete c;
    return rc;
  }
  c->mem = reinterpret_cast<char*>(a);
  c->bytes = bytes - (a - p);
  *out = reinterpret_cast<b2f_flux_cache*>(c);
  return B2F_OK;
}

void b2f_flux_cache_destroy(b2f_flux_cache* cache) {
  FluxCache* c = reinterpret_cast<FluxCache*>(cache);
  if (!c) return;
  cudaFreeHost(c->host);
  delete c;
}

int b2f_flux_cache_reset(b2f_flux_cache* cache) {
  FluxCache* c = reinterpret_cast<FluxCache*>(cache);
  if (!c) return B2F_ERR_INVALID;
  c->valid = false;
  return B2F_OK;
}

int b2f_flux_cache_state(const b2f_flux_cache* cache, int* valid, int* r_slot) {
  const FluxCache* c = reinterpret_cast<const FluxCache*>(cache);
  if (!c || !valid || !r_slot) return B2F_ERR_INVALID;
  *valid = c->valid ? 1 : 0;
  *r_slot = c->slot;
  return B2F_OK;
}

int b2f_flux_forward_cached(b2f_flux* h, b2f_flux_cache* cache, float threshold, const void* hidden, const void* enc,
                            const void* mod, int64_t mod_ld, void* out, int B, int S_img, int S_txt, int n_out_rows,
                            void* ws, size_t ws_bytes, int* hit, float* dist, b2f_stream_t stream_) {
  FluxCtx* c = reinterpret_cast<FluxCtx*>(h);
  FluxCache* k = reinterpret_cast<FluxCache*>(cache);
  if (!c || !c->finalized || !k || !hit || !dist) return B2F_ERR_INVALID;
  if (!(threshold >= 0.f)) {   // negative or NaN
    fprintf(stderr, "[b2f] flux_forward_cached: threshold must be >= 0 (got %g)\n", (double)threshold);
    return B2F_ERR_INVALID;
  }
  if (B <= 0 || S_img <= 0 || S_txt <= 0 || n_out_rows <= 0 || n_out_rows > S_img) return B2F_ERR_INVALID;
  const size_t need = b2f_flux_cache_bytes(h, B, S_img, S_txt, n_out_rows);
  if (k->bytes < need - 256) return B2F_ERR_WORKSPACE;
  if (ws_bytes < b2f_flux_workspace_bytes(h, B, S_img, S_txt)) return B2F_ERR_WORKSPACE;
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  if (!device_info().ok) return B2F_ERR_NODEVICE;

  const int64_t d = c->d;
  const int S = S_img + S_txt, nblk = c->cfg.num_double + c->cfg.num_single;
  const Layout L = layout_of(d, B, S_img, n_out_rows);
  float* r[2] = {reinterpret_cast<float*>(k->mem + L.r[0]), reinterpret_cast<float*>(k->mem + L.r[1])};
  float* R = reinterpret_cast<float*>(k->mem + L.R);
  double* partials = reinterpret_cast<double*>(k->mem + L.partials);
  Decision* dec = reinterpret_cast<Decision*>(k->mem + L.dec);
  bf16_t* xy = reinterpret_cast<bf16_t*>(k->mem + L.xy);
  // the image rows of b2f_flux_forward's h[B, S, d]
  __nv_bfloat16* h_img = reinterpret_cast<__nv_bfloat16*>(fwd_ws(c, ws, B, S_img, S_txt).h + (int64_t)S_txt * d);
  const int64_t h_bs = (int64_t)S * d;

  const bool valid = k->valid && k->ctx == c && k->B == B && k->S_img == S_img && k->S_txt == S_txt &&
                     k->n_out == n_out_rows;
  if (!valid) k->valid = false;
  int rc;
  // head: embedders, the copy of x0, block 0
  if ((rc = flux_forward(c, hidden, enc, mod, mod_ld, out, B, S_img, S_txt, n_out_rows, ws, ws_bytes, 0, 1, xy, st)))
    return rc;
  const int cur = valid ? 1 - k->slot : k->slot;   // the slot r_k goes to
  const int rows = B * S_img;
  cache_residual_kernel<<<L.ctas, kThreads, 0, st>>>(h_img, h_bs, S_img, rows, (int)d,
                                                     reinterpret_cast<__nv_bfloat16*>(xy),
                                                     valid ? r[k->slot] : nullptr, r[cur], partials);
  B2F_LAUNCHED("cache_residual_kernel", 1);
  Decision dh{NAN, 0};
  if (valid) {
    cache_dist_kernel<<<1, kThreads, 0, st>>>(partials, L.ctas, threshold, dec);
    B2F_LAUNCHED("cache_dist_kernel", 1);
    if ((rc = cuda_err(cudaMemcpyAsync(k->host, dec, sizeof(Decision), cudaMemcpyDeviceToHost, st),
                       "flux_forward_cached: decision read")))
      return rc;
    if ((rc = cuda_err(cudaStreamSynchronize(st), "flux_forward_cached: decision wait"))) return rc;
    dh = *k->host;
  }
  const int64_t n8 = (int64_t)B * n_out_rows * d / 8;
  if (dh.hit) {
    cache_apply_kernel<<<grid_for(n8), kThreads, 0, st>>>(h_img, h_bs, n_out_rows, (int)d, R, n8);
    B2F_LAUNCHED("cache_apply_kernel", 1);
    if ((rc = flux_forward(c, hidden, enc, mod, mod_ld, out, B, S_img, S_txt, n_out_rows, ws, ws_bytes, nblk, nblk,
                           nullptr, st)))
      return rc;
  } else {
    if ((rc = flux_forward(c, hidden, enc, mod, mod_ld, out, B, S_img, S_txt, n_out_rows, ws, ws_bytes, 1, nblk,
                           nullptr, st)))
      return rc;
    cache_capture_kernel<<<grid_for(n8), kThreads, 0, st>>>(h_img, h_bs, reinterpret_cast<const __nv_bfloat16*>(xy),
                                                            S_img, n_out_rows, (int)d, R, n8);
    B2F_LAUNCHED("cache_capture_kernel", 1);
    k->slot = cur;
    k->valid = true;
    k->ctx = c;
    k->B = B;
    k->S_img = S_img;
    k->S_txt = S_txt;
    k->n_out = n_out_rows;
  }
  *hit = dh.hit;
  *dist = dh.dist;
  return B2F_OK;
}

}  // extern "C"
