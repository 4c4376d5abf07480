// HBM-bound kernels of the Qwen2.5-VL conditioning prefill (ViT + text decoder), bf16.
// They restate the torch-eager chains of transformers' Qwen2_5_VL modules (SURVEY.md Appendix B;
// reference call site univa/models/qwen2p5vl/modeling_univa_qwen2p5vl.py:373-399, 481-492) with the
// same bf16 rounding points.
#include "host_common.h"
#include "ptx.cuh"

namespace b2f {

namespace {

__device__ __forceinline__ void unpack8l(const uint4& q, float* f) {
  const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 t = unpack_bf16x2(w[j]);
    f[2 * j] = t.x;
    f[2 * j + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 pack8l(const float* f) {
  uint4 q;
  q.x = pack_bf16x2(f[0], f[1]);
  q.y = pack_bf16x2(f[2], f[3]);
  q.z = pack_bf16x2(f[4], f[5]);
  q.w = pack_bf16x2(f[6], f[7]);
  return q;
}

// Qwen2RMSNorm: y = w * bf16(x_f32 * rsqrt(mean(x^2) + eps)); one warp per row, D % 256 == 0.
template <int MAXC>
__global__ void __launch_bounds__(128) rmsnorm_kernel(const __nv_bfloat16* x, long long ldx,
                                                      const __nv_bfloat16* w, __nv_bfloat16* y,
                                                      long long ldy, long long rows, int D, float eps) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long r = (long long)blockIdx.x * 4 + warp;
  if (r >= rows) return;
  const int nchunk = D >> 8;
  float v[MAXC][8];
  float ss = 0.f;
#pragma unroll
  for (int c = 0; c < MAXC; ++c)
    if (c < nchunk) {
      unpack8l(*reinterpret_cast<const uint4*>(x + r * ldx + c * 256 + lane * 8), v[c]);
#pragma unroll
      for (int j = 0; j < 8; ++j) ss += v[c][j] * v[c][j];
    }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float rs = rsqrtf(ss / (float)D + eps);
#pragma unroll
  for (int c = 0; c < MAXC; ++c)
    if (c < nchunk) {
      float g[8], o[8];
      unpack8l(__ldg(reinterpret_cast<const uint4*>(w + c * 256 + lane * 8)), g);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = g[j] * bf16r(v[c][j] * rs);
      *reinterpret_cast<uint4*>(y + r * ldy + c * 256 + lane * 8) = pack8l(o);
    }
}

// rotate-half RoPE in place on `heads` vectors per token: x <- x*cos + rotate_half(x)*sin over the
// first `rot` elements of each head slot of pitch `head_pitch` (rot <= 128, even).
//   fp32_math = 1 (vision): one rounding.   fp32_math = 0 (text, M-RoPE): every product and the sum
//   are rounded to bf16, cos/sin are bf16 values — the eager bf16 chain of apply_multimodal_rotary_pos_emb.
__global__ void __launch_bounds__(256) rope_half_kernel(__nv_bfloat16* x, long long ld, int heads,
                                                        int head_pitch, const float* cos,
                                                        const float* sin, int rot, long long tokens,
                                                        int fp32_math) {
  const long long idx = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);  // (token, head)
  const int lane = threadIdx.x & 31;
  if (idx >= tokens * heads) return;
  const long long t = idx / heads;
  const int h = int(idx - t * heads);
  __nv_bfloat16* p = x + t * ld + (long long)h * head_pitch;
  const int half = rot >> 1;
  for (int i = lane; i < half; i += 32) {
    const float a = __bfloat162float(p[i]), b = __bfloat162float(p[i + half]);
    const float c0 = cos[t * rot + i], s0 = sin[t * rot + i];
    const float c1 = cos[t * rot + i + half], s1 = sin[t * rot + i + half];
    float o0, o1;
    if (fp32_math) {
      o0 = a * c0 - b * s0;
      o1 = b * c1 + a * s1;
    } else {
      o0 = bf16r(a * c0) + bf16r(-b * s0);
      o1 = bf16r(b * c1) + bf16r(a * s1);
    }
    p[i] = __float2bfloat16_rn(o0);
    p[i + half] = __float2bfloat16_rn(o1);
  }
}

// SwiGLU combine: out = bf16( bf16(silu(g)) * u ), g = gu[:, :I], u = gu[:, I:2I]
__global__ void __launch_bounds__(256) swiglu_kernel(const __nv_bfloat16* gu, long long ld,
                                                     __nv_bfloat16* out, long long ldo, long long rows,
                                                     int I) {
  const int vec = I >> 3;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * vec) return;
  const long long r = i / vec;
  const int c = int(i - r * vec) * 8;
  float g[8], u[8], o[8];
  unpack8l(*reinterpret_cast<const uint4*>(gu + r * ld + c), g);
  unpack8l(*reinterpret_cast<const uint4*>(gu + r * ld + I + c), u);
#pragma unroll
  for (int j = 0; j < 8; ++j) o[j] = bf16r(g[j] / (1.0f + __expf(-g[j]))) * u[j];
  *reinterpret_cast<uint4*>(out + r * ldo + c) = pack8l(o);
}

// out[i, :] = table[idx[i], :]   (gather)   or   out[idx[i], :] = src[i, :]   (scatter)
__global__ void __launch_bounds__(256) move_rows_kernel(const __nv_bfloat16* src, long long ld_src,
                                                        __nv_bfloat16* dst, long long ld_dst,
                                                        const long long* idx, long long n, int D,
                                                        int scatter) {
  const int vec = D >> 3;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * vec) return;
  const long long r = i / vec;
  const int c = int(i - r * vec) * 8;
  const long long j = idx[r];
  if (scatter)
    *reinterpret_cast<uint4*>(dst + j * ld_dst + c) = *reinterpret_cast<const uint4*>(src + r * ld_src + c);
  else
    *reinterpret_cast<uint4*>(dst + r * ld_dst + c) = *reinterpret_cast<const uint4*>(src + j * ld_src + c);
}

// T5 gated-GELU combine (T5DenseGatedActDense with gelu_new): out = bf16( bf16(gelu_tanh(g)) * u ),
// g = gu[:, :I] (wi_0 x), u = gu[:, I:2I] (wi_1 x).
__global__ void __launch_bounds__(256) geglu_kernel(const __nv_bfloat16* gu, long long ld,
                                                    __nv_bfloat16* out, long long ldo, long long rows,
                                                    int I) {
  const int vec = I >> 3;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * vec) return;
  const long long r = i / vec;
  const int c = int(i - r * vec) * 8;
  float g[8], u[8], o[8];
  unpack8l(*reinterpret_cast<const uint4*>(gu + r * ld + c), g);
  unpack8l(*reinterpret_cast<const uint4*>(gu + r * ld + I + c), u);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float x = g[j];
    const float t = tanhf(0.7978845608028654f * (x + 0.044715f * x * x * x));
    o[j] = bf16r(0.5f * x * (1.0f + t)) * u[j];
  }
  *reinterpret_cast<uint4*>(out + r * ldo + c) = pack8l(o);
}

// nn.LayerNorm with affine weight and bias (CLIP text encoder): fp32 statistics, one rounding.
template <int MAXC>
__global__ void __launch_bounds__(128) layernorm_kernel(const __nv_bfloat16* x, long long ldx,
                                                        const __nv_bfloat16* w, const __nv_bfloat16* b,
                                                        __nv_bfloat16* y, long long ldy, long long rows,
                                                        int D, float eps) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long r = (long long)blockIdx.x * 4 + warp;
  if (r >= rows) return;
  const int nchunk = D >> 8;
  float v[MAXC][8];
  float sum = 0.f;
#pragma unroll
  for (int c = 0; c < MAXC; ++c)
    if (c < nchunk) {
      unpack8l(*reinterpret_cast<const uint4*>(x + r * ldx + c * 256 + lane * 8), v[c]);
#pragma unroll
      for (int j = 0; j < 8; ++j) sum += v[c][j];
    }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / (float)D;
  float ss = 0.f;
#pragma unroll
  for (int c = 0; c < MAXC; ++c)
    if (c < nchunk) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = v[c][j] - mean;
        ss += d * d;
      }
    }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float rs = rsqrtf(ss / (float)D + eps);
#pragma unroll
  for (int c = 0; c < MAXC; ++c)
    if (c < nchunk) {
      float g[8], bb[8], o[8];
      unpack8l(__ldg(reinterpret_cast<const uint4*>(w + c * 256 + lane * 8)), g);
      unpack8l(__ldg(reinterpret_cast<const uint4*>(b + c * 256 + lane * 8)), bb);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (v[c][j] - mean) * rs * g[j] + bb[j];
      *reinterpret_cast<uint4*>(y + r * ldy + c * 256 + lane * 8) = pack8l(o);
    }
}

// out[i, :] = bf16(tok[ids[i], :] + pos[i % period, :])  (CLIPTextEmbeddings); pos may be null (T5 `shared`)
__global__ void __launch_bounds__(256) embed_kernel(const __nv_bfloat16* tok, long long ld_tok,
                                                    const long long* ids, const __nv_bfloat16* pos,
                                                    long long ld_pos, int period, __nv_bfloat16* out,
                                                    long long ldo, long long n, int D) {
  const int vec = D >> 3;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * vec) return;
  const long long r = i / vec;
  const int c = int(i - r * vec) * 8;
  float a[8];
  unpack8l(*reinterpret_cast<const uint4*>(tok + ids[r] * ld_tok + c), a);
  if (pos) {
    float b[8];
    unpack8l(*reinterpret_cast<const uint4*>(pos + (r % period) * ld_pos + c), b);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] += b[j];
  }
  *reinterpret_cast<uint4*>(out + r * ldo + c) = pack8l(a);
}

}  // namespace

extern "C" int b2f_rmsnorm(const void* x, int64_t ldx, const void* w, void* y, int64_t ldy, int64_t rows, int D,
                           float eps, b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (!x || !w || !y || rows <= 0) return B2F_ERR_INVALID;
  if (D <= 0 || (D & 255) || D > 5120) return B2F_ERR_UNSUPPORTED;
  if ((ldx & 7) || (ldy & 7)) return B2F_ERR_ALIGN;
  const unsigned grid = (unsigned)((rows + 3) / 4);
  auto X = static_cast<const __nv_bfloat16*>(x);
  auto W = static_cast<const __nv_bfloat16*>(w);
  auto Y = static_cast<__nv_bfloat16*>(y);
  if (D <= 1280)
    rmsnorm_kernel<5><<<grid, 128, 0, stream>>>(X, ldx, W, Y, ldy, rows, D, eps);
  else if (D <= 3584)
    rmsnorm_kernel<14><<<grid, 128, 0, stream>>>(X, ldx, W, Y, ldy, rows, D, eps);
  else
    rmsnorm_kernel<20><<<grid, 128, 0, stream>>>(X, ldx, W, Y, ldy, rows, D, eps);
  B2F_LAUNCHED("rmsnorm_kernel", 1);
  return B2F_OK;
}

extern "C" int b2f_rope_half(void* x, int64_t ld, int heads, int head_pitch, const float* cos, const float* sin,
                             int rot, int64_t tokens, int fp32_math, b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (!x || !cos || !sin || heads <= 0 || tokens <= 0 || rot <= 0 || (rot & 1) || rot > head_pitch)
    return B2F_ERR_INVALID;
  const long long total = tokens * heads;
  rope_half_kernel<<<(unsigned)((total + 7) / 8), 256, 0, stream>>>(
      static_cast<__nv_bfloat16*>(x), ld, heads, head_pitch, cos, sin, rot, tokens, fp32_math);
  B2F_LAUNCHED("rope_half_kernel", 1);
  return B2F_OK;
}

extern "C" int b2f_swiglu(const void* gu, int64_t ld, void* out, int64_t ldo, int64_t rows, int I,
                          b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (!gu || !out || rows <= 0 || I <= 0 || (I & 7) || (ld & 7) || (ldo & 7)) return B2F_ERR_INVALID;
  const long long n = rows * (I >> 3);
  swiglu_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(gu), ld, static_cast<__nv_bfloat16*>(out), ldo, rows, I);
  B2F_LAUNCHED("swiglu_kernel", 1);
  return B2F_OK;
}

extern "C" int b2f_move_rows(const void* src, int64_t ld_src, void* dst, int64_t ld_dst, const int64_t* idx, int64_t n,
                             int D, int scatter, b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (!src || !dst || !idx || n <= 0 || D <= 0 || (D & 7) || (ld_src & 7) || (ld_dst & 7))
    return B2F_ERR_INVALID;
  const long long tot = n * (D >> 3);
  move_rows_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(src), ld_src, static_cast<__nv_bfloat16*>(dst), ld_dst,
      reinterpret_cast<const long long*>(idx), n, D, scatter);
  B2F_LAUNCHED("move_rows_kernel", 1);
  return B2F_OK;
}

extern "C" int b2f_geglu(const void* gu, int64_t ld, void* out, int64_t ldo, int64_t rows, int I,
                         b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (!gu || !out || rows <= 0 || I <= 0 || (I & 7) || (ld & 7) || (ldo & 7)) return B2F_ERR_INVALID;
  const long long n = rows * (I >> 3);
  geglu_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(gu), ld, static_cast<__nv_bfloat16*>(out), ldo, rows, I);
  B2F_LAUNCHED("geglu_kernel", 1);
  return B2F_OK;
}

extern "C" int b2f_layernorm(const void* x, int64_t ldx, const void* w, const void* b, void* y, int64_t ldy,
                             int64_t rows, int D, float eps, b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (!x || !w || !b || !y || rows <= 0) return B2F_ERR_INVALID;
  if (D <= 0 || (D & 255) || D > 5120) return B2F_ERR_UNSUPPORTED;
  if ((ldx & 7) || (ldy & 7)) return B2F_ERR_ALIGN;
  const unsigned grid = (unsigned)((rows + 3) / 4);
  auto X = static_cast<const __nv_bfloat16*>(x);
  auto W = static_cast<const __nv_bfloat16*>(w);
  auto Bv = static_cast<const __nv_bfloat16*>(b);
  auto Y = static_cast<__nv_bfloat16*>(y);
  if (D <= 1280)
    layernorm_kernel<5><<<grid, 128, 0, stream>>>(X, ldx, W, Bv, Y, ldy, rows, D, eps);
  else
    layernorm_kernel<20><<<grid, 128, 0, stream>>>(X, ldx, W, Bv, Y, ldy, rows, D, eps);
  B2F_LAUNCHED("layernorm_kernel", 1);
  return B2F_OK;
}

extern "C" int b2f_embed(const void* tok, int64_t ld_tok, const int64_t* ids, const void* pos, int64_t ld_pos,
                         int period, void* out, int64_t ldo, int64_t n, int D, b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (!tok || !ids || !out || n <= 0 || D <= 0 || (D & 7) || (ld_tok & 7) || (ldo & 7)) return B2F_ERR_INVALID;
  if (pos && (period <= 0 || (ld_pos & 7))) return B2F_ERR_INVALID;
  const long long tot = n * (D >> 3);
  embed_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(tok), ld_tok, reinterpret_cast<const long long*>(ids),
      static_cast<const __nv_bfloat16*>(pos), ld_pos, period > 0 ? period : 1,
      static_cast<__nv_bfloat16*>(out), ldo, n, D);
  B2F_LAUNCHED("embed_kernel", 1);
  return B2F_OK;
}

}  // namespace b2f
