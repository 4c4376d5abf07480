// HBM-bound kernels of the FLUX VAE (diffusers AutoencoderKL, SURVEY.md A.4), NHWC bf16:
//   GroupNorm(32 groups, eps, affine) [+ SiLU]  — statistics pass + apply pass
//   nearest 2x upsample, NCHW -> NHWC channel-padded import, row softmax and a bf16 transpose
//   (the last two serve the single-head dh=512 mid-block attention, run as GEMMs).
#include "host_common.h"
#include "ptx.cuh"

namespace b2f {

namespace {

// ---------------------------------------------------------------- GroupNorm statistics
// x: [N, P, C] (P = H*W pixels).  stats: double [N, 32, 2] (sum, sum of squares), zeroed by caller.
// Thread t of a block owns the channel octet (t % (C/8)) and strides over pixels; per-thread fp32
// partials over <= PIX_PER_BLOCK/threads-per-octet pixels, then shared + global double atomics.
constexpr int GN_THREADS = 256;
constexpr int GN_PIX_PER_BLOCK = 512;

__global__ void __launch_bounds__(GN_THREADS) gn_stats_kernel(const __nv_bfloat16* x, double* stats,
                                                              long long P, int C) {
  // Per-thread partial sums go through shared memory and are combined in a FIXED order by one thread per group:
  // with fp32 shared-memory atomics the block sums depended on the arrival order, E[x^2] - mean^2 amplified the
  // last-bit differences, and the VAE (hence the whole edit) was not bit-reproducible run to run.
  __shared__ float part[GN_THREADS][17];
  const int n = blockIdx.y;
  const int octets = C >> 3;
  const int oct = threadIdx.x % octets;
  const int prow = threadIdx.x / octets;
  const int rows_per_iter = GN_THREADS / octets;
  const long long p0 = (long long)blockIdx.x * GN_PIX_PER_BLOCK;
  const long long p1 = min(P, p0 + GN_PIX_PER_BLOCK);
  float s[8] = {0, 0, 0, 0, 0, 0, 0, 0}, q[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  const __nv_bfloat16* base = x + ((long long)n * P) * C + oct * 8;
  if (prow < rows_per_iter) {
    for (long long pp = p0 + prow; pp < p1; pp += rows_per_iter) {
      float f[8];
      unpack8(*reinterpret_cast<const uint4*>(base + pp * C), f);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        s[j] += f[j];
        q[j] += f[j] * f[j];
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    part[threadIdx.x][j] = s[j];
    part[threadIdx.x][8 + j] = q[j];
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    const int cpg = C / 32;  // channels per group: 4, 8 or 16 (1 or 2 for toy widths)
    double a = 0.0, b = 0.0;
    for (int c = threadIdx.x * cpg; c < (threadIdx.x + 1) * cpg; ++c) {
      const int o = c >> 3, j = c & 7;
      for (int r = 0; r < rows_per_iter; ++r) {
        a += (double)part[r * octets + o][j];
        b += (double)part[r * octets + o][8 + j];
      }
    }
    // across blocks: double atomics (order-dependent only at the 1e-16 level)
    atomicAdd(&stats[((long long)n * 32 + threadIdx.x) * 2 + 0], a);
    atomicAdd(&stats[((long long)n * 32 + threadIdx.x) * 2 + 1], b);
  }
}

// y = silu?( bf16( (x - mean) * rstd * gamma + beta ) )   (torch GroupNorm on bf16 rounds to bf16
// before the SiLU module runs)
__global__ void __launch_bounds__(256) gn_apply_kernel(const __nv_bfloat16* x, const double* stats,
                                                       const __nv_bfloat16* gamma,
                                                       const __nv_bfloat16* beta, __nv_bfloat16* y,
                                                       long long P, int C, float eps, int silu) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // octet index
  const int octets = C >> 3;
  const int n = blockIdx.y;
  if (i >= P * octets) return;
  const int oct = int(i % octets);
  const int cpg = C / 32;
  const double cnt = (double)P * cpg;
  float f[8], ga[8], be[8], o[8];
  const long long off = ((long long)n * P) * C + i * 8;
  unpack8(*reinterpret_cast<const uint4*>(x + off), f);
  unpack8(__ldg(reinterpret_cast<const uint4*>(gamma + oct * 8)), ga);
  unpack8(__ldg(reinterpret_cast<const uint4*>(beta + oct * 8)), be);
  // an octet of channels touches at most 8/cpg groups (one for the real widths, cpg >= 8, two for
  // cpg = 4): derive mean / rstd once per distinct group, in double, then stay in fp32
  int g_prev = -1;
  float mean = 0.f, rstd = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int g = (oct * 8 + j) / cpg;
    if (g != g_prev) {
      const double sm = stats[((long long)n * 32 + g) * 2], sq = stats[((long long)n * 32 + g) * 2 + 1];
      const double md = sm / cnt;
      mean = (float)md;
      rstd = rsqrtf((float)fmax(sq / cnt - md * md, 0.0) + eps);
      g_prev = g;
    }
    float v = bf16r((f[j] - mean) * rstd * ga[j] + be[j]);
    if (silu) v = v / (1.0f + __expf(-v));
    o[j] = v;
  }
  *reinterpret_cast<uint4*>(y + off) = pack8(o);
}

// ---------------------------------------------------------------- nearest 2x upsample (NHWC)
__global__ void __launch_bounds__(256) upsample2x_kernel(const uint4* in, uint4* out, int N, int H,
                                                         int W, int C8) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)N * (2 * H) * (2 * W) * C8;
  if (i >= total) return;
  const int c = int(i % C8);
  long long r = i / C8;
  const int x = int(r % (2 * W));
  r /= (2 * W);
  const int y = int(r % (2 * H));
  const int n = int(r / (2 * H));
  out[i] = in[(((long long)n * H + (y >> 1)) * W + (x >> 1)) * C8 + c];
}

// ---------------------------------------------------------------- NCHW (bf16 or fp32) -> NHWC bf16, channels zero-padded to Cpad
template <typename T>
__global__ void __launch_bounds__(256) nchw_to_nhwc_pad_kernel(const T* in, __nv_bfloat16* out, int N,
                                                               int C, int H, int W, int Cpad) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // (n, y, x, octet)
  const int oc = Cpad >> 3;
  const long long total = (long long)N * H * W * oc;
  if (i >= total) return;
  const int o = int(i % oc);
  const long long pix = i / oc;
  const long long hw = (long long)H * W;
  const int n = int(pix / hw);
  const long long p = pix - (long long)n * hw;
  float f[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = o * 8 + j;
    f[j] = c < C ? (float)in[((long long)n * C + c) * hw + p] : 0.f;
  }
  reinterpret_cast<uint4*>(out)[i] = pack8(f);
}

// uint8 NHWC [N, H, W, C] image -> NHWC bf16 in [-1, 1], channels zero-padded to Cpad: the reference's host-side
// `torch.tensor(np.array(img), float32) / 255.0`, `(x - 0.5) / 0.5` and `.to(bf16)` (univa/serve/cli.py:99-116,
// flux_pipeline.py:674) in the kernel that feeds encoder.conv_in — same fp32 operations, one rounding.
__global__ void __launch_bounds__(256) u8_nhwc_to_nhwc_pad_kernel(const uint8_t* in, __nv_bfloat16* out, long long npix,
                                                                  int C, int Cpad) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // (pixel, octet)
  const int oc = Cpad >> 3;
  if (i >= npix * oc) return;
  const int o = int(i % oc);
  const long long pix = i / oc;
  float f[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = o * 8 + j;
    f[j] = c < C ? ((float)in[pix * C + c] / 255.0f - 0.5f) / 0.5f : 0.f;
  }
  reinterpret_cast<uint4*>(out)[i] = pack8(f);
}

// ---------------------------------------------------------------- row softmax, bf16 out
// p = softmax(scale * s) per row over [0, L), one block per row, fp32 math; s is bf16 (in place: p == s) or fp32.  Rows
// are read and written as 8-wide vectors over [0, round_up(L, 8)): the columns [L, round_up(L, 8)) of the last vector
// are left out of the max and the sum and written as zeros (the VAE's attention contracts P.V over the padded length).
__device__ __forceinline__ void load8(const __nv_bfloat16* row, int i, float* f) {
  unpack8(reinterpret_cast<const uint4*>(row)[i], f);
}
__device__ __forceinline__ void load8(const float* row, int i, float* f) {
  const float4 a = reinterpret_cast<const float4*>(row)[2 * i], b = reinterpret_cast<const float4*>(row)[2 * i + 1];
  f[0] = a.x, f[1] = a.y, f[2] = a.z, f[3] = a.w, f[4] = b.x, f[5] = b.y, f[6] = b.z, f[7] = b.w;
}

template <typename T>
__global__ void __launch_bounds__(256) softmax_rows_kernel(const T* s, long long lds, __nv_bfloat16* p, long long ldp,
                                                           int L, float scale) {
  __shared__ float red[8];
  const T* row = s + (long long)blockIdx.x * lds;
  __nv_bfloat16* prow = p + (long long)blockIdx.x * ldp;
  const int nvec = (L + 7) >> 3;
  const float k = scale * 1.4426950408889634f;
  float mx = -INFINITY;
  for (int i = threadIdx.x; i < nvec; i += 256) {
    float f[8];
    load8(row, i, f);
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (i * 8 + j < L) mx = fmaxf(mx, f[j]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) mx = fmaxf(mx, red[w]);
  __syncthreads();
  float sum = 0.f;
  for (int i = threadIdx.x; i < nvec; i += 256) {
    float f[8];
    load8(row, i, f);
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (i * 8 + j < L) sum += exp2f((f[j] - mx) * k);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  sum = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) sum += red[w];
  const float inv = 1.0f / sum;
  for (int i = threadIdx.x; i < nvec; i += 256) {
    float f[8];
    load8(row, i, f);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = i * 8 + j < L ? exp2f((f[j] - mx) * k) * inv : 0.f;
    reinterpret_cast<uint4*>(prow)[i] = pack8(f);
  }
}

// ---------------------------------------------------------------- out[c, r] = in[r, c]  (bf16, 32x32 tiles)
__global__ void __launch_bounds__(256) transpose_kernel(const __nv_bfloat16* in, long long ld_in,
                                                        __nv_bfloat16* out, long long ld_out, int R, int Cc) {
  __shared__ __nv_bfloat16 tile[32][33];
  const int bx = blockIdx.x * 32, by = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int j = ty; j < 32; j += 8) {
    const int r = by + j, c = bx + tx;
    if (r < R && c < Cc) tile[j][tx] = in[(long long)r * ld_in + c];
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const int c = bx + j, r = by + tx;
    if (r < R && c < Cc) out[(long long)c * ld_out + r] = tile[tx][j];
  }
}

}  // namespace

extern "C" int b2f_groupnorm_silu(const void* x, const void* gamma, const void* beta, void* y, void* stats_ws_, int N,
                                  int64_t P, int C, float eps, int silu, b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  double* stats_ws = static_cast<double*>(stats_ws_);
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (!x || !gamma || !beta || !y || !stats_ws || N <= 0 || P <= 0) return B2F_ERR_INVALID;
  if (C % 32 || C % 8 || C > 2048 || (GN_THREADS % (C / 8)) != 0) return B2F_ERR_UNSUPPORTED;
  cudaError_t e = cudaMemsetAsync(stats_ws, 0, sizeof(double) * 64 * N, stream);
  if (e != cudaSuccess) return cuda_err(e, "groupnorm memset");
  dim3 g1((unsigned)((P + GN_PIX_PER_BLOCK - 1) / GN_PIX_PER_BLOCK), N);
  prof_begin(KC_OTHER, stream);
  gn_stats_kernel<<<g1, GN_THREADS, 0, stream>>>(static_cast<const __nv_bfloat16*>(x), stats_ws, P, C);
  const long long oct = P * (C / 8);
  dim3 g2((unsigned)((oct + 255) / 256), N);
  gn_apply_kernel<<<g2, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(x), stats_ws,
                                          static_cast<const __nv_bfloat16*>(gamma),
                                          static_cast<const __nv_bfloat16*>(beta),
                                          static_cast<__nv_bfloat16*>(y), P, C, eps, silu);
  prof_end(KC_OTHER, stream, 0.0, 6.0 * N * (double)P * C);
  B2F_LAUNCHED("groupnorm kernels", 2);
  return B2F_OK;
}

extern "C" int b2f_upsample2x(const void* in, void* out, int N, int H, int W, int C, b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (!in || !out || N <= 0 || H <= 0 || W <= 0 || C <= 0 || (C & 7)) return B2F_ERR_INVALID;
  const long long total = (long long)N * 4 * H * W * (C / 8);
  prof_begin(KC_OTHER, stream);
  upsample2x_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(
      static_cast<const uint4*>(in), static_cast<uint4*>(out), N, H, W, C / 8);
  prof_end(KC_OTHER, stream, 0.0, 2.0 * N * (double)H * W * C * 5.0);
  B2F_LAUNCHED("upsample2x_kernel", 1);
  return B2F_OK;
}

extern "C" int b2f_nchw_to_nhwc_pad(const void* in, int in_is_f32, void* out, int N, int C, int H, int W, int Cpad,
                                    b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (!in || !out || N <= 0 || C <= 0 || H <= 0 || W <= 0 || Cpad < C || (Cpad & 7)) return B2F_ERR_INVALID;
  const long long total = (long long)N * H * W * (Cpad / 8);
  const unsigned grid = (unsigned)((total + 255) / 256);
  if (in_is_f32 == 2)      // uint8 NHWC image
    u8_nhwc_to_nhwc_pad_kernel<<<grid, 256, 0, stream>>>(static_cast<const uint8_t*>(in), static_cast<__nv_bfloat16*>(out),
                                                       (long long)N * H * W, C, Cpad);
  else if (in_is_f32)
    nchw_to_nhwc_pad_kernel<float><<<grid, 256, 0, stream>>>(static_cast<const float*>(in),
                                                             static_cast<__nv_bfloat16*>(out), N, C, H, W, Cpad);
  else
    nchw_to_nhwc_pad_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(
        static_cast<const __nv_bfloat16*>(in), static_cast<__nv_bfloat16*>(out), N, C, H, W, Cpad);
  B2F_LAUNCHED("nchw_to_nhwc_pad_kernel", 1);
  return B2F_OK;
}

extern "C" int b2f_softmax_rows(void* s, int64_t ld, int rows, int L, float scale, b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (!s || rows <= 0 || L <= 0 || (ld & 7) || ld < ((L + 7) & ~7)) return B2F_ERR_INVALID;
  prof_begin(KC_OTHER, stream);
  softmax_rows_kernel<__nv_bfloat16><<<rows, 256, 0, stream>>>(static_cast<__nv_bfloat16*>(s), ld,
                                                               static_cast<__nv_bfloat16*>(s), ld, L, scale);
  prof_end(KC_OTHER, stream, 0.0, 4.0 * (double)rows * L);
  B2F_LAUNCHED("softmax_rows_kernel", 1);
  return B2F_OK;
}

extern "C" int b2f_softmax_rows_f32(const void* s, int64_t lds, void* p, int64_t ldp, int rows, int L, float scale,
                                    b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  const int L8 = (L + 7) & ~7;
  if (!s || !p || rows <= 0 || L <= 0 || (lds & 7) || (ldp & 7) || lds < L8 || ldp < L8) return B2F_ERR_INVALID;
  if ((reinterpret_cast<uintptr_t>(s) | reinterpret_cast<uintptr_t>(p)) & 15) return B2F_ERR_ALIGN;
  prof_begin(KC_OTHER, stream);
  softmax_rows_kernel<float><<<rows, 256, 0, stream>>>(static_cast<const float*>(s), lds,
                                                       static_cast<__nv_bfloat16*>(p), ldp, L, scale);
  prof_end(KC_OTHER, stream, 0.0, 6.0 * (double)rows * L);
  B2F_LAUNCHED("softmax_rows_kernel<float>", 1);
  return B2F_OK;
}

extern "C" int b2f_transpose_bf16(const void* in, int64_t ld_in, void* out, int64_t ld_out, int R, int Cc,
                                  b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (!in || !out || R <= 0 || Cc <= 0) return B2F_ERR_INVALID;
  dim3 grid((Cc + 31) / 32, (R + 31) / 32);
  transpose_kernel<<<grid, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(in), ld_in,
                                             static_cast<__nv_bfloat16*>(out), ld_out, R, Cc);
  B2F_LAUNCHED("transpose_kernel", 1);
  return B2F_OK;
}

}  // namespace b2f
