// HBM-bound fused row kernels of the MMDiT block (SURVEY.md §2b "ATen elementwise / norm kernels").
// Each replaces a chain of separate torch-eager kernels in diffusers; every intermediate that torch
// would have rounded to bf16 is rounded here too, so results track the reference's rounding chain.
#include "host_common.h"
#include "ptx.cuh"

namespace b2f {

namespace {

// ------------------------------------------------------------------------------------------------
// AdaLN modulate:  y = bf16( bf16( bf16(LN(x)) * bf16(1 + scale[b]) ) + shift[b] )
// LN: no affine, eps, biased variance, fp32 statistics (torch.nn.functional.layer_norm on bf16).
// One warp per row, the row lives in registers (D <= 256*MAXC), two-pass statistics.
// Algorithmic bytes per row: 2*D*2 (+ 2*D*2 of scale/shift shared by all rows of a batch item).
constexpr int LN_MAXC = 20;  // D up to 5120

struct LnModParams {
  const __nv_bfloat16* x;
  long long ldx, x_batch_stride;
  const __nv_bfloat16* scale;
  const __nv_bfloat16* shift;
  long long mod_ld;  // stride between batch items of scale/shift
  __nv_bfloat16* out;
  long long ldo, out_batch_stride;
  int batch, rows, D;
  float eps;
  // rows [0, split_row) of every batch item use (scale, shift); rows >= split_row use (scale_b, shift_b)
  // — the text and image streams of a double block in one launch.  split_row = 0: single stream.
  int split_row;
  const __nv_bfloat16* scale_b;
  const __nv_bfloat16* shift_b;
  // FP8 output (b2f_ln_modulate_fp8): `out` holds e4m3 bytes (pitches in bytes), one fp32 scale per row
  float* row_scale;
  long long row_scale_bs;
};

// One warp per row, rows taken grid-stride.  The row stays PACKED in registers (MAXC uint4 per lane, 48 registers
// for D = 3072) and is unpacked again in each of the three passes (sum, centred sum of squares, output): with the
// 96-float copy the kernel ran at 16 warps per SM and 2.5 TB/s in the denoising loop; packed it fits 6 blocks of
// 4 warps per SM, i.e. twice the bytes in flight.
// FP8 = true (b2f_ln_modulate_fp8): the modulated bf16 row replaces the input row in registers, then one warp amax and
// the row rule write e4m3 bytes and the row's scale instead of the bf16 row.
template <int MAXC, bool FP8 = false>
__global__ void __launch_bounds__(128, 6) ln_modulate_kernel(const LnModParams p) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long total = (long long)p.batch * p.rows;
  const int nchunk = p.D >> 8;
  const float inv_d = 1.0f / float(p.D);
  for (long long grow = (long long)blockIdx.x * 4 + warp; grow < total; grow += (long long)gridDim.x * 4) {
    const int b = int(grow / p.rows);
    const int r = int(grow - (long long)b * p.rows);
    const __nv_bfloat16* xr = p.x + b * p.x_batch_stride + r * p.ldx;
    __nv_bfloat16* orow = p.out + b * p.out_batch_stride + r * p.ldo;
    uint4 q[MAXC];
#pragma unroll
    for (int c = 0; c < MAXC; ++c)
      if (c < nchunk) q[c] = *reinterpret_cast<const uint4*>(xr + c * 256 + lane * 8);
    // Every pass works on bf16 PAIRS: a packed word unpacks to two fp32 with a shift and a mask, the statistics run on
    // the packed fp32 pipe (FADD2 / FFMA2), and the modulation, whose operands are bf16 values at every step of the
    // eager chain, runs on packed bf16 arithmetic (an exact product or sum rounded once to bf16, which is what the fp32
    // op followed by a conversion gives): a third of the instructions of the scalar version, which was issue-bound.
    float s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int c = 0; c < MAXC; ++c) {
      if (c < nchunk) {
        const uint32_t w[4] = {q[c].x, q[c].y, q[c].z, q[c].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) fadd2(s0, s1, s0, s1, __uint_as_float(w[j] << 16), __uint_as_float(w[j] & 0xffff0000u));
      }
    }
    const float mean = warp_sum(s0 + s1) * inv_d;
    const float nmean = -mean;
    float ss0 = 0.f, ss1 = 0.f;
#pragma unroll
    for (int c = 0; c < MAXC; ++c) {
      if (c < nchunk) {
        const uint32_t w[4] = {q[c].x, q[c].y, q[c].z, q[c].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float d0, d1;
          fadd2(d0, d1, __uint_as_float(w[j] << 16), __uint_as_float(w[j] & 0xffff0000u), nmean, nmean);
          ffma2(ss0, ss1, d0, d1, d0, d1, ss0, ss1);
        }
      }
    }
    const float rstd = rsqrtf(warp_sum(ss0 + ss1) * inv_d + p.eps);
    const bool second = p.split_row > 0 && r >= p.split_row;
    const __nv_bfloat16* sc = (second ? p.scale_b : p.scale) + (long long)b * p.mod_ld;
    const __nv_bfloat16* sh = (second ? p.shift_b : p.shift) + (long long)b * p.mod_ld;
    const __nv_bfloat162 one2 = __floats2bfloat162_rn(1.0f, 1.0f);
#pragma unroll
    for (int c = 0; c < MAXC; ++c) {
      if (c < nchunk) {
        const uint32_t w[4] = {q[c].x, q[c].y, q[c].z, q[c].w};
        const uint4 a4 = __ldg(reinterpret_cast<const uint4*>(sc + c * 256 + lane * 8));
        const uint4 h4 = __ldg(reinterpret_cast<const uint4*>(sh + c * 256 + lane * 8));
        const uint32_t a[4] = {a4.x, a4.y, a4.z, a4.w}, h[4] = {h4.x, h4.y, h4.z, h4.w};
        uint32_t o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {   // the rounding chain of the eager bf16 ops, two elements per instruction
          float d0, d1;
          fadd2(d0, d1, __uint_as_float(w[j] << 16), __uint_as_float(w[j] & 0xffff0000u), nmean, nmean);
          fmul2(d0, d1, d0, d1, rstd, rstd);
          const uint32_t yw = pack_bf16x2(d0, d1);                               // bf16(LN(x))
          const __nv_bfloat162 y = *reinterpret_cast<const __nv_bfloat162*>(&yw);
          const __nv_bfloat162 t = __hadd2_rn(one2, *reinterpret_cast<const __nv_bfloat162*>(&a[j]));   // bf16(1 + scale)
          const __nv_bfloat162 z = __hmul2_rn(y, t);                                                     // bf16(y * t)
          const __nv_bfloat162 r2 = __hadd2_rn(z, *reinterpret_cast<const __nv_bfloat162*>(&h[j]));      // bf16(z + shift)
          o[j] = *reinterpret_cast<const uint32_t*>(&r2);
        }
        if constexpr (FP8)
          q[c] = make_uint4(o[0], o[1], o[2], o[3]);
        else
          *reinterpret_cast<uint4*>(orow + c * 256 + lane * 8) = make_uint4(o[0], o[1], o[2], o[3]);
      }
    }
    if constexpr (FP8) {
      float m = 0.f;
#pragma unroll
      for (int c = 0; c < MAXC; ++c)
        if (c < nchunk) m = amax8(q[c], m);
      float s, inv;
      row_scale_of(warp_max(m), s, inv);
      uint8_t* orow8 = reinterpret_cast<uint8_t*>(p.out) + b * p.out_batch_stride + r * p.ldo;
#pragma unroll
      for (int c = 0; c < MAXC; ++c) {
        if (c < nchunk) {
          float v[8];
          unpack8(q[c], v);
          *reinterpret_cast<uint2*>(orow8 + c * 256 + lane * 8) = inv > 0.f ? quant_e4m3x8(v, inv) : make_uint2(0, 0);
        }
      }
      if (lane == 0) p.row_scale[b * p.row_scale_bs + r] = s;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Row quantization to e4m3 (include/b2f.h, b2f_quant_fp8_rows): one warp per row of K bf16 values (K % 16 == 0), 8
// values per lane and step.  The first pass takes the amax, the second re-reads the row (from L1 / L2) and converts.
struct QuantParams {
  const __nv_bfloat16* x;
  long long ldx, x_bs;
  uint8_t* q;
  long long ldq, q_bs;
  float* scale;
  long long scale_bs;
  int batch, rows, K;
};

__global__ void __launch_bounds__(256) quant_fp8_rows_kernel(const QuantParams p) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long total = (long long)p.batch * p.rows;
  for (long long grow = (long long)blockIdx.x * 8 + warp; grow < total; grow += (long long)gridDim.x * 8) {
    const int b = int(grow / p.rows);
    const int r = int(grow - (long long)b * p.rows);
    const __nv_bfloat16* xr = p.x + b * p.x_bs + r * p.ldx;
    float m = 0.f;
    for (int k = lane * 8; k < p.K; k += 256) m = amax8(*reinterpret_cast<const uint4*>(xr + k), m);
    float s, inv;
    row_scale_of(warp_max(m), s, inv);
    uint8_t* qr = p.q + b * p.q_bs + r * p.ldq;
    for (int k = lane * 8; k < p.K; k += 256) {
      float v[8];
      unpack8(*reinterpret_cast<const uint4*>(xr + k), v);
      *reinterpret_cast<uint2*>(qr + k) = inv > 0.f ? quant_e4m3x8(v, inv) : make_uint2(0, 0);   // +0, not -0 * 0
    }
    if (lane == 0) p.scale[b * p.scale_bs + r] = s;
  }
}

// ------------------------------------------------------------------------------------------------
// Per-head RMSNorm (eps, weight) + interleaved-pair RoPE on the Q and K column blocks of a fused QKV
// projection buffer [batch, S, >= 2*H*128], into an output of the same layout:
//   y = bf16(x * rsqrt(mean(x^2) + eps));  z = bf16(y * w);  out = bf16(z*cos + rot(z)*sin)
// (diffusers RMSNorm + apply_rotary_emb, SURVEY.md A.2).  Half a warp owns one 128-wide head vector
// (8 elements = 4 RoPE pairs per lane); lanes 0-15 do Q, lanes 16-31 do K of the same head.
// The first `n_a` tokens of every batch item use weight set A (norm_added_q/k: text tokens), the
// rest weight set B (norm_q/k).  The output may be the input (b2f_rmsnorm_rope): a lane reads its 8
// elements of a head with plain loads before it writes them, and no other thread touches them.
// Algorithmic bytes per token: 2 (Q,K) * H*128 * 2 B read + the same written.
struct NormRopeOutParams {
  const __nv_bfloat16* xq;
  const __nv_bfloat16* xk;
  __nv_bfloat16* oq;
  __nv_bfloat16* ok;
  long long ldx, x_batch_stride, ldo, o_batch_stride;
  const __nv_bfloat16 *wq_a, *wk_a, *wq_b, *wk_b;
  const float* cos;  // [S, 128]
  const float* sin;
  int batch, S, H, n_a;
  float eps;
};
__global__ void __launch_bounds__(256) rmsnorm_rope_out_kernel(const NormRopeOutParams p) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long tok = (long long)blockIdx.x * 8 + warp;
  if (tok >= (long long)p.batch * p.S) return;
  const int b = int(tok / p.S);
  const int s = int(tok - (long long)b * p.S);
  const int is_k = lane >> 4;
  const int l16 = lane & 15;
  const __nv_bfloat16* xb = (is_k ? p.xk : p.xq) + b * p.x_batch_stride + s * p.ldx + l16 * 8;
  __nv_bfloat16* ob = (is_k ? p.ok : p.oq) + b * p.o_batch_stride + s * p.ldo + l16 * 8;
  const bool set_a = s < p.n_a;
  const __nv_bfloat16* wptr = is_k ? (set_a ? p.wk_a : p.wk_b) : (set_a ? p.wq_a : p.wq_b);
  float w[8], cs[8], sn[8];
  unpack8(__ldg(reinterpret_cast<const uint4*>(wptr + l16 * 8)), w);
  {
    const float4* c4 = reinterpret_cast<const float4*>(p.cos + (long long)s * 128 + l16 * 8);
    const float4* s4 = reinterpret_cast<const float4*>(p.sin + (long long)s * 128 + l16 * 8);
    const float4 c0 = __ldg(c4), c1 = __ldg(c4 + 1), s0 = __ldg(s4), s1 = __ldg(s4 + 1);
    cs[0] = c0.x; cs[1] = c0.y; cs[2] = c0.z; cs[3] = c0.w;
    cs[4] = c1.x; cs[5] = c1.y; cs[6] = c1.z; cs[7] = c1.w;
    sn[0] = s0.x; sn[1] = s0.y; sn[2] = s0.z; sn[3] = s0.w;
    sn[4] = s1.x; sn[5] = s1.y; sn[6] = s1.z; sn[7] = s1.w;
  }
#pragma unroll 4
  for (int h = 0; h < p.H; ++h) {
    float x[8];
    unpack8(*reinterpret_cast<const uint4*>(xb + h * 128), x);
    float ss = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) ss += x[j] * x[j];
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float r = rsqrtf(ss * (1.0f / 128.0f) + p.eps);
    float z[8], o8[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) z[j] = bf16r(bf16r(x[j] * r) * w[j]);
#pragma unroll
    for (int j = 0; j < 8; j += 2) {
      o8[j] = z[j] * cs[j] - z[j + 1] * sn[j];
      o8[j + 1] = z[j + 1] * cs[j + 1] + z[j] * sn[j + 1];
    }
    *reinterpret_cast<uint4*>(ob + h * 128) = pack8(o8);
  }
}

// ------------------------------------------------------------------------------------------------
// Flow-matching Euler update (diffusers FlowMatchEulerDiscreteScheduler.step, SURVEY.md A.5):
//   x <- bf16( float(x) + float( bf16( bf16(dt) * v ) ) )   with dt = sigma[i+1] - sigma[i] in fp32.
// torch evaluates `dt * model_output` (0-dim fp32 tensor x bf16 tensor) in the common dtype bf16:
// the 0-dim operand is cast to bf16 FIRST, the product is rounded to bf16, the sum is fp32.
// v is the model output restricted to the first `cols`... both are [rows, cols] with pitches.
struct EulerParams {
  __nv_bfloat16* x;
  long long ldx;
  const __nv_bfloat16* v;
  long long ldv;
  long long rows;
  int cols;
  float dt;
};
__global__ void __launch_bounds__(256) euler_step_kernel(const EulerParams p) {
  const int vec_per_row = p.cols >> 3;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.rows * vec_per_row) return;
  const long long r = i / vec_per_row;
  const int c = int(i - r * vec_per_row) * 8;
  float x[8], v[8];
  unpack8(*reinterpret_cast<const uint4*>(p.x + r * p.ldx + c), x);
  unpack8(*reinterpret_cast<const uint4*>(p.v + r * p.ldv + c), v);
  const float dtb = bf16r(p.dt);
#pragma unroll
  for (int j = 0; j < 8; ++j) x[j] = x[j] + bf16r(dtb * v[j]);
  *reinterpret_cast<uint4*>(p.x + r * p.ldx + c) = pack8(x);
}

// y = silu(x) elementwise on a small [rows, cols] bf16 matrix (AdaLN: linear(silu(temb))).
__global__ void __launch_bounds__(256) silu_kernel(const __nv_bfloat16* x, __nv_bfloat16* y, long long n8) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n8) return;
  float f[8];
  unpack8(reinterpret_cast<const uint4*>(x)[i], f);
#pragma unroll
  for (int j = 0; j < 8; ++j) f[j] = f[j] / (1.0f + __expf(-f[j]));
  reinterpret_cast<uint4*>(y)[i] = pack8(f);
}

// Timesteps(256, flip_sin_to_cos=True, downscale_freq_shift=0): out[r] = [cos(t*f) | sin(t*f)],
// f_j = exp(-ln(10000) * j / 128), fp32 math, bf16 output (SURVEY.md A.3).
__global__ void __launch_bounds__(128) temb_sinusoid_kernel(const float* t, __nv_bfloat16* out, int rows) {
  const int r = blockIdx.x, j = threadIdx.x;
  if (r >= rows) return;
  const float f = expf(-9.210340371976184f * (float)j / 128.0f);
  const float a = t[r] * f;
  out[(long long)r * 256 + j] = __float2bfloat16_rn(cosf(a));
  out[(long long)r * 256 + 128 + j] = __float2bfloat16_rn(sinf(a));
}

// temb = bf16(bf16(t + g) + txt);  silu_temb = bf16(silu(temb))   (CombinedTimestepGuidanceTextProjEmbeddings)
__global__ void __launch_bounds__(256) temb_combine_kernel(const __nv_bfloat16* t, const __nv_bfloat16* g,
                                                           const __nv_bfloat16* txt, __nv_bfloat16* temb,
                                                           __nv_bfloat16* silu_temb, long long n8) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n8) return;
  float a[8], b[8], c[8], o[8], s8[8];
  unpack8(reinterpret_cast<const uint4*>(t)[i], a);
  unpack8(reinterpret_cast<const uint4*>(txt)[i], c);
  if (g) {
    unpack8(reinterpret_cast<const uint4*>(g)[i], b);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] = bf16r(a[j] + b[j]);
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    o[j] = bf16r(a[j] + c[j]);
    s8[j] = o[j] / (1.0f + __expf(-o[j]));
  }
  reinterpret_cast<uint4*>(temb)[i] = pack8(o);
  reinterpret_cast<uint4*>(silu_temb)[i] = pack8(s8);
}

// FluxPosEmbed (SURVEY.md A.2): per axis a with dim D_a, pair i: w = theta^(-2i/D_a) in float64,
// ang = pos * w, cos/sin in float64 -> fp32, each repeated twice (repeat_interleave(2)).
struct RopeTabParams {
  const float* ids;  // [S, 3]
  float* cos;
  float* sin;  // [S, 128]
  int S;
  int axes[3];
  double theta;
};
__global__ void __launch_bounds__(64) rope_tables_kernel(const RopeTabParams p) {
  const int s = blockIdx.x, i = threadIdx.x;  // pair index 0..63
  if (s >= p.S) return;
  int a = 0, li = i;
  while (a < 2 && li >= p.axes[a] / 2) {
    li -= p.axes[a] / 2;
    ++a;
  }
  const double dim = (double)p.axes[a];
  const double w = 1.0 / pow(p.theta, (double)(2 * li) / dim);
  const double ang = (double)p.ids[s * 3 + a] * w;
  const float c = (float)cos(ang), sn = (float)sin(ang);
  p.cos[(long long)s * 128 + 2 * i] = c;
  p.cos[(long long)s * 128 + 2 * i + 1] = c;
  p.sin[(long long)s * 128 + 2 * i] = sn;
  p.sin[(long long)s * 128 + 2 * i + 1] = sn;
}

}  // namespace

extern "C" int b2f_rope_tables(const float* ids, int S, const int* axes_dim, double theta, float* cos, float* sin,
                               b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (!ids || !cos || !sin || !axes_dim || S <= 0) return B2F_ERR_INVALID;
  if (axes_dim[0] + axes_dim[1] + axes_dim[2] != 128 || (axes_dim[0] | axes_dim[1] | axes_dim[2]) & 1)
    return B2F_ERR_UNSUPPORTED;
  RopeTabParams p{ids, cos, sin, S, {axes_dim[0], axes_dim[1], axes_dim[2]}, theta};
  rope_tables_kernel<<<S, 64, 0, stream>>>(p);
  B2F_LAUNCHED("rope_tables_kernel", 1);
  return B2F_OK;
}

extern "C" int b2f_temb_sinusoid(const float* t, void* out, int rows, b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (!t || !out || rows <= 0) return B2F_ERR_INVALID;
  temb_sinusoid_kernel<<<rows, 128, 0, stream>>>(t, static_cast<__nv_bfloat16*>(out), rows);
  B2F_LAUNCHED("temb_sinusoid_kernel", 1);
  return B2F_OK;
}

extern "C" int b2f_temb_combine(const void* t, const void* g, const void* txt, void* temb, void* silu_temb, int64_t n,
                                b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (!t || !txt || !temb || !silu_temb || n <= 0 || (n & 7)) return B2F_ERR_INVALID;
  const long long n8 = n >> 3;
  temb_combine_kernel<<<(unsigned)((n8 + 255) / 256), 256, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(t), static_cast<const __nv_bfloat16*>(g),
      static_cast<const __nv_bfloat16*>(txt), static_cast<__nv_bfloat16*>(temb),
      static_cast<__nv_bfloat16*>(silu_temb), n8);
  B2F_LAUNCHED("temb_combine_kernel", 1);
  return B2F_OK;
}

extern "C" int b2f_ln_modulate(const void* x, int64_t ldx, int64_t x_batch_stride, const void* scale, const void* shift,
                               int64_t mod_ld, void* out, int64_t ldo, int64_t out_batch_stride, int batch, int rows,
                               int D, float eps, int split_row, const void* scale_b, const void* shift_b,
                               b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (!x || !scale || !shift || !out || batch <= 0 || rows <= 0) return B2F_ERR_INVALID;
  if (D <= 0 || (D & 255) || D > 256 * LN_MAXC) return B2F_ERR_UNSUPPORTED;
  if ((ldx & 7) || (ldo & 7) || (mod_ld & 7) || (x_batch_stride & 7) || (out_batch_stride & 7))
    return B2F_ERR_ALIGN;
  LnModParams p{static_cast<const __nv_bfloat16*>(x), ldx, x_batch_stride,
                static_cast<const __nv_bfloat16*>(scale), static_cast<const __nv_bfloat16*>(shift),
                mod_ld, static_cast<__nv_bfloat16*>(out), ldo, out_batch_stride, batch, rows, D, eps,
                split_row, static_cast<const __nv_bfloat16*>(scale_b), static_cast<const __nv_bfloat16*>(shift_b),
                nullptr, 0};
  if (split_row > 0 && (!scale_b || !shift_b)) return B2F_ERR_INVALID;
  const long long total = (long long)batch * rows;
  // grid-stride rows: at most 12 four-row blocks per SM (two generations of the 6 resident ones)
  const long long want = (total + 3) / 4;
  const long long cap = (long long)device_info().num_sms * 12;
  const unsigned grid = (unsigned)(want < cap ? want : cap);
  prof_begin(KC_LNMOD, stream);
  struct ProfEnd {
    cudaStream_t s; double b;
    ~ProfEnd() { prof_end(KC_LNMOD, s, 0.0, b); }
  } prof_end_guard{stream, 4.0 * (double)total * D};
  if (D <= 1024)
    ln_modulate_kernel<4><<<grid, 128, 0, stream>>>(p);
  else if (D <= 3072)
    ln_modulate_kernel<12><<<grid, 128, 0, stream>>>(p);
  else
    ln_modulate_kernel<LN_MAXC><<<grid, 128, 0, stream>>>(p);
  B2F_LAUNCHED("ln_modulate_kernel", 1);
  return B2F_OK;
}

extern "C" int b2f_ln_modulate_fp8(const void* x, int64_t ldx, int64_t x_batch_stride, const void* scale,
                                   const void* shift, int64_t mod_ld, void* out, int64_t ldo, int64_t out_batch_stride,
                                   float* row_scale, int64_t row_scale_batch_stride, int batch, int rows, int D,
                                   float eps, int split_row, const void* scale_b, const void* shift_b,
                                   b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (!x || !scale || !shift || !out || !row_scale || batch <= 0 || rows <= 0) return B2F_ERR_INVALID;
  if (D <= 0 || (D & 255) || D > 3072) return B2F_ERR_UNSUPPORTED;   // the 20-chunk row (D > 3072) would spill
  if ((ldx & 7) || (ldo & 15) || (mod_ld & 7) || (x_batch_stride & 7) || (out_batch_stride & 15) ||
      (reinterpret_cast<uintptr_t>(out) & 15) || (reinterpret_cast<uintptr_t>(row_scale) & 3))
    return B2F_ERR_ALIGN;
  if (split_row > 0 && (!scale_b || !shift_b)) return B2F_ERR_INVALID;
  LnModParams p{static_cast<const __nv_bfloat16*>(x), ldx, x_batch_stride,
                static_cast<const __nv_bfloat16*>(scale), static_cast<const __nv_bfloat16*>(shift),
                mod_ld, static_cast<__nv_bfloat16*>(out), ldo, out_batch_stride, batch, rows, D, eps,
                split_row, static_cast<const __nv_bfloat16*>(scale_b), static_cast<const __nv_bfloat16*>(shift_b),
                row_scale, row_scale_batch_stride};
  const long long total = (long long)batch * rows;
  const long long want = (total + 3) / 4;
  const long long cap = (long long)device_info().num_sms * 12;
  const unsigned grid = (unsigned)(want < cap ? want : cap);
  prof_begin(KC_LNMOD, stream);
  if (D <= 1024)
    ln_modulate_kernel<4, true><<<grid, 128, 0, stream>>>(p);
  else
    ln_modulate_kernel<12, true><<<grid, 128, 0, stream>>>(p);
  prof_end(KC_LNMOD, stream, 0.0, 3.0 * (double)total * D + 4.0 * total);
  B2F_LAUNCHED("ln_modulate_kernel<fp8>", 1);
  return B2F_OK;
}

extern "C" int b2f_quant_fp8_rows(const void* x, int64_t ldx, int64_t x_batch_stride, void* q, int64_t ldq,
                                  int64_t q_batch_stride, float* scale, int64_t scale_batch_stride, int batch, int rows,
                                  int K, b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (!x || !q || !scale || batch <= 0 || rows <= 0 || K <= 0) return B2F_ERR_INVALID;
  if ((K & 15) || (ldx & 7) || (x_batch_stride & 7) || (ldq & 15) || (q_batch_stride & 15) ||
      ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(q)) & 15) ||
      (reinterpret_cast<uintptr_t>(scale) & 3))
    return B2F_ERR_ALIGN;
  QuantParams p{static_cast<const __nv_bfloat16*>(x), ldx, x_batch_stride, static_cast<uint8_t*>(q), ldq,
                q_batch_stride, scale, scale_batch_stride, batch, rows, K};
  const long long total = (long long)batch * rows;
  const long long want = (total + 7) / 8;
  const long long cap = (long long)device_info().num_sms * 16;
  const unsigned grid = (unsigned)(want < cap ? want : cap);
  prof_begin(KC_OTHER, stream);
  quant_fp8_rows_kernel<<<grid, 256, 0, stream>>>(p);
  prof_end(KC_OTHER, stream, 0.0, 3.0 * (double)total * K + 4.0 * total);
  B2F_LAUNCHED("quant_fp8_rows_kernel", 1);
  return B2F_OK;
}

extern "C" int b2f_rmsnorm_rope(void* q, void* k, int64_t ld, int64_t batch_stride, const void* wq_a, const void* wk_a,
                                const void* wq_b, const void* wk_b, const float* cos, const float* sin, int batch,
                                int S, int H, int head_dim, int n_a, float eps, b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (!q || !k || !wq_b || !wk_b || !cos || !sin || batch <= 0 || S <= 0 || H <= 0)
    return B2F_ERR_INVALID;
  if (head_dim != 128) return B2F_ERR_UNSUPPORTED;
  if (n_a > 0 && (!wq_a || !wk_a)) return B2F_ERR_INVALID;
  if ((ld & 7) || (batch_stride & 7)) return B2F_ERR_ALIGN;
  NormRopeOutParams p{static_cast<const __nv_bfloat16*>(q), static_cast<const __nv_bfloat16*>(k),
                      static_cast<__nv_bfloat16*>(q), static_cast<__nv_bfloat16*>(k), ld, batch_stride, ld, batch_stride,
                      static_cast<const __nv_bfloat16*>(wq_a), static_cast<const __nv_bfloat16*>(wk_a),
                      static_cast<const __nv_bfloat16*>(wq_b), static_cast<const __nv_bfloat16*>(wk_b),
                      cos, sin, batch, S, H, n_a, eps};
  const long long total = (long long)batch * S;
  prof_begin(KC_NORMROPE, stream);
  rmsnorm_rope_out_kernel<<<(unsigned)((total + 7) / 8), 256, 0, stream>>>(p);
  prof_end(KC_NORMROPE, stream, 0.0, 8.0 * (double)total * H * 128);
  B2F_LAUNCHED("rmsnorm_rope_out_kernel", 1);
  return B2F_OK;
}

extern "C" int b2f_rmsnorm_rope_out(const void* xq, const void* xk, int64_t ldx, int64_t x_bs, void* oq, void* ok,
                                    int64_t ldo, int64_t o_bs, const void* wq_a, const void* wk_a, const void* wq_b,
                                    const void* wk_b, const float* cos, const float* sin, int batch, int S, int H,
                                    int n_a, float eps, b2f_stream_t stream_) {
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  if (!xq || !xk || !oq || !ok || !wq_b || !wk_b || !cos || !sin || batch <= 0 || S <= 0 || H <= 0) return B2F_ERR_INVALID;
  if (n_a > 0 && (!wq_a || !wk_a)) return B2F_ERR_INVALID;
  if ((ldx | x_bs | ldo | o_bs) & 7) return B2F_ERR_ALIGN;
  NormRopeOutParams p{};
  p.xq = static_cast<const __nv_bfloat16*>(xq);
  p.xk = static_cast<const __nv_bfloat16*>(xk);
  p.oq = static_cast<__nv_bfloat16*>(oq);
  p.ok = static_cast<__nv_bfloat16*>(ok);
  p.ldx = ldx; p.x_batch_stride = x_bs; p.ldo = ldo; p.o_batch_stride = o_bs;
  p.wq_a = static_cast<const __nv_bfloat16*>(n_a > 0 ? wq_a : wq_b);
  p.wk_a = static_cast<const __nv_bfloat16*>(n_a > 0 ? wk_a : wk_b);
  p.wq_b = static_cast<const __nv_bfloat16*>(wq_b);
  p.wk_b = static_cast<const __nv_bfloat16*>(wk_b);
  p.cos = cos; p.sin = sin; p.batch = batch; p.S = S; p.H = H; p.n_a = n_a; p.eps = eps;
  const long long tokens = (long long)batch * S;
  prof_begin(KC_NORMROPE, st);
  rmsnorm_rope_out_kernel<<<(unsigned)((tokens + 7) / 8), 256, 0, st>>>(p);
  prof_end(KC_NORMROPE, st, 0, 8.0 * tokens * H * 128);
  B2F_LAUNCHED("rmsnorm_rope_out_kernel", 1);
  return B2F_OK;
}

extern "C" int b2f_euler_step(void* x, int64_t ldx, const void* v, int64_t ldv, int64_t rows, int cols, float dt,
                              b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (!x || !v || rows <= 0 || cols <= 0) return B2F_ERR_INVALID;
  if ((cols & 7) || (ldx & 7) || (ldv & 7)) return B2F_ERR_ALIGN;
  EulerParams p{static_cast<__nv_bfloat16*>(x), ldx, static_cast<const __nv_bfloat16*>(v), ldv, rows,
                cols, dt};
  const long long n = rows * (cols >> 3);
  euler_step_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(p);
  B2F_LAUNCHED("euler_step_kernel", 1);
  return B2F_OK;
}

extern "C" int b2f_silu(const void* x, void* y, int64_t n, b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (!x || !y || n <= 0 || (n & 7)) return B2F_ERR_INVALID;
  const long long n8 = n >> 3;
  silu_kernel<<<(unsigned)((n8 + 255) / 256), 256, 0, stream>>>(
      static_cast<const __nv_bfloat16*>(x), static_cast<__nv_bfloat16*>(y), n8);
  B2F_LAUNCHED("silu_kernel", 1);
  return B2F_OK;
}

}  // namespace b2f
