// Warp-specialised bf16 GEMM for sm_90a:  out[M,N] = epi(A[M,K] · W[N,K]^T + bias).
//
//   warpgroup 0 (1 lane)  TMA producer      cp.async.bulk.tensor → 128B-swizzled smem ring
//   warpgroups 1, 2       wgmma consumers   m64n128k16, 64 rows of the 128 x 128 tile each, fp32 in registers
//   epilogue              accumulators staged in smem → bias/act/gate/resid → global, one row per thread
//
// Both operands of the forward GEMM are K-major ([rows, K] row-major), which is what nn.Linear stores
// (SURVEY.md A.6) — no transposes anywhere.  The building blocks are shared with conv.cu (gemm_sm90.cuh).
//
// Replaces: torch.nn.functional.linear → cuBLASLt (diffusers FluxTransformer2DModel linears,
// reference call site univa/utils/flux_pipeline.py:1067; SURVEY.md §2b row 1).
#include <atomic>
#include <cstdlib>

#include "gemm_sm90.cuh"

namespace b2f {

extern std::atomic<uint64_t> g_launch_count;

namespace {

using namespace sm90;

struct GemmParams {
  int batch, M, N, K;  // M rows per batch item
  const __nv_bfloat16* bias;
  __nv_bfloat16* out;
  long long ldc, out_bs;
  int epi;
  const __nv_bfloat16* resid;
  long long ldr, resid_bs;
  const __nv_bfloat16* gate;
  long long gate_ld;
  int m_blocks_per_batch;
  int num_m_blocks, num_n_blocks, panel_n;
  // B2F_EPI_QKV_NORM_ROPE: N = 3*d_model laid out [Q | K | V], heads of 128 columns
  const __nv_bfloat16* nw_q;
  const __nv_bfloat16* nw_k;
  const float* rope_cos;  // [S, 128] fp32, row = rope_row0 + row-in-batch
  const float* rope_sin;
  int rope_row0, d_model;
  float norm_eps;
  // optional second output block: columns [split_n, N) go to out2 (own pitch) with epilogue epi2
  // (single-stream block: [Q|K|V | proj_mlp] in one launch, the MLP part GELU'd into the cat buffer)
  int split_n, epi2;
  __nv_bfloat16* out2;
  long long ldc2, out2_bs;
  // MODE 2 (wgrad): the contraction runs over kbatch x K rows (tokens of every batch item)
  int kbatch, kb_per_batch;
};

// Operand layouts of the kernel templates below.
//   MODE 0  forward:  out[M,N] = A[M,K] . W[N,K]^T          A, W K-major (contraction contiguous)
//   MODE 1  dgrad:    out[M,N] = A[M,K] . Wt[K,N]            A K-major, B MN-major: dX = dY . W with W as stored [out,in]
//   MODE 2  wgrad:    out[M,N] = sum_b At[b,K,M]^T . Bt[b,K,N]   both MN-major (tokens are the rows of both), fp32 output
// An MN-major 64(k) x 64(mn) box is one 128B-swizzled 8 KB TMA box; a tile of `mn` columns is mn/64 boxes 8 KB apart
// (descriptor LBO = 8192, SBO = 1024, 16 k-rows = 2048 bytes per wgmma k-step) — the layout the attention kernels
// use for V.

__device__ __forceinline__ void tile_coords(const GemmParams& p, int t, int& m_blk, int& n_blk) {
  // Panels of `panel_n` n-blocks; inside a panel n runs fastest so that the W panel stays in L2
  // while A streams through once per panel.
  const int panel_tiles = p.panel_n * p.num_m_blocks;
  const int panel = t / panel_tiles;
  const int r = t - panel * panel_tiles;
  const int w = min(p.panel_n, p.num_n_blocks - panel * p.panel_n);
  m_blk = r / w;
  n_blk = panel * p.panel_n + (r - m_blk * w);
}

// gelu_tanh(x) = 0.5 x (1 + tanh(u)) = x * sigmoid(2u), u = k0 (x + k1 x^3): one ex2 and one fast division instead of the
// branchy tanhf (which made the K = 3072 GEMMs with a GELU epilogue epilogue-bound: 1096 instead of 1257 TFLOP/s in the
// denoising loop).  Relative error ~1e-6, far below the bf16 rounding of the result.
__device__ __forceinline__ float gelu_tanh_f(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  const float u = x * fmaf(x * x, k0 * k1, k0);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(u * -2.8853900817779268f));   // exp(-2u)
  return __fdividef(x, 1.0f + e);
}
__device__ __forceinline__ float silu_f(float x) { return __fdividef(x, 1.0f + __expf(-x)); }
__device__ __forceinline__ float dgelu_tanh_f(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  const float t = tanhf(k0 * (x + k1 * x * x * x));
  return 0.5f * (1.0f + t) + 0.5f * x * (1.0f - t * t) * k0 * (1.0f + 3.0f * k1 * x * x);
}
__device__ __forceinline__ float dsilu_f(float x) {
  const float s = 1.0f / (1.0f + __expf(-x));
  return s * (1.0f + x * (1.0f - s));
}

// Epilogue for 32 accumulator columns of one output row: bias / activation / gate / residual with the
// bf16 rounding points of the torch-eager chain, then 16-byte stores.
__device__ __forceinline__ void epilogue_chunk(const GemmParams& p, const int epi, const uint32_t (&acc)[32], int n0,
                                               __nv_bfloat16* out_row, const __nv_bfloat16* res_row,
                                               const __nv_bfloat16* gate_row) {
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    const int n = n0 + g * 8;
    if (n >= p.N) break;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = __uint_as_float(acc[g * 8 + j]);
    if (p.bias) {
      const uint4 bq = __ldg(reinterpret_cast<const uint4*>(p.bias + n));
      const uint32_t bw[4] = {bq.x, bq.y, bq.z, bq.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 b2 = unpack_bf16x2(bw[j]);
        v[2 * j] += b2.x;
        v[2 * j + 1] += b2.y;
      }
    }
    if (epi == B2F_EPI_GELU_TANH) {
#pragma unroll
      for (int j = 0; j < 8; j += 2) {
        bf16r2(v[j], v[j + 1]);            // packed rounding (the scalar conversion runs on the slow XU pipe)
        v[j] = gelu_tanh_f(v[j]);
        v[j + 1] = gelu_tanh_f(v[j + 1]);
      }
    } else if (epi == B2F_EPI_GELU_ERF) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float x = bf16r(v[j]);
        v[j] = 0.5f * x * (1.0f + erff(x * 0.70710678118654752f));
      }
    } else if (epi == B2F_EPI_SILU) {
#pragma unroll
      for (int j = 0; j < 8; j += 2) {
        bf16r2(v[j], v[j + 1]);
        v[j] = silu_f(v[j]);
        v[j + 1] = silu_f(v[j + 1]);
      }
    } else if (epi == B2F_EPI_QUICK_GELU) {
      // transformers QuickGELUActivation in bf16 eager: x * sigmoid(1.702 * x), each op rounded
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float x = bf16r(v[j]);
        const float t = bf16r(1.702f * x);
        v[j] = x * bf16r(1.0f / (1.0f + __expf(-t)));
      }
    } else if (epi == B2F_EPI_GATE_RESID) {
      const uint4 gq = __ldg(reinterpret_cast<const uint4*>(gate_row + n));
      const uint4 rq = *reinterpret_cast<const uint4*>(res_row + n);
      const uint32_t gw[4] = {gq.x, gq.y, gq.z, gq.w};
      const uint32_t rw[4] = {rq.x, rq.y, rq.z, rq.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 g2 = unpack_bf16x2(gw[j]);
        const float2 r2 = unpack_bf16x2(rw[j]);
        float y0 = v[2 * j], y1 = v[2 * j + 1];
        bf16r2(y0, y1);
        y0 *= g2.x;
        y1 *= g2.y;
        bf16r2(y0, y1);
        v[2 * j] = r2.x + y0;
        v[2 * j + 1] = r2.y + y1;
      }
    }
    else if (epi == B2F_EPI_DGELU || epi == B2F_EPI_DSILU) {
      // backward of the activation fused into the dgrad GEMM: out = bf16(acc) * act'(u), u = the saved
      // pre-activation (read through the resid pointer)
      const uint4 uq = *reinterpret_cast<const uint4*>(res_row + n);
      const uint32_t uw[4] = {uq.x, uq.y, uq.z, uq.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 u2 = unpack_bf16x2(uw[j]);
        const float d0 = epi == B2F_EPI_DGELU ? dgelu_tanh_f(u2.x) : dsilu_f(u2.x);
        const float d1 = epi == B2F_EPI_DGELU ? dgelu_tanh_f(u2.y) : dsilu_f(u2.y);
        v[2 * j] = bf16r(v[2 * j]) * d0;
        v[2 * j + 1] = bf16r(v[2 * j + 1]) * d1;
      }
    } else if (epi == B2F_EPI_F32 || epi == B2F_EPI_F32_ACC) {
      float* o = reinterpret_cast<float*>(out_row) + n;
      float4 a0 = make_float4(v[0], v[1], v[2], v[3]), a1 = make_float4(v[4], v[5], v[6], v[7]);
      if (epi == B2F_EPI_F32_ACC) {
        const float4 p0 = *reinterpret_cast<const float4*>(o), p1 = *reinterpret_cast<const float4*>(o + 4);
        a0.x += p0.x; a0.y += p0.y; a0.z += p0.z; a0.w += p0.w;
        a1.x += p1.x; a1.y += p1.y; a1.z += p1.z; a1.w += p1.w;
      }
      *reinterpret_cast<float4*>(o) = a0;
      *reinterpret_cast<float4*>(o + 4) = a1;
      continue;
    }
    else if (epi == B2F_EPI_RESID) {
      const uint4 rq = *reinterpret_cast<const uint4*>(res_row + n);
      const uint32_t rw[4] = {rq.x, rq.y, rq.z, rq.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 r2 = unpack_bf16x2(rw[j]);
        float y0 = v[2 * j], y1 = v[2 * j + 1];
        bf16r2(y0, y1);
        v[2 * j] = r2.x + y0;
        v[2 * j + 1] = r2.y + y1;
      }
    }
    uint4 o;
    o.x = pack_bf16x2(v[0], v[1]);
    o.y = pack_bf16x2(v[2], v[3]);
    o.z = pack_bf16x2(v[4], v[5]);
    o.w = pack_bf16x2(v[6], v[7]);
    *reinterpret_cast<uint4*>(out_row + n) = o;
  }
}

// One 128-column head of a fused QKV projection for one token, straight from the staged accumulators:
//   x = bf16(acc + bias);  y = bf16(x * rsqrt(mean(x^2) + eps));  z = bf16(y * w);
//   out = bf16(z * cos + rot(z) * sin)        (diffusers RMSNorm + apply_rotary_emb, SURVEY.md A.2)
// — the same rounding chain as rmsnorm_rope_kernel, but without the extra HBM round trip.  Every rounding is the packed
// cvt.rn.bf16x2.
__device__ __forceinline__ void epilogue_head_norm_rope(const GemmParams& p, const float* crow, int n_head0,
                                                        long long row, __nv_bfloat16* out_row, bool is_k) {
  const __nv_bfloat16* w = is_k ? p.nw_k : p.nw_q;
  // pass 1: sum of squares of x = bf16(acc + bias) over the head
  float ss = 0.f;
#pragma unroll 1
  for (int cc = 0; cc < 4; ++cc) {
    uint32_t acc[32];
    load_chunk(crow, cc * 32, acc);
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const int c = cc * 32 + g * 8;
      const uint4 bq = p.bias ? __ldg(reinterpret_cast<const uint4*>(p.bias + n_head0 + c)) : make_uint4(0, 0, 0, 0);
      const uint32_t bw[4] = {bq.x, bq.y, bq.z, bq.w};
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const float2 b2 = unpack_bf16x2(bw[jj]);
        float x0 = __uint_as_float(acc[g * 8 + 2 * jj]) + b2.x, x1 = __uint_as_float(acc[g * 8 + 2 * jj + 1]) + b2.y;
        bf16r2(x0, x1);
        ss = fmaf(x0, x0, ss);
        ss = fmaf(x1, x1, ss);
      }
    }
  }
  const float r = rsqrtf(ss * (1.0f / 128.0f) + p.norm_eps);
  const float* cs = p.rope_cos + ((long long)p.rope_row0 + row) * 128;
  const float* sn = p.rope_sin + ((long long)p.rope_row0 + row) * 128;
  // pass 2: normalise, weight, rotate, store
#pragma unroll 1
  for (int cc = 0; cc < 4; ++cc) {
    uint32_t acc[32];
    load_chunk(crow, cc * 32, acc);
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const int c = cc * 32 + g * 8;
      const uint4 bq = p.bias ? __ldg(reinterpret_cast<const uint4*>(p.bias + n_head0 + c)) : make_uint4(0, 0, 0, 0);
      const uint4 wq = __ldg(reinterpret_cast<const uint4*>(w + c));
      const uint32_t bw[4] = {bq.x, bq.y, bq.z, bq.w};
      const uint32_t ww[4] = {wq.x, wq.y, wq.z, wq.w};
      const float4 c0 = __ldg(reinterpret_cast<const float4*>(cs + c)), c1 = __ldg(reinterpret_cast<const float4*>(cs + c + 4));
      const float4 s0 = __ldg(reinterpret_cast<const float4*>(sn + c)), s1 = __ldg(reinterpret_cast<const float4*>(sn + c + 4));
      const float cc8[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
      const float sc8[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
      uint32_t o[4];
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const float2 b2 = unpack_bf16x2(bw[jj]);
        const float2 w2 = unpack_bf16x2(ww[jj]);
        float z0 = __uint_as_float(acc[g * 8 + 2 * jj]) + b2.x, z1 = __uint_as_float(acc[g * 8 + 2 * jj + 1]) + b2.y;
        bf16r2(z0, z1);          // x
        z0 *= r;
        z1 *= r;
        bf16r2(z0, z1);          // y = bf16(x * r)
        z0 *= w2.x;
        z1 *= w2.y;
        bf16r2(z0, z1);          // z = bf16(y * w)
        o[jj] = pack_bf16x2(z0 * cc8[2 * jj] - z1 * sc8[2 * jj], z1 * cc8[2 * jj + 1] + z0 * sc8[2 * jj + 1]);
      }
      *reinterpret_cast<uint4*>(out_row + n_head0 + c) = make_uint4(o[0], o[1], o[2], o[3]);
    }
  }
}

// row pointer of the output; fp32 outputs (wgrad) have their pitch in floats
__device__ __forceinline__ __nv_bfloat16* out_row_ptr(const GemmParams& p, int bidx, long long row) {
  if (p.epi == B2F_EPI_F32 || p.epi == B2F_EPI_F32_ACC)
    return reinterpret_cast<__nv_bfloat16*>(reinterpret_cast<float*>(p.out) + bidx * p.out_bs + row * p.ldc);
  return p.out + bidx * p.out_bs + row * p.ldc;
}

// Epilogue of one output row for the calling thread: its `half` (0 / 1) of the tile's 128 columns, read from the
// staged accumulators.  A fused QKV head is the whole tile: the half-0 thread of the row runs it.
__device__ __forceinline__ void epilogue_row(const GemmParams& p, const float* crow, int half, int n_blk, bool row_ok,
                                             long long row, __nv_bfloat16* out_row, const __nv_bfloat16* res_row,
                                             const __nv_bfloat16* gate_row, __nv_bfloat16* out_row2) {
  if (!row_ok) return;
  if (p.epi == B2F_EPI_QKV_NORM_ROPE) {
    if (half == 1) return;
    const int n_head0 = n_blk * BLOCK_N;
    const int which = n_head0 / p.d_model;  // 0 = Q, 1 = K, 2 = V, >= 3: second output block
    if (which < 2 && n_head0 < p.N) {
      epilogue_head_norm_rope(p, crow, n_head0, row, out_row, which == 1);
      return;
    }
    const bool second = p.split_n > 0 && n_head0 >= p.split_n;
    __nv_bfloat16* orow = second ? out_row2 : out_row;
    const int epi = second ? p.epi2 : B2F_EPI_BIAS;
#pragma unroll 1
    for (int cc = 0; cc < 4; ++cc) {
      if (n_head0 + cc * 32 >= p.N) break;
      uint32_t acc[32];
      load_chunk(crow, cc * 32, acc);
      epilogue_chunk(p, epi, acc, n_head0 + cc * 32, orow, res_row, gate_row);
    }
    return;
  }
#pragma unroll 1
  for (int c0 = 0; c0 < BLOCK_N / 2; c0 += 32) {
    const int n0 = n_blk * BLOCK_N + half * (BLOCK_N / 2) + c0;
    if (n0 >= p.N) break;
    uint32_t acc[32];
    load_chunk(crow, half * (BLOCK_N / 2) + c0, acc);
    epilogue_chunk(p, p.epi, acc, n0, out_row, res_row, gate_row);
  }
}

template <int MODE>
__global__ void __launch_bounds__(THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  const Smem s = carve(smem_raw);
  const int wg = threadIdx.x >> 7;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
  }
  init_barriers(s);

  int m_blk, n_blk;
  tile_coords(p, blockIdx.x, m_blk, n_blk);
  const int num_kb = MODE == 2 ? p.kbatch * p.kb_per_batch : (p.K + BLOCK_K - 1) / BLOCK_K;
  const int bb = m_blk / p.m_blocks_per_batch;
  const int mb = m_blk - bb * p.m_blocks_per_batch;

  if (wg == 0) {
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&s.empty[stage], phase ^ 1);
        uint8_t* sa = s.ring + stage * STAGE_BYTES;
        uint8_t* sb = sa + A_BYTES;
        mbar_expect_tx(&s.full[stage], STAGE_BYTES);
        if (MODE == 2) {
          const int kbb = kb / p.kb_per_batch;
          const int kr = (kb - kbb * p.kb_per_batch) * BLOCK_K;
#pragma unroll
          for (int i = 0; i < BLOCK_M / 64; ++i)
            tma_load_3d(sa + i * MN_BOX_BYTES, &tmA, &s.full[stage], m_blk * BLOCK_M + 64 * i, kr, kbb);
#pragma unroll
          for (int i = 0; i < BLOCK_N / 64; ++i)
            tma_load_3d(sb + i * MN_BOX_BYTES, &tmB, &s.full[stage], n_blk * BLOCK_N + 64 * i, kr, kbb);
        } else {
          tma_load_3d(sa, &tmA, &s.full[stage], kb * BLOCK_K, mb * BLOCK_M, bb);
          if (MODE == 1) {
#pragma unroll
            for (int i = 0; i < BLOCK_N / 64; ++i)
              tma_load_2d(sb + i * MN_BOX_BYTES, &tmB, &s.full[stage], n_blk * BLOCK_N + 64 * i, kb * BLOCK_K);
          } else {
            tma_load_2d(sb, &tmB, &s.full[stage], kb * BLOCK_K, n_blk * BLOCK_N);
          }
        }
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
    return;
  }
  float acc[64];
  mainloop<MODE == 2, MODE >= 1>(s, num_kb, wg - 1, acc);
  stage_accumulators(s, wg - 1, acc);

  const int e = threadIdx.x - 128;
  const int row_in_tile = e & (BLOCK_M - 1), half = e >> 7;
  const long long row = (long long)mb * BLOCK_M + row_in_tile;
  const bool row_ok = row < p.M;
  const __nv_bfloat16* gate_row = p.gate ? p.gate + (long long)bb * p.gate_ld : nullptr;
  __nv_bfloat16* out_row = out_row_ptr(p, bb, row);
  const __nv_bfloat16* res_row = p.resid ? p.resid + bb * p.resid_bs + row * p.ldr : nullptr;
  __nv_bfloat16* out_row2 = p.out2 ? p.out2 + bb * p.out2_bs + row * p.ldc2 - p.split_n : nullptr;
  epilogue_row(p, s.cbuf + row_in_tile * CROW, half, n_blk, row_ok, row, out_row, res_row, gate_row, out_row2);
}

template <int MODE>
int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, GemmParams p, cudaStream_t stream) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gemm_bf16_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    if (e != cudaSuccess) return cuda_err(e, "gemm smem attribute");
    attr_set = true;
  }
  p.m_blocks_per_batch = (p.M + BLOCK_M - 1) / BLOCK_M;
  p.num_m_blocks = p.batch * p.m_blocks_per_batch;
  p.num_n_blocks = (p.N + BLOCK_N - 1) / BLOCK_N;
  p.panel_n = 16;
  const int num_tiles = p.num_m_blocks * p.num_n_blocks;
  const double kk = MODE == 2 ? (double)p.kbatch * p.K : (double)p.K;
  prof_begin(KC_GEMM, stream);
  gemm_bf16_kernel<MODE><<<num_tiles, THREADS, SMEM_BYTES, stream>>>(tmA, tmB, p);
  {
    char tag_[96];
    snprintf(tag_, sizeof tag_, "gemm m%d %dx%dx%d b%d e%d", MODE, p.M, p.N, (int)kk, p.batch, p.epi);
    prof_end_tagged(KC_GEMM, stream, 2.0 * p.batch * (double)p.M * p.N * kk,
                    2.0 * ((double)p.batch * p.M * kk + (double)p.N * kk + (double)p.batch * p.M * p.N), tag_);
  }
  g_launch_count.fetch_add(1, std::memory_order_relaxed);
  B2F_CHECK_LAUNCH("gemm_bf16_kernel");
  return B2F_OK;
}

}  // namespace

struct QkvExtra {
  const void *nw_q, *nw_k;
  const float *cos, *sin;
  int rope_row0, d_model;
  float eps;
  int n_extra, epi_extra;   // optional second output block of n_extra columns
  void* out_extra;
  int64_t ld_extra, bs_extra;
};

static int gemm_bf16_impl(const void* A, int64_t lda, int64_t a_bs, const void* W, int64_t ldw,
              const void* bias, void* out, int64_t ldc, int64_t out_bs, int batch, int M, int N,
              int K, int epilogue, const void* resid, int64_t ldr, int64_t resid_bs, const void* gate,
              int64_t gate_ld, const QkvExtra* qx, cudaStream_t stream) {
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (batch <= 0 || M <= 0 || N <= 0 || K <= 0 || !A || !W || !out) return B2F_ERR_INVALID;
  if ((K & 7) || (N & 7) || (lda & 7) || (ldw & 7) || (ldc & 7) || (a_bs & 7) || (out_bs & 7))
    return B2F_ERR_ALIGN;
  if ((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(W) |
       reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(bias) |
       reinterpret_cast<uintptr_t>(resid) | reinterpret_cast<uintptr_t>(gate)) & 15)
    return B2F_ERR_ALIGN;
  if (epilogue < 0 || epilogue > B2F_EPI_QUICK_GELU) return B2F_ERR_INVALID;  // backward epilogues: gemm_dgrad / gemm_wgrad
  if (epilogue == B2F_EPI_QKV_NORM_ROPE) {
    if (!qx || !qx->nw_q || !qx->nw_k || !qx->cos || !qx->sin || qx->d_model <= 0) return B2F_ERR_INVALID;
    if (N != 3 * qx->d_model + qx->n_extra || (qx->d_model % 128) || (qx->n_extra & 7)) return B2F_ERR_UNSUPPORTED;
    if (qx->n_extra && (!qx->out_extra || (qx->ld_extra & 7) || (qx->bs_extra & 7) ||
                        (reinterpret_cast<uintptr_t>(qx->out_extra) & 15)))
      return B2F_ERR_INVALID;
    if ((reinterpret_cast<uintptr_t>(qx->nw_q) | reinterpret_cast<uintptr_t>(qx->nw_k) |
         reinterpret_cast<uintptr_t>(qx->cos) | reinterpret_cast<uintptr_t>(qx->sin)) & 15)
      return B2F_ERR_ALIGN;
  }
  if (epilogue == B2F_EPI_GATE_RESID) {
    if (!resid || !gate || (ldr & 7) || (gate_ld & 7) || (resid_bs & 7)) return B2F_ERR_INVALID;
  }
  if (epilogue == B2F_EPI_RESID) {
    if (!resid || (ldr & 7) || (resid_bs & 7)) return B2F_ERR_INVALID;
  }
  GemmParams p{};
  p.batch = batch;
  p.M = M;
  p.N = N;
  p.K = K;
  p.bias = static_cast<const __nv_bfloat16*>(bias);
  p.out = static_cast<__nv_bfloat16*>(out);
  p.ldc = ldc;
  p.out_bs = out_bs;
  p.epi = epilogue;
  p.resid = static_cast<const __nv_bfloat16*>(resid);
  p.ldr = ldr;
  p.resid_bs = resid_bs;
  p.gate = static_cast<const __nv_bfloat16*>(gate);
  p.gate_ld = gate_ld;
  if (qx) {
    p.nw_q = static_cast<const __nv_bfloat16*>(qx->nw_q);
    p.nw_k = static_cast<const __nv_bfloat16*>(qx->nw_k);
    p.rope_cos = qx->cos;
    p.rope_sin = qx->sin;
    p.rope_row0 = qx->rope_row0;
    p.d_model = qx->d_model;
    p.norm_eps = qx->eps;
    if (qx->n_extra) {
      p.split_n = 3 * qx->d_model;
      p.epi2 = qx->epi_extra;
      p.out2 = static_cast<__nv_bfloat16*>(qx->out_extra);
      p.ldc2 = qx->ld_extra;
      p.out2_bs = qx->bs_extra;
    }
  }

  CUtensorMap tmA, tmB;
  int rc = make_tmap_3d_rows(&tmA, A, (uint64_t)K, (uint64_t)M, (uint64_t)batch, (uint64_t)lda,
                             batch > 1 ? (uint64_t)a_bs : (uint64_t)M * lda);
  if (rc != B2F_OK) return rc;
  rc = make_tmap_2d_bf16(&tmB, W, (uint64_t)N, (uint64_t)K, (uint64_t)ldw, BLOCK_N, BLOCK_K);
  if (rc != B2F_OK) return rc;
  return launch_gemm<0>(tmA, tmB, p, stream);
}

int gemm_bf16(const void* A, int64_t lda, int64_t a_bs, const void* W, int64_t ldw,
              const void* bias, void* out, int64_t ldc, int64_t out_bs, int batch, int M, int N,
              int K, int epilogue, const void* resid, int64_t ldr, int64_t resid_bs, const void* gate,
              int64_t gate_ld, cudaStream_t stream) {
  if (epilogue == B2F_EPI_QKV_NORM_ROPE) return B2F_ERR_INVALID;  // needs the extended entry point
  return gemm_bf16_impl(A, lda, a_bs, W, ldw, bias, out, ldc, out_bs, batch, M, N, K, epilogue, resid, ldr,
                        resid_bs, gate, gate_ld, nullptr, stream);
}

// dX[batch, M, N] = epi(dY[batch, M, K] . W[K, N]) with W exactly as nn.Linear stores it ([out = K, in = N]): the
// backward-data GEMM of every linear layer on the training path (reference train_denoiser.py:1172,
// accelerator.backward -> autograd of F.linear).  Epilogues: B2F_EPI_BIAS (plain store), B2F_EPI_DGELU /
// B2F_EPI_DSILU (times act'(u), u = `resid` [batch, M, N]), B2F_EPI_RESID (accumulate into another gradient).
int gemm_dgrad(const void* dY, int64_t ldy, int64_t dy_bs, const void* W, int64_t ldw, void* dX, int64_t ldx,
               int64_t dx_bs, int batch, int M, int N, int K, int epilogue, const void* aux, int64_t ld_aux,
               int64_t aux_bs, cudaStream_t stream) {
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (batch <= 0 || M <= 0 || N <= 0 || K <= 0 || !dY || !W || !dX) return B2F_ERR_INVALID;
  if ((K & 7) || (N & 7) || (ldy & 7) || (ldw & 7) || (ldx & 7) || (dy_bs & 7) || (dx_bs & 7)) return B2F_ERR_ALIGN;
  if ((reinterpret_cast<uintptr_t>(dY) | reinterpret_cast<uintptr_t>(W) | reinterpret_cast<uintptr_t>(dX) |
       reinterpret_cast<uintptr_t>(aux)) & 15)
    return B2F_ERR_ALIGN;
  if (epilogue != B2F_EPI_BIAS && epilogue != B2F_EPI_DGELU && epilogue != B2F_EPI_DSILU && epilogue != B2F_EPI_RESID)
    return B2F_ERR_INVALID;
  if (epilogue != B2F_EPI_BIAS && (!aux || (ld_aux & 7) || (aux_bs & 7))) return B2F_ERR_INVALID;
  GemmParams p{};
  p.batch = batch;
  p.M = M;
  p.N = N;
  p.K = K;
  p.out = static_cast<__nv_bfloat16*>(dX);
  p.ldc = ldx;
  p.out_bs = dx_bs;
  p.epi = epilogue;
  p.resid = static_cast<const __nv_bfloat16*>(aux);
  p.ldr = ld_aux;
  p.resid_bs = aux_bs;
  CUtensorMap tmA, tmB;
  int rc = make_tmap_3d_rows(&tmA, dY, (uint64_t)K, (uint64_t)M, (uint64_t)batch, (uint64_t)ldy,
                             batch > 1 ? (uint64_t)dy_bs : (uint64_t)M * ldy);
  if (rc != B2F_OK) return rc;
  rc = make_tmap_2d_bf16(&tmB, W, (uint64_t)K, (uint64_t)N, (uint64_t)ldw, 64, 64);   // 64 (k) x 64 (n) boxes
  if (rc != B2F_OK) return rc;
  return launch_gemm<1>(tmA, tmB, p, stream);
}

// dW[M, N] (+)= sum_b dY[b, :, M]^T . X[b, :, N]  (fp32 output, contraction over the `rows` tokens of every batch
// item): the backward-weight GEMM of the trainable projections (reference train_denoiser.py:71-119 names them).
// dY: [batch, rows, >= M] view, X: [batch, rows, >= N] view (token pitches ldy / ldx, batch pitches in elements).
int gemm_wgrad(const void* dY, int64_t ldy, int64_t dy_bs, const void* X, int64_t ldx, int64_t x_bs, float* dW,
               int64_t ldw, int batch, int rows, int M, int N, int accumulate, cudaStream_t stream) {
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (batch <= 0 || rows <= 0 || M <= 0 || N <= 0 || !dY || !X || !dW) return B2F_ERR_INVALID;
  if ((M & 7) || (N & 7) || (ldy & 7) || (ldx & 7) || (dy_bs & 7) || (x_bs & 7) || (ldw & 3)) return B2F_ERR_ALIGN;
  if ((reinterpret_cast<uintptr_t>(dY) | reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(dW)) & 15)
    return B2F_ERR_ALIGN;
  GemmParams p{};
  p.batch = 1;
  p.M = M;
  p.N = N;
  p.K = rows;
  p.kbatch = batch;
  p.kb_per_batch = (rows + BLOCK_K - 1) / BLOCK_K;
  p.out = reinterpret_cast<__nv_bfloat16*>(dW);
  p.ldc = ldw;
  p.out_bs = 0;
  p.epi = accumulate ? B2F_EPI_F32_ACC : B2F_EPI_F32;
  CUtensorMap tmA, tmB;
  int rc = make_tmap_3d_rows(&tmA, dY, (uint64_t)M, (uint64_t)rows, (uint64_t)batch, (uint64_t)ldy,
                             batch > 1 ? (uint64_t)dy_bs : (uint64_t)rows * ldy, 64);
  if (rc != B2F_OK) return rc;
  rc = make_tmap_3d_rows(&tmB, X, (uint64_t)N, (uint64_t)rows, (uint64_t)batch, (uint64_t)ldx,
                         batch > 1 ? (uint64_t)x_bs : (uint64_t)rows * ldx, 64);
  if (rc != B2F_OK) return rc;
  return launch_gemm<2>(tmA, tmB, p, stream);
}

int gemm_qkv_norm_rope(const void* A, int64_t lda, int64_t a_bs, const void* W, int64_t ldw,
                       const void* bias, void* out, int64_t ldc, int64_t out_bs, int batch, int M,
                       int d_model, int K, const void* nw_q, const void* nw_k, const float* cos,
                       const float* sin, int rope_row0, float eps, int n_extra, void* out_extra,
                       int64_t ld_extra, int64_t bs_extra, int epi_extra, cudaStream_t stream) {
  QkvExtra qx{nw_q, nw_k, cos, sin, rope_row0, d_model, eps, n_extra, epi_extra, out_extra, ld_extra, bs_extra};
  return gemm_bf16_impl(A, lda, a_bs, W, ldw, bias, out, ldc, out_bs, batch, M, 3 * d_model + n_extra, K,
                        B2F_EPI_QKV_NORM_ROPE, nullptr, 0, 0, nullptr, 0, &qx, stream);
}

}  // namespace b2f
