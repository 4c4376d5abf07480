// Persistent, warp-specialised bf16 GEMM for sm_90a with ping-pong consumers:  out[M,N] = epi(A[M,K] · W[N,K]^T + bias).
//
//   grid                  min(tiles, SMs) CTAs; CTA b takes the 128 x 128 tiles b, b + grid, ... in panel order
//   warpgroup 0 (1 lane)  TMA producer      cp.async.bulk.tensor → 128B-swizzled smem ring of STAGES stages, streamed
//                                           across tile boundaries (setmaxnreg.dec to 40 registers)
//   warpgroups 1, 2       wgmma consumers   each owns whole tiles, alternating (the CTA's tiles 0, 2, ... / 1, 3, ...):
//                                           two m64n128k16 per k16 step, 128 fp32 accumulators per thread
//                                           (setmaxnreg.inc to 232); named barriers make them take turns on the main
//                                           loop, so one runs its MMAs while the other runs its epilogue
//   epilogue              x = bf16(acc + bias) from registers → the consumer's own bf16 staging tile →
//                         act/gate/resid → global with 16-byte accesses, 16 threads per row; a fused QKV head runs one
//                         thread per row; the fp32 wgrad output goes straight from registers
//
// Every output element sees the same k16 accumulation order as a one-tile-per-CTA kernel with the same k-blocks.
// Both operands of the forward GEMM are K-major ([rows, K] row-major), which is what nn.Linear stores
// (SURVEY.md A.6) — no transposes anywhere.  The tile shape and ring layout are shared with conv.cu (gemm_sm90.cuh).
//
// Replaces: torch.nn.functional.linear → cuBLASLt (diffusers FluxTransformer2DModel linears,
// reference call site univa/utils/flux_pipeline.py:1067; SURVEY.md §2b row 1).
#include <algorithm>
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

// Epilogue of one 8-column group of one output row from x = bf16(acc + bias) (bf16(acc) without a bias):
// activation / gate / residual with the bf16 rounding points of the torch-eager chain, then one 16-byte store.
// Every chain starts by rounding acc + bias to bf16, which the staging tile already did; rounding x again is exact.
// rq: the 8 residual (GATE_RESID / RESID) or saved pre-activation (DGELU / DSILU) values, gq: the 8 gate values.
__device__ __forceinline__ void epilogue_group(const int epi, float (&v)[8], const uint4 rq, const uint4 gq,
                                               __nv_bfloat16* out) {
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
  } else if (epi == B2F_EPI_DGELU || epi == B2F_EPI_DSILU) {
    // backward of the activation fused into the dgrad GEMM: out = bf16(acc) * act'(u), u = the saved
    // pre-activation (read through the resid pointer)
    const uint32_t uw[4] = {rq.x, rq.y, rq.z, rq.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 u2 = unpack_bf16x2(uw[j]);
      const float d0 = epi == B2F_EPI_DGELU ? dgelu_tanh_f(u2.x) : dsilu_f(u2.x);
      const float d1 = epi == B2F_EPI_DGELU ? dgelu_tanh_f(u2.y) : dsilu_f(u2.y);
      v[2 * j] = bf16r(v[2 * j]) * d0;
      v[2 * j + 1] = bf16r(v[2 * j + 1]) * d1;
    }
  } else if (epi == B2F_EPI_RESID) {
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
  *reinterpret_cast<uint4*>(out) = o;
}

__device__ __forceinline__ void unpack_bf16x8(const uint4 q, float (&v)[8]) {
  const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 f = unpack_bf16x2(w[j]);
    v[2 * j] = f.x;
    v[2 * j + 1] = f.y;
  }
}

// One 128-column head of a fused QKV projection for one token, from its row of the staged tile x = bf16(acc + bias):
//   y = bf16(x * rsqrt(mean(x^2) + eps));  z = bf16(y * w);
//   out = bf16(z * cos + rot(z) * sin)        (diffusers RMSNorm + apply_rotary_emb, SURVEY.md A.2)
// — the same rounding chain as rmsnorm_rope_kernel, but without the extra HBM round trip.  The sum of squares runs over
// the columns in order, one thread per row.  Every rounding is the packed cvt.rn.bf16x2.
__device__ __forceinline__ void epilogue_head_norm_rope(const GemmParams& p, const uint8_t* srow, int n_head0,
                                                        long long row, __nv_bfloat16* out_row, bool is_k) {
  const __nv_bfloat16* w = is_k ? p.nw_k : p.nw_q;
  float ss = 0.f;
#pragma unroll 4
  for (int g = 0; g < BLOCK_N / 8; ++g) {
    float x[8];
    unpack_bf16x8(*reinterpret_cast<const uint4*>(srow + g * 16), x);
#pragma unroll
    for (int j = 0; j < 8; ++j) ss = fmaf(x[j], x[j], ss);
  }
  const float r = rsqrtf(ss * (1.0f / 128.0f) + p.norm_eps);
  const float* cs = p.rope_cos + ((long long)p.rope_row0 + row) * 128;
  const float* sn = p.rope_sin + ((long long)p.rope_row0 + row) * 128;
#pragma unroll 4
  for (int g = 0; g < BLOCK_N / 8; ++g) {
    const int c = g * 8;
    float x[8];
    unpack_bf16x8(*reinterpret_cast<const uint4*>(srow + g * 16), x);
    const uint4 wq = __ldg(reinterpret_cast<const uint4*>(w + c));
    const uint32_t ww[4] = {wq.x, wq.y, wq.z, wq.w};
    const float4 c0 = __ldg(reinterpret_cast<const float4*>(cs + c)), c1 = __ldg(reinterpret_cast<const float4*>(cs + c + 4));
    const float4 s0 = __ldg(reinterpret_cast<const float4*>(sn + c)), s1 = __ldg(reinterpret_cast<const float4*>(sn + c + 4));
    const float cc8[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
    const float sc8[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
    uint32_t o[4];
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const float2 w2 = unpack_bf16x2(ww[jj]);
      float z0 = x[2 * jj], z1 = x[2 * jj + 1];
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

// ---------------------------------------------------------------------------------------------------- the kernel
// Shared memory: the STAGES-deep operand ring, then one bf16 staging tile per consumer, then the ring's barriers.
constexpr int SROW = BLOCK_N * 2 + 16;     // byte pitch of a staged bf16 row: 16-byte accesses of 8 rows hit 32 banks
constexpr int STAGING_BYTES = BLOCK_M * SROW;
constexpr int PP_SMEM_BYTES = STAGES * STAGE_BYTES + 2 * STAGING_BYTES + 2 * STAGES * 8 + 1024;
// Named barriers (0 is __syncthreads):
constexpr int BAR_TURN = 2;   // + consumer: that consumer's turn on the tensor cores (256 threads: one arrives, one waits)
constexpr int BAR_EPI = 4;    // + consumer: its own warpgroup around the staging tile (128 threads)
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;   // 128 x 40 + 256 x 232 <= 65536
static_assert(128 * PRODUCER_REGS + 256 * CONSUMER_REGS <= 65536, "register split exceeds the register file");

__device__ __forceinline__ void tile_origin(const GemmParams& p, int t, int& n_blk, int& bb, int& mb) {
  int m_blk;
  tile_coords(p, t, m_blk, n_blk);
  bb = m_blk / p.m_blocks_per_batch;
  mb = m_blk - bb * p.m_blocks_per_batch;
}

// Persistent, warp-specialised GEMM with ping-pong consumers.  CTA b takes tiles b, b + grid, b + 2 grid, ... in panel
// order; its consumer warpgroups take turns on them (consumer 0: the CTA's tiles 0, 2, 4, ..., consumer 1: 1, 3, ...),
// each owning a whole 128 x 128 tile (two m64n128k16 per k16 step).  While one runs its tile's MMAs the other runs the
// epilogue of its previous tile, and the producer streams k-blocks through the ring across tile boundaries.
// LoRA K-extension of the forward GEMM (LORA = true, MODE 0 only): after a tile's K/64 k-blocks of (A, W) the
// producer streams num_kb2 more from (T [batch, M, r_pad], Bcat [N, r_pad]) through the same ring and the consumers
// run them into the same accumulators, so acc = A W^T + T Bcat^T before an unchanged epilogue.  With colscale set
// (the down projection T = bf16(colscale[n] cs_mul (X Acat^T)), bias NULL, epilogue BIAS), the staged value is
// bf16(acc * fp32(colscale[n] * cs_mul)).  LORA = false has an empty parameter and compiles to the plain kernel.
template <bool LORA>
struct LoraParams {};
template <>
struct LoraParams<true> {
  CUtensorMap tmT, tmBc;
  int num_kb2;
  const float* colscale;
  float cs_mul;
};

template <int MODE, bool LORA = false>
__global__ void __launch_bounds__(THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const GemmParams p, const __grid_constant__ LoraParams<LORA> lx) {
  constexpr int TA = MODE == 2, TB = MODE >= 1;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* ring = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(ring + STAGES * STAGE_BYTES + 2 * STAGING_BYTES);
  uint64_t* empty = full + STAGES;
  const int wg = threadIdx.x >> 7;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if constexpr (LORA) {
      if (lx.num_kb2 > 0) {
        tma_prefetch_desc(&lx.tmT);
        tma_prefetch_desc(&lx.tmBc);
      }
    }
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 4);   // one arrive per warp of the consumer that read the stage
    }
    fence_mbar_init();
  }
  __syncthreads();

  const int num_tiles = p.num_m_blocks * p.num_n_blocks;
  const int n_local = (num_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;   // this CTA's tiles
  const int num_kb = MODE == 2 ? p.kbatch * p.kb_per_batch : (p.K + BLOCK_K - 1) / BLOCK_K;
  int num_kb_all = num_kb;   // k-blocks per tile, the LoRA ones last
  if constexpr (LORA) num_kb_all += lx.num_kb2;

  if (wg == 0) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int i = 0; i < n_local; ++i) {
        int n_blk, bb, mb;
        tile_origin(p, blockIdx.x + i * gridDim.x, n_blk, bb, mb);
        const int m_blk = bb * p.m_blocks_per_batch + mb;
        for (int kb = 0; kb < num_kb_all; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          uint8_t* sa = ring + stage * STAGE_BYTES;
          uint8_t* sb = sa + A_BYTES;
          mbar_expect_tx(&full[stage], STAGE_BYTES);
          if (MODE == 2) {
            const int kbb = kb / p.kb_per_batch;
            const int kr = (kb - kbb * p.kb_per_batch) * BLOCK_K;
#pragma unroll
            for (int h = 0; h < BLOCK_M / 64; ++h)
              tma_load_3d(sa + h * MN_BOX_BYTES, &tmA, &full[stage], m_blk * BLOCK_M + 64 * h, kr, kbb);
#pragma unroll
            for (int h = 0; h < BLOCK_N / 64; ++h)
              tma_load_3d(sb + h * MN_BOX_BYTES, &tmB, &full[stage], n_blk * BLOCK_N + 64 * h, kr, kbb);
          } else {
            const CUtensorMap* mapA = &tmA;
            const CUtensorMap* mapB = &tmB;
            int kc = kb * BLOCK_K;
            if constexpr (LORA) {
              if (kb >= num_kb) {   // the LoRA k-blocks: (T, Bcat) in place of (A, W)
                mapA = &lx.tmT;
                mapB = &lx.tmBc;
                kc = (kb - num_kb) * BLOCK_K;
              }
            }
            tma_load_3d(sa, mapA, &full[stage], kc, mb * BLOCK_M, bb);
            if (MODE == 1) {
#pragma unroll
              for (int h = 0; h < BLOCK_N / 64; ++h)
                tma_load_2d(sb + h * MN_BOX_BYTES, mapB, &full[stage], n_blk * BLOCK_N + 64 * h, kc);
            } else {
              tma_load_2d(sb, mapB, &full[stage], kc, n_blk * BLOCK_N);
            }
          }
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
    return;
  }
  setmaxnreg_inc<CONSUMER_REGS>();

  const int c = wg - 1;                       // consumer 0 / 1
  const int tid = threadIdx.x & 127, w = tid >> 5, lane = tid & 31;
  uint8_t* stg = ring + STAGES * STAGE_BYTES + c * STAGING_BYTES;
  // Descriptors of stage 0.  Rows 64..127 of the A tile start 8 KB in: 64 K-major rows of 128 B, or the second
  // [64 k][64 m] box of an MN-major A.
  const uint32_t ring_u = smem_u32(ring);
  const uint64_t da0 = make_sdesc_sw128(ring_u, TA ? MN_BOX_BYTES : 16, 1024);
  const uint64_t da1 = make_sdesc_sw128(ring_u + 8192, TA ? MN_BOX_BYTES : 16, 1024);
  const uint64_t db0 = make_sdesc_sw128(ring_u + A_BYTES, TB ? MN_BOX_BYTES : 16, 1024);
  constexpr int A_KSTEP = TA ? 2048 : 32;
  constexpr int B_KSTEP = TB ? 2048 : 32;
  if (c == 1) named_bar_arrive(BAR_TURN + 0, 256);   // consumer 0 takes the first turn

  for (int i = c; i < n_local; i += 2) {
    int n_blk, bb, mb;
    tile_origin(p, blockIdx.x + i * gridDim.x, n_blk, bb, mb);

    // ---- main loop: this consumer's turn on the tensor cores.  Its tile's k-blocks are ring slots
    // i * num_kb_all .. (i + 1) * num_kb_all - 1 in the producer's order.
    float acc0[64], acc1[64];   // rows 0..63 / 64..127 of the tile
#pragma unroll
    for (int j = 0; j < 64; ++j) {
      acc0[j] = 0.f;
      acc1[j] = 0.f;
    }
    named_bar_sync(BAR_TURN + c, 256);
    const int slot0 = i * num_kb_all;
    int stage = slot0 % STAGES, prev = -1;
    uint32_t phase = (slot0 / STAGES) & 1;
    for (int kb = 0; kb < num_kb_all; ++kb) {
      mbar_wait(&full[stage], phase);
      const uint64_t soff = uint64_t((stage * STAGE_BYTES) >> 4);
      reg_fence(acc0);
      reg_fence(acc1);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BLOCK_K / 16; ++k) {
        const uint64_t ka = soff + uint64_t((k * A_KSTEP) >> 4), kb16 = soff + uint64_t((k * B_KSTEP) >> 4);
        wgmma_m64n128_ss<TA, TB>(acc0, da0 + ka, db0 + kb16, 1u);
        wgmma_m64n128_ss<TA, TB>(acc1, da1 + ka, db0 + kb16, 1u);
      }
      wgmma_commit();
      wgmma_wait<1>();   // the previous stage's MMAs are complete: hand it back to the producer
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[prev]);
      }
      prev = stage;
      if (++stage == STAGES) {
        stage = 0;
        phase ^= 1;
      }
    }
    if (i + 1 < n_local) named_bar_arrive(BAR_TURN + (c ^ 1), 256);   // the other consumer's tile goes next
    wgmma_wait<0>();
    reg_fence(acc0);
    reg_fence(acc1);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[prev]);

    // ---- epilogue, overlapping the other consumer's main loop.  Accumulator element j of a thread is row
    // 16 w + lane / 4 + 8 ((j / 2) & 1), column 8 (j / 4) + 2 (lane % 4) + (j & 1) of its 64-row half.
    const int r_lo = 16 * w + (lane >> 2);
    if (MODE == 2) {
      // fp32 weight gradient straight from the registers: a quad writes 32 contiguous bytes per 8-column group.  With
      // accumulate, the prior values of a thread's row are all read before its first store.
      const bool acc_in = p.epi == B2F_EPI_F32_ACC;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float* a = h ? acc1 : acc0;
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const long long row = (long long)mb * BLOCK_M + 64 * h + r_lo + 8 * rr;
          if (row >= p.M) continue;
          float* orow = reinterpret_cast<float*>(p.out) + row * p.ldc + n_blk * BLOCK_N + 2 * (lane & 3);
          const int n_left = p.N - n_blk * BLOCK_N - 2 * (lane & 3);   // columns 8 j of orow are valid while 8 j < n_left
          float2 q[BLOCK_N / 8];
#pragma unroll
          for (int j = 0; j < BLOCK_N / 8; ++j) {
            q[j] = make_float2(0.f, 0.f);
            if (acc_in && 8 * j < n_left) q[j] = *reinterpret_cast<const float2*>(orow + 8 * j);
          }
#pragma unroll
          for (int j = 0; j < BLOCK_N / 8; ++j) {
            if (8 * j >= n_left) break;
            float2 v = make_float2(a[4 * j + 2 * rr], a[4 * j + 2 * rr + 1]);
            if (acc_in) {
              v.x += q[j].x;
              v.y += q[j].y;
            }
            *reinterpret_cast<float2*>(orow + 8 * j) = v;
          }
        }
      }
      continue;
    }
    // x = bf16(acc + bias) into this consumer's staging tile, once its previous tile's epilogue is done reading it
    named_bar_sync(BAR_EPI + c, 128);
#pragma unroll
    for (int j = 0; j < BLOCK_N / 8; ++j) {
      const int col = 8 * j + 2 * (lane & 3);
      const int n = n_blk * BLOCK_N + col;
      const bool has_bias = p.bias && n < p.N;
      const float2 b2 = has_bias ? unpack_bf16x2(__ldg(reinterpret_cast<const uint32_t*>(p.bias + n))) : make_float2(0.f, 0.f);
      float2 cs2 = make_float2(1.f, 1.f);
      if constexpr (LORA) {
        if (lx.colscale && n < p.N) {
          cs2 = __ldg(reinterpret_cast<const float2*>(lx.colscale + n));
          cs2.x *= lx.cs_mul;
          cs2.y *= lx.cs_mul;
        }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float* a = h ? acc1 : acc0;
        float x0 = a[4 * j], x1 = a[4 * j + 1], x2 = a[4 * j + 2], x3 = a[4 * j + 3];
        if (has_bias) {
          x0 += b2.x;
          x1 += b2.y;
          x2 += b2.x;
          x3 += b2.y;
        }
        if constexpr (LORA) {
          if (lx.colscale) {
            x0 *= cs2.x;
            x1 *= cs2.y;
            x2 *= cs2.x;
            x3 *= cs2.y;
          }
        }
        uint8_t* s0 = stg + (64 * h + r_lo) * SROW + col * 2;
        *reinterpret_cast<uint32_t*>(s0) = pack_bf16x2(x0, x1);
        *reinterpret_cast<uint32_t*>(s0 + 8 * SROW) = pack_bf16x2(x2, x3);
      }
    }
    named_bar_sync(BAR_EPI + c, 128);

    const int n_tile0 = n_blk * BLOCK_N;
    const __nv_bfloat16* gate_row = p.gate ? p.gate + (long long)bb * p.gate_ld : nullptr;
    int epi = p.epi;
    __nv_bfloat16* out_base = p.out + bb * p.out_bs;
    long long ld = p.ldc;
    if (epi == B2F_EPI_QKV_NORM_ROPE) {
      const int which = n_tile0 / p.d_model;  // 0 = Q, 1 = K, 2 = V, >= 3: second output block
      if (which < 2) {
        // one normalised head per tile: one thread per row
        const long long row = (long long)mb * BLOCK_M + tid;
        if (row < p.M)
          epilogue_head_norm_rope(p, stg + tid * SROW, n_tile0, row, out_base + row * ld, which == 1);
        continue;
      }
      const bool second = p.split_n > 0 && n_tile0 >= p.split_n;
      epi = second ? p.epi2 : B2F_EPI_BIAS;
      if (second) {
        out_base = p.out2 + bb * p.out2_bs - p.split_n;
        ld = p.ldc2;
      }
    }
    // 16 threads per row, one 8-column group each: a warp reads and writes two 256-byte row segments.  Rows go in
    // batches of 4 per thread whose residual / pre-activation loads are all issued before the first store, so their
    // latencies overlap; a batch, not all 16 rows, keeps the unrolled activation code small.
    const int cg = tid & 15;
    const int n = n_tile0 + 8 * cg;
    if (n < p.N) {
      constexpr int RB = 4;
      const int r0 = tid >> 4;
      const bool reads_resid = epi == B2F_EPI_GATE_RESID || epi == B2F_EPI_RESID || epi == B2F_EPI_DGELU ||
                               epi == B2F_EPI_DSILU;
      const uint4 gq = epi == B2F_EPI_GATE_RESID ? __ldg(reinterpret_cast<const uint4*>(gate_row + n))
                                                 : make_uint4(0, 0, 0, 0);
#pragma unroll 1
      for (int rb = r0; rb < BLOCK_M; rb += 8 * RB) {     // tile rows rb + 8 r, r < RB
        const long long row0 = (long long)mb * BLOCK_M + rb;
        if (row0 >= p.M) break;
        uint4 rq[RB];
#pragma unroll
        for (int r = 0; r < RB; ++r) {
          const long long row = row0 + 8 * r;
          rq[r] = make_uint4(0, 0, 0, 0);
          if (reads_resid && row < p.M)
            rq[r] = *reinterpret_cast<const uint4*>(p.resid + bb * p.resid_bs + row * p.ldr + n);
        }
#pragma unroll
        for (int r = 0; r < RB; ++r) {
          const long long row = row0 + 8 * r;
          if (row >= p.M) break;
          float v[8];
          unpack_bf16x8(*reinterpret_cast<const uint4*>(stg + (rb + 8 * r) * SROW + cg * 16), v);
          epilogue_group(epi, v, rq[r], gq, out_base + row * ld + n);
        }
      }
    }
  }
}

template <int MODE, bool LORA = false>
int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, GemmParams p, cudaStream_t stream,
                const LoraParams<LORA>& lx = LoraParams<LORA>{}) {
  static_assert(!LORA || MODE == 0, "the LoRA K-extension is forward-only");
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gemm_bf16_kernel<MODE, LORA>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         PP_SMEM_BYTES);
    if (e != cudaSuccess) return cuda_err(e, "gemm smem attribute");
    attr_set = true;
  }
  p.m_blocks_per_batch = (p.M + BLOCK_M - 1) / BLOCK_M;
  p.num_m_blocks = p.batch * p.m_blocks_per_batch;
  p.num_n_blocks = (p.N + BLOCK_N - 1) / BLOCK_N;
  p.panel_n = 16;
  const int num_tiles = p.num_m_blocks * p.num_n_blocks;
  const int grid = std::min(num_tiles, device_info().num_sms);   // persistent: at most one CTA per SM
  int k_ext = 0;
  bool down = false;
  if constexpr (LORA) {
    k_ext = lx.num_kb2 * BLOCK_K;
    down = lx.colscale != nullptr;
  }
  const double kk = MODE == 2 ? (double)p.kbatch * p.K : (double)p.K + k_ext;
  prof_begin(KC_GEMM, stream);
  gemm_bf16_kernel<MODE, LORA><<<grid, THREADS, PP_SMEM_BYTES, stream>>>(tmA, tmB, p, lx);
  {
    char tag_[96];
    if (LORA)
      snprintf(tag_, sizeof tag_, "gemm lora %dx%dx%d+%d b%d e%d%s", p.M, p.N, p.K, k_ext, p.batch, p.epi,
               down ? " down" : "");
    else
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

// LoRA operands of one forward launch (see LoraParams): T [batch, M, r_pad] (row pitch ldt, batch pitch t_bs) and
// Bcat [N, r_pad] (pitch ldbc) extend the contraction by r_pad (a multiple of 64; 0: no extension); colscale != NULL
// makes the launch a down projection.
struct LoraExt {
  const void* T;
  int64_t ldt, t_bs;
  const void* Bc;
  int64_t ldbc;
  int r_pad;
  const float* colscale;
  float cs_mul;
};

static int gemm_bf16_impl(const void* A, int64_t lda, int64_t a_bs, const void* W, int64_t ldw,
              const void* bias, void* out, int64_t ldc, int64_t out_bs, int batch, int M, int N,
              int K, int epilogue, const void* resid, int64_t ldr, int64_t resid_bs, const void* gate,
              int64_t gate_ld, const QkvExtra* qx, cudaStream_t stream, const LoraExt* lx = nullptr) {
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
  if (!lx) return launch_gemm<0>(tmA, tmB, p, stream);

  if (lx->r_pad < 0 || (lx->r_pad % BLOCK_K)) return B2F_ERR_INVALID;
  if (lx->colscale && (lx->r_pad || bias || epilogue != B2F_EPI_BIAS)) return B2F_ERR_INVALID;
  if (!lx->colscale && !lx->r_pad) return B2F_ERR_INVALID;
  if (lx->colscale && (reinterpret_cast<uintptr_t>(lx->colscale) & 15)) return B2F_ERR_ALIGN;
  LoraParams<true> lp;
  lp.tmT = tmA;   // unread without an extension
  lp.tmBc = tmB;
  lp.num_kb2 = lx->r_pad / BLOCK_K;
  lp.colscale = lx->colscale;
  lp.cs_mul = lx->cs_mul;
  if (lx->r_pad) {
    if (!lx->T || !lx->Bc) return B2F_ERR_INVALID;
    if ((lx->ldt & 7) || (lx->t_bs & 7) || (lx->ldbc & 7) || lx->ldt < lx->r_pad || lx->ldbc < lx->r_pad ||
        ((reinterpret_cast<uintptr_t>(lx->T) | reinterpret_cast<uintptr_t>(lx->Bc)) & 15))
      return B2F_ERR_ALIGN;
    rc = make_tmap_3d_rows(&lp.tmT, lx->T, (uint64_t)lx->r_pad, (uint64_t)M, (uint64_t)batch, (uint64_t)lx->ldt,
                           batch > 1 ? (uint64_t)lx->t_bs : (uint64_t)M * lx->ldt);
    if (rc != B2F_OK) return rc;
    rc = make_tmap_2d_bf16(&lp.tmBc, lx->Bc, (uint64_t)N, (uint64_t)lx->r_pad, (uint64_t)lx->ldbc, BLOCK_N, BLOCK_K);
    if (rc != B2F_OK) return rc;
  }
  return launch_gemm<0, true>(tmA, tmB, p, stream, lp);
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

// ---------------------------------------------------------------------------------------------------- LoRA
// out = epi(A W^T + T Bcat^T + bias): the forward GEMM with r_pad / 64 extra k-blocks per tile (LoraExt).
int gemm_bf16_lora(const void* A, int64_t lda, int64_t a_bs, const void* W, int64_t ldw, const void* bias, void* out,
                   int64_t ldc, int64_t out_bs, int batch, int M, int N, int K, int epilogue, const void* resid,
                   int64_t ldr, int64_t resid_bs, const void* gate, int64_t gate_ld, const void* T, int64_t ldt,
                   int64_t t_bs, const void* Bc, int64_t ldbc, int r_pad, cudaStream_t stream) {
  if (epilogue == B2F_EPI_QKV_NORM_ROPE || r_pad <= 0) return B2F_ERR_INVALID;
  const LoraExt lx{T, ldt, t_bs, Bc, ldbc, r_pad, nullptr, 1.f};
  return gemm_bf16_impl(A, lda, a_bs, W, ldw, bias, out, ldc, out_bs, batch, M, N, K, epilogue, resid, ldr,
                        resid_bs, gate, gate_ld, nullptr, stream, &lx);
}

int gemm_qkv_norm_rope_lora(const void* A, int64_t lda, int64_t a_bs, const void* W, int64_t ldw, const void* bias,
                            void* out, int64_t ldc, int64_t out_bs, int batch, int M, int d_model, int K,
                            const void* nw_q, const void* nw_k, const float* cos, const float* sin, int rope_row0,
                            float eps, int n_extra, void* out_extra, int64_t ld_extra, int64_t bs_extra,
                            int epi_extra, const void* T, int64_t ldt, int64_t t_bs, const void* Bc, int64_t ldbc,
                            int r_pad, cudaStream_t stream) {
  if (r_pad <= 0) return B2F_ERR_INVALID;
  QkvExtra qx{nw_q, nw_k, cos, sin, rope_row0, d_model, eps, n_extra, epi_extra, out_extra, ld_extra, bs_extra};
  const LoraExt lx{T, ldt, t_bs, Bc, ldbc, r_pad, nullptr, 1.f};
  return gemm_bf16_impl(A, lda, a_bs, W, ldw, bias, out, ldc, out_bs, batch, M, 3 * d_model + n_extra, K,
                        B2F_EPI_QKV_NORM_ROPE, nullptr, 0, 0, nullptr, 0, &qx, stream, &lx);
}

// LoRA down projection: out[batch, M, N] = bf16((A W^T)[., n] * fp32(colscale[n] * cs_mul)), W = Acat [N, K].
int gemm_colscale(const void* A, int64_t lda, int64_t a_bs, const void* W, int64_t ldw, void* out, int64_t ldc,
                  int64_t out_bs, int batch, int M, int N, int K, const float* colscale, float cs_mul,
                  cudaStream_t stream) {
  if (!colscale) return B2F_ERR_INVALID;
  const LoraExt lx{nullptr, 0, 0, nullptr, 0, 0, colscale, cs_mul};
  return gemm_bf16_impl(A, lda, a_bs, W, ldw, nullptr, out, ldc, out_bs, batch, M, N, K, B2F_EPI_BIAS, nullptr, 0, 0,
                        nullptr, 0, nullptr, stream, &lx);
}

}  // namespace b2f
