// Persistent, warp-specialised bf16 GEMM for sm_90a with ping-pong consumers:  out[M,N] = epi(A[M,K] · W[N,K]^T + bias).
//
//   grid                  min(tiles, SMs) CTAs; CTA b takes the 128 x 128 tiles b, b + grid, ... in panel order
//   warpgroup 0 (1 lane)  TMA producer      cp.async.bulk.tensor → 128B-swizzled smem ring of STAGES stages, streamed
//                                           across tile boundaries (setmaxnreg.dec to 40 registers)
//   warpgroups 1, 2       wgmma consumers   each owns whole tiles, alternating (the CTA's tiles 0, 2, ... / 1, 3, ...):
//                                           two m64n128k16 per k16 step, 128 fp32 accumulators per thread
//                                           (setmaxnreg.inc to 232); named barriers make them take turns on the main
//                                           loop, so one runs its MMAs while the other runs its epilogue
//   FP8 mode              e4m3 A and W (per-token / per-channel fp32 scales), m64n128k32 e4m3 wgmma; see Fp8Params
//   epilogue              x = bf16(acc + bias) from registers → the consumer's own bf16 staging tile →
//                         act/gate/resid → global with 16-byte accesses, 16 threads per row; a fused QKV head runs one
//                         thread per row (the epilogue tail, shared with the wide tile); the fp32 wgrad output goes
//                         straight from registers
//
// gemm_wide_kernel     the plain forward GEMM on 128 x 256 tiles for the loop's large linears: both consumers on one tile,
//                      one m64n256k16 each per k16 step, a 3-stage ring of 48 KB stages, the same epilogue tail with
//                      32 threads per row; launch_gemm picks the tile per launch from the shape (tile_width)
//
// Every output element sees the same k16 accumulation order as a one-tile-per-CTA kernel with the same k-blocks, on
// either tile.
// Both operands of the forward GEMM are K-major ([rows, K] row-major), which is what nn.Linear stores
// (SURVEY.md A.6) — no transposes anywhere.  The tile shape and ring layout are shared with conv.cu (gemm_sm90.cuh).
//
// Replaces: torch.nn.functional.linear → cuBLASLt (diffusers FluxTransformer2DModel linears,
// reference call site univa/utils/flux_pipeline.py:1067; SURVEY.md §2b row 1).
#include <algorithm>
#include <cstdlib>

#include "gemm_sm90.cuh"

namespace b2f {

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

// One 128-column head of a fused QKV projection for one token, from its row of the staged tile x = bf16(acc + bias):
//   y = bf16(x * rsqrt(mean(x^2) + eps));  z = bf16(y * w);
//   out = bf16(z * cos + rot(z) * sin)        (diffusers RMSNorm + apply_rotary_emb, SURVEY.md A.2)
// — the same rounding chain as rmsnorm_rope_out_kernel, but without the extra HBM round trip.  The sum of squares runs over
// the columns in order, one thread per row.  Every rounding is the packed cvt.rn.bf16x2.
__device__ __forceinline__ void epilogue_head_norm_rope(const GemmParams& p, const uint8_t* srow, int n_head0,
                                                        long long row, __nv_bfloat16* out_row, bool is_k) {
  const __nv_bfloat16* w = is_k ? p.nw_k : p.nw_q;
  float ss = 0.f;
#pragma unroll 4
  for (int g = 0; g < BLOCK_N / 8; ++g) {
    float x[8];
    // uint4(...) unpacks a register copy (here and below): unpacking through a reference to the staged bytes changes
    // this tile's register allocation
    unpack8(uint4(*reinterpret_cast<const uint4*>(srow + g * 16)), x);
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
    unpack8(uint4(*reinterpret_cast<const uint4*>(srow + g * 16)), x);
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

// ---------------------------------------------------------------------------------------------------- epilogue tail
// What both forward kernels run once a consumer's accumulators are final: stage_bias into the consumer's staging rows,
// tile_out to find where the tile goes, then epilogue_head_norm_rope or epilogue_rows from the staged rows.

// x = bf16(acc + bias) of a thread's 2 x 2 accumulator group a[0..3] (rows r, r + 8; columns col, col + 1, whose bias
// is b2) into a staging tile of PITCH bytes per row, s pointing at (r, col).
template <int PITCH>
__device__ __forceinline__ void stage_bias(uint8_t* s, const float* a, bool has_bias, float2 b2) {
  float x0 = a[0], x1 = a[1], x2 = a[2], x3 = a[3];
  if (has_bias) {
    x0 += b2.x;
    x1 += b2.y;
    x2 += b2.x;
    x3 += b2.y;
  }
  *reinterpret_cast<uint32_t*>(s) = pack_bf16x2(x0, x1);
  *reinterpret_cast<uint32_t*>(s + 8 * PITCH) = pack_bf16x2(x2, x3);
}

// Where the tile whose first column is n_tile0, of batch item bb, goes.  With the fused QKV epilogue a tile of Q or K
// heads (norm 0 / 1) goes through epilogue_head_norm_rope, a V tile is a plain bias store, and a tile at or past
// split_n goes to the second output block with epi2.  Every other tile stores epi(x) at base + row * ld + column.
struct TileOut {
  int norm;   // 0 / 1: RMS-normalised Q / K heads; -1: none
  int epi;
  __nv_bfloat16* base;
  long long ld;
};
// One return for every tile: an early return for the Q / K tiles merges base into a value NVVM no longer knows to be a
// global pointer, and the epilogues' 16-byte stores become generic ones.
__device__ __forceinline__ TileOut tile_out(const GemmParams& p, int n_tile0, int bb) {
  TileOut o{-1, p.epi, p.out + bb * p.out_bs, p.ldc};
  if (o.epi == B2F_EPI_QKV_NORM_ROPE) {
    const int which = n_tile0 / p.d_model;   // 0 = Q, 1 = K, 2 = V, >= 3: second output block
    if (which < 2) {
      o.norm = which;
    } else {
      const bool second = p.split_n > 0 && n_tile0 >= p.split_n;
      o.epi = second ? p.epi2 : B2F_EPI_BIAS;
      if (second) {
        o.base = p.out2 + bb * p.out2_bs - p.split_n;
        o.ld = p.ldc2;
      }
    }
  }
  return o;
}

// epi over ROWS staged rows of PITCH bytes, global rows row_c, row_c + 1, ...: TPR threads per row, one 8-column group
// each, so the 128 threads of a consumer cover STEP = 128 / TPR rows at a time.  A thread's rows go in batches of RB
// whose residual / pre-activation loads are all issued before the first store, so their latencies overlap; a batch,
// not all of them, keeps the unrolled activation code small.  BWD: the backward epilogues (DGELU / DSILU) can occur.
template <int TPR, int ROWS, int PITCH, bool BWD>
__device__ __forceinline__ void epilogue_rows(const GemmParams& p, const TileOut& o, const uint8_t* stg, int tid,
                                              long long row_c, int n_tile0, int bb) {
  constexpr int STEP = 128 / TPR, RB = 4;
  const int cg = tid % TPR;
  const int n = n_tile0 + 8 * cg;
  if (n >= p.N) return;
  const bool reads_resid = o.epi == B2F_EPI_GATE_RESID || o.epi == B2F_EPI_RESID ||
                           (BWD && (o.epi == B2F_EPI_DGELU || o.epi == B2F_EPI_DSILU));
  const __nv_bfloat16* gate_row = p.gate ? p.gate + (long long)bb * p.gate_ld : nullptr;
  const uint4 gq = o.epi == B2F_EPI_GATE_RESID ? __ldg(reinterpret_cast<const uint4*>(gate_row + n))
                                               : make_uint4(0, 0, 0, 0);
#pragma unroll 1
  for (int rb = tid / TPR; rb < ROWS; rb += STEP * RB) {   // staged rows rb + STEP r, r < RB
    const long long row0 = row_c + rb;
    if (row0 >= p.M) break;
    uint4 rq[RB];
#pragma unroll
    for (int r = 0; r < RB; ++r) {
      const long long row = row0 + STEP * r;
      rq[r] = make_uint4(0, 0, 0, 0);
      if (reads_resid && row < p.M)
        rq[r] = *reinterpret_cast<const uint4*>(p.resid + bb * p.resid_bs + row * p.ldr + n);
    }
#pragma unroll
    for (int r = 0; r < RB; ++r) {
      const long long row = row0 + STEP * r;
      if (row >= p.M) break;
      float v[8];
      unpack8(uint4(*reinterpret_cast<const uint4*>(stg + (rb + STEP * r) * PITCH + cg * 16)), v);
      epilogue_group(o.epi, v, rq[r], gq, o.base + row * o.ld + n);
    }
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

// FP8 mode (FP8 = true, MODE 0 only): A and W are e4m3 with one fp32 scale per row of A (a_scale, per token) and per
// row of W (w_scale, per output channel).  A k-block is still 128 bytes of K, now 128 elements, so the ring, the swizzle
// and the 32-byte descriptor step are unchanged; each k32 step is one m64n128k32 e4m3 wgmma.  The staged value is
// x = bf16(fmaf(acc, fp32(a_scale[m] * w_scale[n]), bias[n])) (bf16(acc * scale) without a bias), and every epilogue
// runs from x as in the bf16 kernel.  FP8 = false has an empty parameter and compiles to the plain kernel.
// FP8 with LORA (an unfused adapter on an FP8 linear; no colscale): the bf16 (T, Bcat) k-blocks are 128 bytes wide too,
// so they follow the e4m3 ones through the same ring.  Before its first LoRA k-block a consumer drains its MMAs and
// scales its accumulators in registers, acc *= fp32(a_scale[m] * w_scale[n]); the LoRA k-blocks then accumulate into
// them with m64n128k16 bf16 wgmma, and the staged value is x = bf16(acc + bias) as in the bf16 kernel.  The drain costs
// one emptied pipeline per tile; pre-scaling T by 1 / a_scale and Bcat by 1 / w_scale would avoid it, but on the loop's
// K = 3072 shapes the drain and the extra k-block together cost 6-16 % of the FP8 GEMM (H100 80GB HBM3, 700 W,
// scripts/bench_lora.py --fp8), small beside the adapter's down projection, so the scaling stays in registers.
template <bool FP8>
struct Fp8Params {};
template <>
struct Fp8Params<true> {
  const float* a_scale;
  long long a_scale_bs;
  const float* w_scale;
};

// One k-block of a consumer's main loop: wait for its stage, issue its MMAs (m64n128k32 e4m3 or m64n128k16 bf16, two
// per k step: rows 0..63 and 64..127 of the tile), and hand the previous stage back to the producer once they are done.
template <bool E4M3, int TA, int TB>
__device__ __forceinline__ void consume_kblock(float (&acc0)[64], float (&acc1)[64], uint64_t* full, uint64_t* empty,
                                               int& stage, uint32_t& phase, int& prev, uint64_t da0,
                                               uint64_t da1, uint64_t db0, int lane) {
  constexpr int A_KSTEP = TA ? 2048 : 32;
  constexpr int B_KSTEP = TB ? 2048 : 32;
  mbar_wait(&full[stage], phase);
  const uint64_t soff = uint64_t((stage * STAGE_BYTES) >> 4);
  reg_fence(acc0);
  reg_fence(acc1);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < BLOCK_K / 16; ++k) {
    const uint64_t ka = soff + uint64_t((k * A_KSTEP) >> 4), kb16 = soff + uint64_t((k * B_KSTEP) >> 4);
    if constexpr (E4M3) {
      wgmma_m64n128k32_e4m3_ss(acc0, da0 + ka, db0 + kb16, 1u);
      wgmma_m64n128k32_e4m3_ss(acc1, da1 + ka, db0 + kb16, 1u);
    } else {
      wgmma_m64n128_ss<TA, TB>(acc0, da0 + ka, db0 + kb16, 1u);
      wgmma_m64n128_ss<TA, TB>(acc1, da1 + ka, db0 + kb16, 1u);
    }
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

// FP8 with LORA: acc *= fp32(a_scale[m] * w_scale[n]) on a consumer's drained accumulators (element j of a thread is
// row 16 w + lane / 4 + 8 ((j / 2) & 1), column 8 (j / 4) + 2 (lane % 4) + (j & 1) of its 64-row half; scales are 0
// past M and N, as in the FP8 epilogue).
__device__ __forceinline__ void fp8_rescale(const GemmParams& p, const Fp8Params<true>& fx, int bb, int mb, int n_blk,
                                            int w, int lane, float (&acc0)[64], float (&acc1)[64]) {
  const int r_lo = 16 * w + (lane >> 2);
  float sa[2][2];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const long long row = (long long)mb * BLOCK_M + 64 * h + r_lo + 8 * rr;
      sa[h][rr] = row < p.M ? __ldg(fx.a_scale + bb * fx.a_scale_bs + row) : 0.f;
    }
#pragma unroll
  for (int j = 0; j < BLOCK_N / 8; ++j) {
    const int n = n_blk * BLOCK_N + 8 * j + 2 * (lane & 3);
    const float2 ws2 = n < p.N ? __ldg(reinterpret_cast<const float2*>(fx.w_scale + n)) : make_float2(0.f, 0.f);
    acc0[4 * j] *= sa[0][0] * ws2.x;
    acc0[4 * j + 1] *= sa[0][0] * ws2.y;
    acc0[4 * j + 2] *= sa[0][1] * ws2.x;
    acc0[4 * j + 3] *= sa[0][1] * ws2.y;
    acc1[4 * j] *= sa[1][0] * ws2.x;
    acc1[4 * j + 1] *= sa[1][0] * ws2.y;
    acc1[4 * j + 2] *= sa[1][1] * ws2.x;
    acc1[4 * j + 3] *= sa[1][1] * ws2.y;
  }
}

template <int MODE, bool LORA = false, bool FP8 = false>
__global__ void __launch_bounds__(THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const GemmParams p, const __grid_constant__ LoraParams<LORA> lx,
                 const __grid_constant__ Fp8Params<FP8> fx) {
  constexpr int TA = MODE == 2, TB = MODE >= 1;
  constexpr int KB_ELEMS = FP8 ? BLOCK_K * 2 : BLOCK_K;   // elements of K per 128-byte k-block
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
  const int num_kb = MODE == 2 ? p.kbatch * p.kb_per_batch : (p.K + KB_ELEMS - 1) / KB_ELEMS;
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
            int kc = kb * KB_ELEMS;
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
    // FP8 with LoRA: the e4m3 k-blocks, then the scales, then the bf16 LoRA k-blocks, each in a loop of one wgmma type
    // (a branch between the two types inside one loop makes ptxas serialize every wgmma of the kernel)
    const int kb_main = FP8 && LORA ? num_kb : num_kb_all;
    for (int kb = 0; kb < kb_main; ++kb)
      consume_kblock<FP8, TA, TB>(acc0, acc1, full, empty, stage, phase, prev, da0, da1, db0, lane);
    if constexpr (FP8 && LORA) {
      wgmma_wait<0>();
      reg_fence(acc0);
      reg_fence(acc1);
      fp8_rescale(p, fx, bb, mb, n_blk, w, lane, acc0, acc1);
      for (int kb = num_kb; kb < num_kb_all; ++kb)
        consume_kblock<false, 0, 0>(acc0, acc1, full, empty, stage, phase, prev, da0, da1, db0, lane);
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
    float sa[2][2];   // FP8: the token scales of this thread's rows 64 h + r_lo + 8 rr (0 past M)
    if constexpr (FP8 && !LORA) {
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const long long row = (long long)mb * BLOCK_M + 64 * h + r_lo + 8 * rr;
          sa[h][rr] = row < p.M ? __ldg(fx.a_scale + bb * fx.a_scale_bs + row) : 0.f;
        }
    }
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
      if constexpr (FP8 && !LORA) {
        const float2 ws2 = n < p.N ? __ldg(reinterpret_cast<const float2*>(fx.w_scale + n)) : make_float2(0.f, 0.f);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float* a = h ? acc1 : acc0;
          const float s0 = sa[h][0] * ws2.x, s1 = sa[h][0] * ws2.y, s2 = sa[h][1] * ws2.x, s3 = sa[h][1] * ws2.y;
          float x0, x1, x2, x3;
          if (has_bias) {
            x0 = fmaf(a[4 * j], s0, b2.x);
            x1 = fmaf(a[4 * j + 1], s1, b2.y);
            x2 = fmaf(a[4 * j + 2], s2, b2.x);
            x3 = fmaf(a[4 * j + 3], s3, b2.y);
          } else {
            x0 = a[4 * j] * s0;
            x1 = a[4 * j + 1] * s1;
            x2 = a[4 * j + 2] * s2;
            x3 = a[4 * j + 3] * s3;
          }
          uint8_t* s0p = stg + (64 * h + r_lo) * SROW + col * 2;
          *reinterpret_cast<uint32_t*>(s0p) = pack_bf16x2(x0, x1);
          *reinterpret_cast<uint32_t*>(s0p + 8 * SROW) = pack_bf16x2(x2, x3);
        }
      } else if constexpr (LORA) {
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
          if (lx.colscale) {
            x0 *= cs2.x;
            x1 *= cs2.y;
            x2 *= cs2.x;
            x3 *= cs2.y;
          }
          uint8_t* s0 = stg + (64 * h + r_lo) * SROW + col * 2;
          *reinterpret_cast<uint32_t*>(s0) = pack_bf16x2(x0, x1);
          *reinterpret_cast<uint32_t*>(s0 + 8 * SROW) = pack_bf16x2(x2, x3);
        }
      } else {
#pragma unroll
        for (int h = 0; h < 2; ++h)
          stage_bias<SROW>(stg + (64 * h + r_lo) * SROW + col * 2, (h ? acc1 : acc0) + 4 * j, has_bias, b2);
      }
    }
    named_bar_sync(BAR_EPI + c, 128);

    // 16 threads per row: a warp reads and writes two 256-byte row segments
    const int n_tile0 = n_blk * BLOCK_N;
    const TileOut o = tile_out(p, n_tile0, bb);
    if (o.norm >= 0) {
      // one normalised head per tile: one thread per row
      const long long row = (long long)mb * BLOCK_M + tid;
      if (row < p.M) epilogue_head_norm_rope(p, stg + tid * SROW, n_tile0, row, o.base + row * o.ld, o.norm == 1);
      continue;
    }
    epilogue_rows<16, BLOCK_M, SROW, MODE != 0>(p, o, stg, tid, (long long)mb * BLOCK_M, n_tile0, bb);
  }
}

// ---------------------------------------------------------------------------------------------------- the wide tile
// The plain forward GEMM (MODE 0, bf16, no LoRA, no FP8) on 128 x 256 tiles, for the large linears of the denoising
// loop.  Both consumer warpgroups work on the same tile: consumer c owns rows [64 c, 64 c + 64) and issues one
// m64n256k16 per k16 step, 128 fp32 accumulators per thread as in the ping-pong kernel.  Per unit of tensor work this
// reads about 17 % fewer operand bytes from shared memory (2 KB of A and 8 KB of W per 64 x 256 x 16 MACs instead of
// 2 + 4 KB per 64 x 128 x 16) and moves 25 % fewer bytes through L2 and TMA (48 KB per 128 x 256 x 64 tile-k-block
// instead of 32 KB per 128 x 128 x 64).  The price is that the epilogues no longer overlap the MMAs; the producer still
// streams the next tile's first k-blocks into the ring while they run.  Each consumer runs the epilogue tail on its own
// 64 rows, so the two consumers meet only at the ring's barriers.
// A stage is 48 KB: three stages and a 128 x (256 + 8) bf16 staging tile take 210 KB of the 227 KB (211 KB with the
// barriers and the alignment pad); a fourth stage would leave room for only half the staging tile.  W arrives as two
// 128-row TMA boxes, so both tiles share one W map.
// Every output element sees the same k16 steps in the same order, and the same rounding chain from x = bf16(acc + bias),
// as on the 128 x 128 tile.
// Sharing the W tile across a 2-CTA cluster along M (each CTA loads its A tile and half of W, multicast to both; each
// consumer warp releases a stage to both CTAs' empty barriers; grid from cudaOccupancyMaxActiveClusters, which gave 66)
// was built and gave bit-identical results, but ran 26-48 % slower on the loop's shapes (sustained TFLOP/s, H100 SXM
// 80 GB, 700 W, cluster against this kernel: proj_out 405-406 / 606-611, ff2 433-434 / 653-660, ff1 428-431 / 576-578,
// to_out 410-412 / 560, single-block qkv+mlp 409-410 / 548-554, text ff1 227-230 / 433-439), so each CTA loads its own
// W tile.
constexpr int WIDE_N = 256;
constexpr int WIDE_STAGES = 3;
constexpr int WIDE_STAGE_BYTES = A_BYTES + WIDE_N * BLOCK_K * 2;
constexpr int WIDE_SROW = WIDE_N * 2 + 16;   // as SROW: 16-byte accesses of 8 rows hit 32 banks
constexpr int WIDE_SMEM_BYTES = WIDE_STAGES * WIDE_STAGE_BYTES + BLOCK_M * WIDE_SROW + 2 * WIDE_STAGES * 8 + 1024;
static_assert(WIDE_SMEM_BYTES <= 227 * 1024, "wide tile exceeds the shared memory of an SM");

__global__ void __launch_bounds__(THREADS, 1)
gemm_wide_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* ring = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(ring + WIDE_STAGES * WIDE_STAGE_BYTES + BLOCK_M * WIDE_SROW);
  uint64_t* empty = full + WIDE_STAGES;
  const int wg = threadIdx.x >> 7;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < WIDE_STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 8);   // one arrive per consumer warp: both consumers read every stage
    }
    fence_mbar_init();
  }
  __syncthreads();

  const int num_tiles = p.num_m_blocks * p.num_n_blocks;
  const int n_local = (num_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  const int num_kb = (p.K + BLOCK_K - 1) / BLOCK_K;

  if (wg == 0) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int i = 0; i < n_local; ++i) {
        int n_blk, bb, mb;
        tile_origin(p, blockIdx.x + i * gridDim.x, n_blk, bb, mb);
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          uint8_t* sa = ring + stage * WIDE_STAGE_BYTES;
          uint8_t* sb = sa + A_BYTES;
          mbar_expect_tx(&full[stage], WIDE_STAGE_BYTES);
          tma_load_3d(sa, &tmA, &full[stage], kb * BLOCK_K, mb * BLOCK_M, bb);
          tma_load_2d(sb, &tmB, &full[stage], kb * BLOCK_K, n_blk * WIDE_N);
          tma_load_2d(sb + B_BYTES, &tmB, &full[stage], kb * BLOCK_K, n_blk * WIDE_N + BLOCK_N);
          if (++stage == WIDE_STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
    return;
  }
  setmaxnreg_inc<CONSUMER_REGS>();

  const int c = wg - 1;
  const int tid = threadIdx.x & 127, w = tid >> 5, lane = tid & 31;
  uint8_t* stg = ring + WIDE_STAGES * WIDE_STAGE_BYTES + 64 * c * WIDE_SROW;   // this consumer's 64 staged rows
  const uint32_t ring_u = smem_u32(ring);
  const uint64_t da0 = make_sdesc_sw128(ring_u + 8192 * c, 16, 1024);   // rows 64 c.. of the A tile start 8 KB c in
  const uint64_t db0 = make_sdesc_sw128(ring_u + A_BYTES, 16, 1024);
  int stage = 0;
  uint32_t phase = 0;
  for (int i = 0; i < n_local; ++i) {
    int n_blk, bb, mb;
    tile_origin(p, blockIdx.x + i * gridDim.x, n_blk, bb, mb);

    float acc[128];
#pragma unroll
    for (int j = 0; j < 128; ++j) acc[j] = 0.f;
    int prev = -1;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&full[stage], phase);
      const uint64_t soff = uint64_t((stage * WIDE_STAGE_BYTES) >> 4);
      reg_fence(acc);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BLOCK_K / 16; ++k) {
        const uint64_t ks = soff + uint64_t((k * 32) >> 4);
        wgmma_m64n256_ss<0, 0>(acc, da0 + ks, db0 + ks, 1u);
      }
      wgmma_commit();
      wgmma_wait<1>();   // the previous stage's MMAs are complete: hand it back to the producer
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[prev]);
      }
      prev = stage;
      if (++stage == WIDE_STAGES) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();
    reg_fence(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[prev]);

    // ---- epilogue of rows [64 c, 64 c + 64).  Accumulator element j of a thread is row 16 w + lane / 4 + 8 ((j / 2) & 1),
    // column 8 (j / 4) + 2 (lane % 4) + (j & 1) of this consumer's rows.
    const int r_lo = 16 * w + (lane >> 2);
    named_bar_sync(BAR_EPI + c, 128);   // this consumer's previous epilogue is done reading the staging rows
#pragma unroll
    for (int j = 0; j < WIDE_N / 8; ++j) {
      const int col = 8 * j + 2 * (lane & 3);
      const int n = n_blk * WIDE_N + col;
      const bool has_bias = p.bias && n < p.N;
      const float2 b2 = has_bias ? unpack_bf16x2(__ldg(reinterpret_cast<const uint32_t*>(p.bias + n))) : make_float2(0.f, 0.f);
      stage_bias<WIDE_SROW>(stg + r_lo * WIDE_SROW + col * 2, acc + 4 * j, has_bias, b2);
    }
    named_bar_sync(BAR_EPI + c, 128);

    // 32 threads per row: a warp reads and writes one 512-byte row segment
    const int n_tile0 = n_blk * WIDE_N;
    const long long row_c = (long long)mb * BLOCK_M + 64 * c;   // first row of this consumer's half
    const TileOut o = tile_out(p, n_tile0, bb);   // d_model % 256 == 0: both heads of a tile are in the same block
    if (o.norm >= 0) {
      // two normalised heads per tile: one thread per (row, head)
      const int r = tid & 63, h = tid >> 6;
      const long long row = row_c + r;
      if (row < p.M)
        epilogue_head_norm_rope(p, stg + r * WIDE_SROW + h * 256, n_tile0 + 128 * h, row, o.base + row * o.ld,
                                o.norm == 1);
      continue;
    }
    epilogue_rows<32, 64, WIDE_SROW, false>(p, o, stg, tid, row_c, n_tile0, bb);
  }
}

// 0: the launcher picks the tile; 128 / 256: b2f_gemm_set_tile_override forced it (tests and benchmarks).
int g_tile_override = 0;

// Time of one 128 x 256 tile over that of one 128 x 128 tile: WIDE_COST_LOOP + (WIDE_COST_EPI + WIDE_COST_NORM q) / K,
// q the share of the columns that are RMS-normalised QKV heads.  The main loop of the wide tile runs faster per FLOP
// (the constant part, below 2), but its epilogue no longer hides behind the other consumer's MMAs (the part that falls
// with K; the one-thread-per-head norm epilogue exposes more).  Fitted to scripts/bench_kernels.py --what loop
// --sustained on an H100 80GB HBM3 at 700 W: the ratio measured 1.89 (to_out, K 3072), 1.84 (ff1, K 3072), 1.98 (image
// QKV, K 3072), 1.56 (ff2, K 12288) and 1.53 (proj_out, K 15360).
constexpr double WIDE_COST_LOOP = 1.45, WIDE_COST_EPI = 1280.0, WIDE_COST_NORM = 530.0;

// Tile width of a plain forward launch.  A persistent launch takes ceil(tiles / SMs) rounds of tiles, so the wide tile
// wins where its rounds, each the cost ratio above times as long, add up to less.  On 132 SMs the single blocks'
// proj_out (M 8736, N 3072) runs 828 wide tiles in 7 rounds against 1656 narrow ones in 13 (7 x 1.53 < 13) and goes
// wide; the image QKV (2304 wide tiles in 18 rounds against 35, 18 x 1.98 > 35) and the M = 544 text linears with
// N = 3072 or 9216 (no fewer rounds on the wide tile) stay on 128.  The fused QKV epilogue needs d_model % 256 == 0, so
// that a wide tile never straddles the Q / K / V blocks.
int tile_width(const GemmParams& p) {
  if (p.epi == B2F_EPI_QKV_NORM_ROPE && p.d_model % WIDE_N) return BLOCK_N;
  if (g_tile_override) return g_tile_override;
  const int sms = device_info().num_sms;
  const long long rounds128 = ((long long)p.num_m_blocks * ((p.N + BLOCK_N - 1) / BLOCK_N) + sms - 1) / sms;
  const long long rounds256 = ((long long)p.num_m_blocks * ((p.N + WIDE_N - 1) / WIDE_N) + sms - 1) / sms;
  const double q = p.epi == B2F_EPI_QKV_NORM_ROPE ? 2.0 * p.d_model / p.N : 0.0;
  const double cost = WIDE_COST_LOOP + (WIDE_COST_EPI + WIDE_COST_NORM * q) / p.K;
  return rounds256 * cost < rounds128 ? WIDE_N : BLOCK_N;
}

template <int MODE, bool LORA = false, bool FP8 = false>
int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, GemmParams p, cudaStream_t stream,
                const LoraParams<LORA>& lx = LoraParams<LORA>{}, const Fp8Params<FP8>& fx = Fp8Params<FP8>{}) {
  static_assert(!LORA || MODE == 0, "the LoRA K-extension is forward-only");
  static_assert(!FP8 || MODE == 0, "FP8 is a mode of the forward GEMM");
  static bool attr_set = false, wide_attr_set = false;
  if (int rc = set_max_smem_once(attr_set, PP_SMEM_BYTES, "gemm smem attribute", gemm_bf16_kernel<MODE, LORA, FP8>))
    return rc;
  if (MODE == 0 && !LORA && !FP8)
    if (int rc = set_max_smem_once(wide_attr_set, WIDE_SMEM_BYTES, "gemm smem attribute", gemm_wide_kernel)) return rc;
  p.m_blocks_per_batch = (p.M + BLOCK_M - 1) / BLOCK_M;
  p.num_m_blocks = p.batch * p.m_blocks_per_batch;
  const int tile_n = MODE == 0 && !LORA && !FP8 ? tile_width(p) : BLOCK_N;
  p.num_n_blocks = (p.N + tile_n - 1) / tile_n;
  p.panel_n = 16 * BLOCK_N / tile_n;   // the same W-panel footprint on either tile
  const int num_tiles = p.num_m_blocks * p.num_n_blocks;
  const int grid = std::min(num_tiles, device_info().num_sms);   // persistent: at most one CTA per SM
  int k_ext = 0;
  bool down = false;
  if constexpr (LORA) {
    k_ext = lx.num_kb2 * BLOCK_K;
    down = lx.colscale != nullptr;
  }
  const double kk = MODE == 2 ? (double)p.kbatch * p.K : (double)p.K + k_ext;
  // operand bytes per row of A and of W: the main k-blocks (e4m3 or bf16), then the bf16 LoRA ones
  const double kbytes = (FP8 ? 1.0 : 2.0) * (MODE == 2 ? kk : (double)p.K) + 2.0 * k_ext;
  prof_begin(KC_GEMM, stream);
  if (tile_n == WIDE_N)
    gemm_wide_kernel<<<grid, THREADS, WIDE_SMEM_BYTES, stream>>>(tmA, tmB, p);
  else
    gemm_bf16_kernel<MODE, LORA, FP8><<<grid, THREADS, PP_SMEM_BYTES, stream>>>(tmA, tmB, p, lx, fx);
  {
    char tag_[96];
    if (FP8 && LORA)
      snprintf(tag_, sizeof tag_, "gemm fp8 lora %dx%dx%d+%d b%d e%d", p.M, p.N, p.K, k_ext, p.batch, p.epi);
    else if (FP8)
      snprintf(tag_, sizeof tag_, "gemm fp8 %dx%dx%d b%d e%d", p.M, p.N, p.K, p.batch, p.epi);
    else if (LORA)
      snprintf(tag_, sizeof tag_, "gemm lora %dx%dx%d+%d b%d e%d%s", p.M, p.N, p.K, k_ext, p.batch, p.epi,
               down ? " down" : "");
    else
      snprintf(tag_, sizeof tag_, "gemm m%d %dx%dx%d b%d e%d t%d", MODE, p.M, p.N, (int)kk, p.batch, p.epi, tile_n);
    prof_end_tagged(KC_GEMM, stream, 2.0 * p.batch * (double)p.M * p.N * kk,
                    kbytes * ((double)p.batch * p.M + p.N) + 2.0 * (double)p.batch * p.M * p.N, tag_);
  }
  B2F_LAUNCHED(tile_n == WIDE_N ? "gemm_wide_kernel" : "gemm_bf16_kernel", 1);
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

// FP8 operands of one forward launch: A and W are e4m3, a_scale fp32 [batch, M] (batch pitch a_scale_bs), w_scale
// fp32 [N].
struct Fp8Ext {
  const float* a_scale;
  int64_t a_scale_bs;
  const float* w_scale;
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

// Checks the LoRA operands of one launch and fills its LoraParams (tmA / tmB stand in for the maps of an absent
// extension; they are never read then).
static int lora_params(const LoraExt* lx, const CUtensorMap& tmA, const CUtensorMap& tmB, int batch, int M, int N,
                       const void* bias, int epilogue, LoraParams<true>* lp) {
  if (lx->r_pad < 0 || (lx->r_pad % BLOCK_K)) return B2F_ERR_INVALID;
  if (lx->colscale && (lx->r_pad || bias || epilogue != B2F_EPI_BIAS)) return B2F_ERR_INVALID;
  if (!lx->colscale && !lx->r_pad) return B2F_ERR_INVALID;
  if (lx->colscale && (reinterpret_cast<uintptr_t>(lx->colscale) & 15)) return B2F_ERR_ALIGN;
  lp->tmT = tmA;
  lp->tmBc = tmB;
  lp->num_kb2 = lx->r_pad / BLOCK_K;
  lp->colscale = lx->colscale;
  lp->cs_mul = lx->cs_mul;
  if (lx->r_pad) {
    if (!lx->T || !lx->Bc) return B2F_ERR_INVALID;
    if ((lx->ldt & 7) || (lx->t_bs & 7) || (lx->ldbc & 7) || lx->ldt < lx->r_pad || lx->ldbc < lx->r_pad ||
        ((reinterpret_cast<uintptr_t>(lx->T) | reinterpret_cast<uintptr_t>(lx->Bc)) & 15))
      return B2F_ERR_ALIGN;
    int rc = make_tmap_3d_rows(&lp->tmT, lx->T, (uint64_t)lx->r_pad, (uint64_t)M, (uint64_t)batch, (uint64_t)lx->ldt,
                               batch > 1 ? (uint64_t)lx->t_bs : (uint64_t)M * lx->ldt);
    if (rc != B2F_OK) return rc;
    rc = make_tmap_2d_bf16(&lp->tmBc, lx->Bc, (uint64_t)N, (uint64_t)lx->r_pad, (uint64_t)lx->ldbc, BLOCK_N, BLOCK_K);
    if (rc != B2F_OK) return rc;
  }
  return B2F_OK;
}

static int gemm_bf16_impl(const void* A, int64_t lda, int64_t a_bs, const void* W, int64_t ldw,
              const void* bias, void* out, int64_t ldc, int64_t out_bs, int batch, int M, int N,
              int K, int epilogue, const void* resid, int64_t ldr, int64_t resid_bs, const void* gate,
              int64_t gate_ld, const QkvExtra* qx, cudaStream_t stream, const LoraExt* lx = nullptr,
              const Fp8Ext* fx = nullptr) {
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (batch <= 0 || M <= 0 || N <= 0 || K <= 0 || !A || !W || !out) return B2F_ERR_INVALID;
  if ((K & 7) || (N & 7) || (lda & 7) || (ldw & 7) || (ldc & 7) || (a_bs & 7) || (out_bs & 7))
    return B2F_ERR_ALIGN;
  if (fx) {   // byte operands: TMA needs 16-byte pitches
    if ((lx && lx->colscale) || !fx->a_scale || !fx->w_scale) return B2F_ERR_INVALID;
    if ((K & 15) || (lda & 15) || (ldw & 15) || (a_bs & 15) || (reinterpret_cast<uintptr_t>(fx->w_scale) & 15) ||
        (reinterpret_cast<uintptr_t>(fx->a_scale) & 3))
      return B2F_ERR_ALIGN;
  }
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
  int rc;
  if (fx) {
    rc = make_tmap_u8_rows(&tmA, A, 3, (uint64_t)K, (uint64_t)M, (uint64_t)batch, (uint64_t)lda,
                           batch > 1 ? (uint64_t)a_bs : (uint64_t)M * lda);
    if (rc != B2F_OK) return rc;
    rc = make_tmap_u8_rows(&tmB, W, 2, (uint64_t)K, (uint64_t)N, 1, (uint64_t)ldw, 0);
    if (rc != B2F_OK) return rc;
    Fp8Params<true> fp;
    fp.a_scale = fx->a_scale;
    fp.a_scale_bs = fx->a_scale_bs;
    fp.w_scale = fx->w_scale;
    if (!lx || !lx->r_pad) return launch_gemm<0, false, true>(tmA, tmB, p, stream, LoraParams<false>{}, fp);
    LoraParams<true> lp;
    if ((rc = lora_params(lx, tmA, tmB, batch, M, N, bias, epilogue, &lp)) != B2F_OK) return rc;
    return launch_gemm<0, true, true>(tmA, tmB, p, stream, lp, fp);
  }
  rc = make_tmap_3d_rows(&tmA, A, (uint64_t)K, (uint64_t)M, (uint64_t)batch, (uint64_t)lda,
                         batch > 1 ? (uint64_t)a_bs : (uint64_t)M * lda);
  if (rc != B2F_OK) return rc;
  rc = make_tmap_2d_bf16(&tmB, W, (uint64_t)N, (uint64_t)K, (uint64_t)ldw, BLOCK_N, BLOCK_K);
  if (rc != B2F_OK) return rc;
  if (!lx) return launch_gemm<0>(tmA, tmB, p, stream);
  LoraParams<true> lp;
  if ((rc = lora_params(lx, tmA, tmB, batch, M, N, bias, epilogue, &lp)) != B2F_OK) return rc;
  return launch_gemm<0, true>(tmA, tmB, p, stream, lp);
}

extern "C" int b2f_gemm_bf16(const void* A, int64_t lda, int64_t a_bs, const void* W, int64_t ldw, const void* bias,
                             void* out, int64_t ldc, int64_t out_bs, int batch, int M, int N, int K, int epilogue,
                             const void* resid, int64_t ldr, int64_t resid_bs, const void* gate, int64_t gate_ld,
                             b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (epilogue == B2F_EPI_QKV_NORM_ROPE) return B2F_ERR_INVALID;  // needs the extended entry point
  return gemm_bf16_impl(A, lda, a_bs, W, ldw, bias, out, ldc, out_bs, batch, M, N, K, epilogue, resid, ldr,
                        resid_bs, gate, gate_ld, nullptr, stream);
}

extern "C" int b2f_gemm_set_tile_override(int tile_n) {
  if (tile_n != 0 && tile_n != BLOCK_N && tile_n != WIDE_N) return B2F_ERR_INVALID;
  g_tile_override = tile_n;
  return B2F_OK;
}

// dX[batch, M, N] = epi(dY[batch, M, K] . W[K, N]) with W exactly as nn.Linear stores it ([out = K, in = N]): the
// backward-data GEMM of every linear layer on the training path (reference train_denoiser.py:1172,
// accelerator.backward -> autograd of F.linear).  Epilogues: B2F_EPI_BIAS (plain store), B2F_EPI_DGELU /
// B2F_EPI_DSILU (times act'(u), u = `resid` [batch, M, N]), B2F_EPI_RESID (accumulate into another gradient).
extern "C" int b2f_gemm_dgrad(const void* dY, int64_t ldy, int64_t dy_bs, const void* W, int64_t ldw, void* dX,
                              int64_t ldx, int64_t dx_bs, int batch, int M, int N, int K, int epilogue, const void* aux,
                              int64_t ld_aux, int64_t aux_bs, b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
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
extern "C" int b2f_gemm_wgrad(const void* dY, int64_t ldy, int64_t dy_bs, const void* X, int64_t ldx, int64_t x_bs,
                              float* dW, int64_t ldw, int batch, int rows, int M, int N, int accumulate,
                              b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
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

extern "C" int b2f_gemm_qkv_norm_rope(const void* A, int64_t lda, int64_t a_bs, const void* W, int64_t ldw,
                                      const void* bias, void* out, int64_t ldc, int64_t out_bs, int batch, int M,
                                      int d_model, int K, const void* nw_q, const void* nw_k, const float* cos,
                                      const float* sin, int rope_row0, float eps, int n_extra, void* out_extra,
                                      int64_t ld_extra, int64_t bs_extra, int epi_extra, b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  QkvExtra qx{nw_q, nw_k, cos, sin, rope_row0, d_model, eps, n_extra, epi_extra, out_extra, ld_extra, bs_extra};
  return gemm_bf16_impl(A, lda, a_bs, W, ldw, bias, out, ldc, out_bs, batch, M, 3 * d_model + n_extra, K,
                        B2F_EPI_QKV_NORM_ROPE, nullptr, 0, 0, nullptr, 0, &qx, stream);
}

// ---------------------------------------------------------------------------------------------------- FP8
// b2f_gemm_bf16 / b2f_gemm_qkv_norm_rope with e4m3 operands and per-token / per-channel fp32 scales (Fp8Params).
extern "C" int b2f_gemm_fp8(const void* A, int64_t lda, int64_t a_bs, const float* a_scale, int64_t a_scale_bs,
                            const void* W, int64_t ldw, const float* w_scale, const void* bias, void* out, int64_t ldc,
                            int64_t out_bs, int batch, int M, int N, int K, int epilogue, const void* resid, int64_t ldr,
                            int64_t resid_bs, const void* gate, int64_t gate_ld, b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (epilogue == B2F_EPI_QKV_NORM_ROPE) return B2F_ERR_INVALID;
  const Fp8Ext fx{a_scale, a_scale_bs, w_scale};
  return gemm_bf16_impl(A, lda, a_bs, W, ldw, bias, out, ldc, out_bs, batch, M, N, K, epilogue, resid, ldr,
                        resid_bs, gate, gate_ld, nullptr, stream, nullptr, &fx);
}

extern "C" int b2f_gemm_qkv_norm_rope_fp8(const void* A, int64_t lda, int64_t a_bs, const float* a_scale,
                                          int64_t a_scale_bs, const void* W, int64_t ldw, const float* w_scale,
                                          const void* bias, void* out, int64_t ldc, int64_t out_bs, int batch, int M,
                                          int d_model, int K, const void* nw_q, const void* nw_k, const float* cos,
                                          const float* sin, int rope_row0, float eps, int n_extra, void* out_extra,
                                          int64_t ld_extra, int64_t bs_extra, int epi_extra, b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  QkvExtra qx{nw_q, nw_k, cos, sin, rope_row0, d_model, eps, n_extra, epi_extra, out_extra, ld_extra, bs_extra};
  const Fp8Ext fx{a_scale, a_scale_bs, w_scale};
  return gemm_bf16_impl(A, lda, a_bs, W, ldw, bias, out, ldc, out_bs, batch, M, 3 * d_model + n_extra, K,
                        B2F_EPI_QKV_NORM_ROPE, nullptr, 0, 0, nullptr, 0, &qx, stream, nullptr, &fx);
}

// b2f_gemm_fp8 / b2f_gemm_qkv_norm_rope_fp8 with the LoRA K-extension of b2f_gemm_bf16_lora: r_pad / 64 bf16 k-blocks of
// (T, Bcat) after the e4m3 ones, accumulated into the scaled FP8 accumulators (Fp8Params).
extern "C" int b2f_gemm_fp8_lora(const void* A, int64_t lda, int64_t a_bs, const float* a_scale, int64_t a_scale_bs,
                                 const void* W, int64_t ldw, const float* w_scale, const void* bias, void* out,
                                 int64_t ldc, int64_t out_bs, int batch, int M, int N, int K, int epilogue,
                                 const void* resid, int64_t ldr, int64_t resid_bs, const void* gate, int64_t gate_ld,
                                 const void* T, int64_t ldt, int64_t t_bs, const void* Bc, int64_t ldbc, int r_pad,
                                 b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (epilogue == B2F_EPI_QKV_NORM_ROPE || r_pad <= 0) return B2F_ERR_INVALID;
  const Fp8Ext fx{a_scale, a_scale_bs, w_scale};
  const LoraExt lx{T, ldt, t_bs, Bc, ldbc, r_pad, nullptr, 1.f};
  return gemm_bf16_impl(A, lda, a_bs, W, ldw, bias, out, ldc, out_bs, batch, M, N, K, epilogue, resid, ldr,
                        resid_bs, gate, gate_ld, nullptr, stream, &lx, &fx);
}

extern "C" int b2f_gemm_qkv_norm_rope_fp8_lora(const void* A, int64_t lda, int64_t a_bs, const float* a_scale,
                                               int64_t a_scale_bs, const void* W, int64_t ldw, const float* w_scale,
                                               const void* bias, void* out, int64_t ldc, int64_t out_bs, int batch,
                                               int M, int d_model, int K, const void* nw_q, const void* nw_k,
                                               const float* cos, const float* sin, int rope_row0, float eps,
                                               int n_extra, void* out_extra, int64_t ld_extra, int64_t bs_extra,
                                               int epi_extra, const void* T, int64_t ldt, int64_t t_bs, const void* Bc,
                                               int64_t ldbc, int r_pad, b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (r_pad <= 0) return B2F_ERR_INVALID;
  QkvExtra qx{nw_q, nw_k, cos, sin, rope_row0, d_model, eps, n_extra, epi_extra, out_extra, ld_extra, bs_extra};
  const Fp8Ext fx{a_scale, a_scale_bs, w_scale};
  const LoraExt lx{T, ldt, t_bs, Bc, ldbc, r_pad, nullptr, 1.f};
  return gemm_bf16_impl(A, lda, a_bs, W, ldw, bias, out, ldc, out_bs, batch, M, 3 * d_model + n_extra, K,
                        B2F_EPI_QKV_NORM_ROPE, nullptr, 0, 0, nullptr, 0, &qx, stream, &lx, &fx);
}

// ---------------------------------------------------------------------------------------------------- LoRA
// out = epi(A W^T + T Bcat^T + bias): the forward GEMM with r_pad / 64 extra k-blocks per tile (LoraExt).
extern "C" int b2f_gemm_bf16_lora(const void* A, int64_t lda, int64_t a_bs, const void* W, int64_t ldw,
                                  const void* bias, void* out, int64_t ldc, int64_t out_bs, int batch, int M, int N,
                                  int K, int epilogue, const void* resid, int64_t ldr, int64_t resid_bs,
                                  const void* gate, int64_t gate_ld, const void* T, int64_t ldt, int64_t t_bs,
                                  const void* Bc, int64_t ldbc, int r_pad, b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (epilogue == B2F_EPI_QKV_NORM_ROPE || r_pad <= 0) return B2F_ERR_INVALID;
  const LoraExt lx{T, ldt, t_bs, Bc, ldbc, r_pad, nullptr, 1.f};
  return gemm_bf16_impl(A, lda, a_bs, W, ldw, bias, out, ldc, out_bs, batch, M, N, K, epilogue, resid, ldr,
                        resid_bs, gate, gate_ld, nullptr, stream, &lx);
}

extern "C" int b2f_gemm_qkv_norm_rope_lora(const void* A, int64_t lda, int64_t a_bs, const void* W, int64_t ldw,
                                           const void* bias, void* out, int64_t ldc, int64_t out_bs, int batch, int M,
                                           int d_model, int K, const void* nw_q, const void* nw_k, const float* cos,
                                           const float* sin, int rope_row0, float eps, int n_extra, void* out_extra,
                                           int64_t ld_extra, int64_t bs_extra, int epi_extra, const void* T,
                                           int64_t ldt, int64_t t_bs, const void* Bc, int64_t ldbc, int r_pad,
                                           b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (r_pad <= 0) return B2F_ERR_INVALID;
  QkvExtra qx{nw_q, nw_k, cos, sin, rope_row0, d_model, eps, n_extra, epi_extra, out_extra, ld_extra, bs_extra};
  const LoraExt lx{T, ldt, t_bs, Bc, ldbc, r_pad, nullptr, 1.f};
  return gemm_bf16_impl(A, lda, a_bs, W, ldw, bias, out, ldc, out_bs, batch, M, 3 * d_model + n_extra, K,
                        B2F_EPI_QKV_NORM_ROPE, nullptr, 0, 0, nullptr, 0, &qx, stream, &lx);
}

// LoRA down projection: out[batch, M, N] = bf16((A W^T)[., n] * fp32(colscale[n] * cs_mul)), W = Acat [N, K].
extern "C" int b2f_gemm_colscale(const void* A, int64_t lda, int64_t a_bs, const void* W, int64_t ldw, void* out,
                                 int64_t ldc, int64_t out_bs, int batch, int M, int N, int K, const float* colscale,
                                 float cs_mul, b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!colscale) return B2F_ERR_INVALID;
  const LoraExt lx{nullptr, 0, 0, nullptr, 0, 0, colscale, cs_mul};
  return gemm_bf16_impl(A, lda, a_bs, W, ldw, nullptr, out, ldc, out_bs, batch, M, N, K, B2F_EPI_BIAS, nullptr, 0, 0,
                        nullptr, 0, nullptr, stream, &lx);
}

}  // namespace b2f
