// Building blocks of the warp-specialised wgmma GEMMs for sm_90a: the 128 x 128 x 64 tile, the STAGES-deep ring of
// 128B-swizzled A | B stages a TMA producer fills, and (for conv.cu) a one-tile-per-CTA consumer path.
//
// gemm.cu uses the tile and ring constants with its own persistent ping-pong kernel (each consumer warpgroup owns
// whole tiles; see there), and BLOCK_M / BLOCK_K / A_BYTES with its 128 x 256 forward tile (both consumers on one tile,
// W as two 128-row boxes of B_BYTES, its own 3-stage ring).  conv.cu uses everything below:
//   warpgroup 0 (1 lane)   TMA producer      cp.async.bulk.tensor -> 128B-swizzled smem ring of STAGES stages
//   warpgroups 1, 2        consumers         wgmma m64n128k16 on rows [64 c, 64 c + 64) of the 128 x 128 tile,
//                                            fp32 accumulators in registers
// After the main loop each consumer stages its accumulators in shared memory (row-major fp32), and the 256 consumer
// threads run the epilogue one output row per thread (two threads per row, 64 columns each).
#pragma once
#include "host_common.h"
#include "ptx.cuh"

namespace b2f {
namespace sm90 {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_N = 128;
constexpr int BLOCK_K = 64;      // 64 bf16 = 128 B = one swizzle row
constexpr int STAGES = 4;
constexpr int THREADS = 384;     // producer warpgroup + 2 consumer warpgroups
constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;
constexpr int B_BYTES = BLOCK_N * BLOCK_K * 2;
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int CROW = BLOCK_N + 4;                       // fp32 pitch of the staged accumulator tile (bank spread)
constexpr int C_BYTES = BLOCK_M * CROW * 4;
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + C_BYTES + 2 * STAGES * 8 + 1024;
constexpr int MN_BOX_BYTES = 64 * 64 * 2;              // one [64 k][64 mn] box of an MN-major operand

struct Smem {
  uint8_t* ring;
  float* cbuf;
  uint64_t* full;
  uint64_t* empty;
};

__device__ __forceinline__ Smem carve(uint8_t* smem_raw) {
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  Smem s;
  s.ring = base;
  s.cbuf = reinterpret_cast<float*>(base + STAGES * STAGE_BYTES);
  s.full = reinterpret_cast<uint64_t*>(base + STAGES * STAGE_BYTES + C_BYTES);
  s.empty = s.full + STAGES;
  return s;
}

__device__ __forceinline__ void init_barriers(const Smem& s) {
  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&s.full[i], 1);
      mbar_init(&s.empty[i], 8);   // one arrive per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();
}

// Consumer main loop of warpgroup `wg` (0 / 1).  TA / TB: A / B are MN-major.  A K-major A stage is [128 rows][64 k]
// (this warpgroup's 64 rows start 8 KB in for wg = 1); an MN-major one is two [64 k][64 m] boxes, box wg being this
// warpgroup's rows.  A K-major B stage is [128 n][64 k]; an MN-major one is two [64 k][64 n] boxes.
template <int TA, int TB>
__device__ __forceinline__ void mainloop(const Smem& s, int num_kb, int wg, float (&acc)[64]) {
  const uint32_t ring = smem_u32(s.ring);
  const uint64_t da0 = make_sdesc_sw128(ring + wg * 8192, TA ? MN_BOX_BYTES : 16, 1024);
  const uint64_t db0 = make_sdesc_sw128(ring + A_BYTES, TB ? MN_BOX_BYTES : 16, 1024);
  constexpr int A_KSTEP = TA ? 2048 : 32;
  constexpr int B_KSTEP = TB ? 2048 : 32;
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  int stage = 0, prev = -1;
  uint32_t phase = 0;
  for (int kb = 0; kb < num_kb; ++kb) {
    mbar_wait(&s.full[stage], phase);
    const uint64_t soff = uint64_t((stage * STAGE_BYTES) >> 4);
    reg_fence(acc);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BLOCK_K / 16; ++k)
      wgmma_m64n128_ss<TA, TB>(acc, da0 + soff + uint64_t((k * A_KSTEP) >> 4), db0 + soff + uint64_t((k * B_KSTEP) >> 4),
                               1u);
    wgmma_commit();
    wgmma_wait<1>();   // the previous stage's MMAs are complete: hand it back to the producer
    if (prev >= 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&s.empty[prev]);
    }
    prev = stage;
    if (++stage == STAGES) {
      stage = 0;
      phase ^= 1;
    }
  }
  wgmma_wait<0>();
  reg_fence(acc);
}

// Accumulators of warpgroup `wg` -> rows [64 wg, 64 wg + 64) of the staged fp32 tile; then all 256 consumer threads
// synchronise (named barrier 1) so that any of them may read any row.
__device__ __forceinline__ void stage_accumulators(const Smem& s, int wg, const float (&acc)[64]) {
  const int w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
  const int r0 = wg * 64 + w * 16 + (l >> 2);
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int c = 8 * j + 2 * (l & 3);
    *reinterpret_cast<float2*>(s.cbuf + r0 * CROW + c) = make_float2(acc[4 * j], acc[4 * j + 1]);
    *reinterpret_cast<float2*>(s.cbuf + (r0 + 8) * CROW + c) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
  }
  named_bar_sync(1, 256);
}

// 32 staged accumulator columns of one row as raw fp32 bit patterns
__device__ __forceinline__ void load_chunk(const float* crow, int c0, uint32_t (&a)[32]) {
#pragma unroll
  for (int i = 0; i < 32; i += 4) {
    const float4 v = *reinterpret_cast<const float4*>(crow + c0 + i);
    a[i] = __float_as_uint(v.x);
    a[i + 1] = __float_as_uint(v.y);
    a[i + 2] = __float_as_uint(v.z);
    a[i + 3] = __float_as_uint(v.w);
  }
}

}  // namespace sm90
}  // namespace b2f
