// Shared definitions of the attention kernels (attention.cu: forward kernel and host dispatch; attention_bwd.cu:
// backward kernels).
#pragma once
#include "host_common.h"
#include "ptx.cuh"

namespace b2f {
namespace attn {

constexpr int DH = 128;
constexpr int BQ = 128;   // query rows per CTA (64 per consumer warpgroup)
constexpr int BKV = 128;  // rows per K/V block
constexpr int KV_SLOTS = 2;
constexpr int TILE_BYTES = 128 * DH * 2;  // 32 KB: [128 rows][128 dh] as two [128][64] swizzled halves
constexpr int HALF_BYTES = TILE_BYTES / 2;
constexpr int ATTN_THREADS = 384;         // producer warpgroup + 2 consumer warpgroups
constexpr int ATTN_SMEM = (1 + 2 * KV_SLOTS) * TILE_BYTES + 256 + 1024;

struct AttnParams {
  int B, H, Hkv, Sq, Skv;
  float scale_log2;
  int causal;
  __nv_bfloat16* out;
  long long ldo;
  // additive score bias (BIAS kernels only): score = bias_scale * q.k + bias[h, q, kv]
  const __nv_bfloat16* bias;
  long long bias_h_stride, bias_row_stride;
  float bias_scale;
  // optional log-sum-exp output for the backward pass, base-2 domain: lse2[b, h, q] = max2 + log2(sum), where the scores
  // are scale_log2 * q.k; element (b, h, q) at lse + (b*H + h)*lse_stride + q
  float* lse;
  long long lse_stride;
};

static __device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// Row reductions over the four lanes of a quad (the threads sharing an accumulator row of a wgmma result).
static __device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
static __device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// One 16-column k-chunk of an m64nXk16 accumulator (fp32, layout of ptx.cuh) packed to bf16 as the register A operand
// of the next wgmma: chunk kk covers accumulator elements [8 kk, 8 kk + 8).
template <int R>
static __device__ __forceinline__ void pack_a_frag(const float (&s)[R], int kk, uint32_t (&a)[4]) {
  a[0] = pack_bf16x2(s[8 * kk + 0], s[8 * kk + 1]);
  a[1] = pack_bf16x2(s[8 * kk + 2], s[8 * kk + 3]);
  a[2] = pack_bf16x2(s[8 * kk + 4], s[8 * kk + 5]);
  a[3] = pack_bf16x2(s[8 * kk + 6], s[8 * kk + 7]);
}

}  // namespace attn
}  // namespace b2f
