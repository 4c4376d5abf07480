// Shared definitions of the attention kernels (attention.cu: bf16 forward kernel and host dispatch; attention_fp8.cu:
// FP8 quantizer and forward kernel; attention_bwd.cu: backward kernels).
#pragma once
#include "host_common.h"
#include "ptx.cuh"

namespace b2f {
namespace attn {

constexpr int DH = 128;
constexpr int BQ = 128;   // query rows per CTA (64 per consumer warpgroup)
constexpr int BKV = 128;  // rows per K/V block
constexpr int KV_SLOTS = 2;  // four (the FP8 kernel's shared memory has room) measured no faster on an H100
constexpr int TILE_BYTES = 128 * DH * 2;  // 32 KB: [128 rows][128 dh] as two [128][64] swizzled halves
constexpr int HALF_BYTES = TILE_BYTES / 2;
constexpr int ATTN_THREADS = 384;         // producer warpgroup + 2 consumer warpgroups
constexpr int PRODUCER_REGS = 24;         // setmaxnreg budgets: the producer gives registers back, the consumers take them
constexpr int CONSUMER_REGS = 240;

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
  // per-item text window (WIN kernel only): int32 [B, 2] (lo, hi) on the device; keys k < S_txt valid iff lo <= k < hi
  const int32_t* win;
  int S_txt;
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

// Accumulator layout of an m64nN wgmma result (ptx.cuh): a consumer thread owns rows row0 and row0 + 8 of its
// warpgroup's 64 and, in every 8-column group, columns colq and colq + 1; its element i lies at row row0 + acc_row(i)
// and column acc_col(i, colq), so elements 4g .. 4g + 3 are (row0, 8g + colq), (row0, + 1), (row0 + 8, ..), (.., + 1).
static __device__ __forceinline__ int acc_row(int i) { return 8 * ((i >> 1) & 1); }
static __device__ __forceinline__ int acc_col(int i, int colq) { return 8 * (i >> 2) + colq + (i & 1); }

// A consumer thread's coordinates: consumer warpgroup c (0, 1), its warp w and lane, its first row and first column
// (above) in a CTA whose stationary rows start at row0_cta.
struct ConsumerPos {
  int c, w, lane, row0, colq;
};
static __device__ __forceinline__ ConsumerPos consumer_pos(int wg, int row0_cta) {
  const int c = wg - 1, w = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  return {c, w, lane, row0_cta + c * 64 + w * 16 + (lane >> 2), 2 * (lane & 3)};
}

// A consumer warp is done with a slot: once all its lanes are, lane 0 arrives on the slot's empty barrier (whose count
// is one arrive per consumer warp).
static __device__ __forceinline__ void consumer_release(uint64_t* empty, int lane) {
  __syncwarp();
  if (lane == 0) mbar_arrive(empty);
}

// Shared memory of the forward kernels for K / V tiles of TILE bytes (and a Q tile of the same size): Q, KV_SLOTS K
// tiles, KV_SLOTS V tiles, then the barriers q_full and, per slot, k_full, k_empty, v_full, v_empty.
template <int TILE>
struct FwdSmem {
  static constexpr int BYTES = (1 + 2 * KV_SLOTS) * TILE + 256 + 1024;   // barriers, and the base's 1024-byte alignment
  uint8_t *q, *k, *v;
  uint64_t *q_full, *k_full, *k_empty, *v_full, *v_empty;

  __device__ __forceinline__ explicit FwdSmem(uint8_t* raw) {
    q = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 1023) & ~uintptr_t(1023));
    k = q + TILE;
    v = k + KV_SLOTS * TILE;
    q_full = reinterpret_cast<uint64_t*>(v + KV_SLOTS * TILE);
    k_full = q_full + 1;
    k_empty = k_full + KV_SLOTS;
    v_full = k_empty + KV_SLOTS;
    v_empty = v_full + KV_SLOTS;
  }

  // by one thread, before the CTA's first barrier
  __device__ __forceinline__ void init_barriers() const {
    mbar_init(q_full, 1);
    for (int i = 0; i < KV_SLOTS; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&v_full[i], 1);
      mbar_init(&k_empty[i], 8);   // one arrive per consumer warp
      mbar_init(&v_empty[i], 8);
    }
    fence_mbar_init();
  }

  // The TMA producer's K / V ring: block j goes through slot j % KV_SLOTS once the consumers have released the slot's
  // previous block; load_k(j, dst, bar) and load_v(j, dst, bar) issue the TILE bytes of K / V block j.
  template <class LoadK, class LoadV>
  __device__ __forceinline__ void produce_kv(int n_kv, LoadK load_k, LoadV load_v) const {
    for (int j = 0; j < n_kv; ++j) {
      const int slot = j % KV_SLOTS;
      const uint32_t phase = (j / KV_SLOTS) & 1;
      mbar_wait(&k_empty[slot], phase ^ 1);
      mbar_expect_tx(&k_full[slot], TILE);
      load_k(j, k + slot * TILE, &k_full[slot]);
      mbar_wait(&v_empty[slot], phase ^ 1);
      mbar_expect_tx(&v_full[slot], TILE);
      load_v(j, v + slot * TILE, &v_full[slot]);
    }
  }
};

// One online-softmax step over a block's scores s (this thread's 64 accumulator elements, two rows) with the running
// base-2 row maxima m and partial row sums l: s becomes p = ex2(s * scale - m_new + OFFSET), l = alpha * l + rowsum(p),
// and alpha = ex2(m_old - m_new) is returned for the caller's rescale of O.  A row masked so far (m_new = -inf) gets
// p = 0 and alpha = 0.
template <int OFFSET>
static __device__ __forceinline__ void softmax_step(float (&s)[64], float (&m)[2], float (&l)[2], float scale,
                                                    float (&alpha)[2]) {
  float neg_m[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < 64; ++i)
      if (acc_row(i) == 8 * r) mx = fmaxf(mx, s[i]);
    mx = quad_max(mx);
    const float m_new = fmaxf(m[r], mx * scale);
    alpha[r] = m[r] == -INFINITY ? 0.f : ex2(m[r] - m_new);
    // OFFSET 0 keeps -m_new, not 0 - m_new: the two differ in the sign of a zero result, and the subtraction costs one
    // instruction more
    neg_m[r] = m_new == -INFINITY ? 0.f : OFFSET == 0 ? -m_new : float(OFFSET) - m_new;
    m[r] = m_new;
  }
  float sum[2] = {0.f, 0.f};
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const int r = acc_row(i) / 8;
    s[i] = ex2(fmaf(s[i], scale, neg_m[r]));
    sum[r] += s[i];
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) l[r] = l[r] * alpha[r] + sum[r];
}

// Row r (0, 1) of this thread's m64n128 accumulator acc, times mul, as bf16 at out_row + 8 jj + colq (jj < 16).
static __device__ __forceinline__ void store_row_bf16(__nv_bfloat16* out_row, const float (&acc)[64], int r, int colq,
                                                      float mul) {
#pragma unroll
  for (int jj = 0; jj < 16; ++jj) {
    const int i = 4 * jj + 2 * r;
    *reinterpret_cast<uint32_t*>(out_row + 8 * jj + colq) = pack_bf16x2(acc[i] * mul, acc[i + 1] * mul);
  }
}

// The text window (lo, hi) of item b, clamped to [0, S_txt] so that out-of-range values never index out of bounds.
static __device__ __forceinline__ int2 text_window(const int32_t* win, int b, int S_txt) {
  const int lo = min(max(win[2 * b], 0), S_txt);
  return make_int2(lo, min(max(win[2 * b + 1], lo), S_txt));
}
// A text token outside its item's window tw.
static __device__ __forceinline__ bool in_text_gap(int tok, int2 tw, int S_txt) {
  return tok < S_txt && (tok < tw.x || tok >= tw.y);
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
