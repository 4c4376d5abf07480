// Backward of the fused softmax attention (head_dim 128, non-causal, H == Hkv: the FLUX joint attention) for sm_90a.
//
// Given Q, K, V, dO, the forward's base-2 log-sum-exp rows lse2[b,h,q] and delta[b,h,q] = rowsum(dO * O):
//   P  = exp2(scale_log2 * Q K^T - lse2)          (the normalised probabilities, recomputed, never stored)
//   dP = dO V^T;   dS = P * (dP - delta)
//   dV = P^T dO;   dK = scale * dS^T Q;   dQ = scale * dS K
// Two launches of one kernel template, both free of atomics (deterministic):
//   MODE 0 (dK, dV): a CTA owns 128 K/V rows of one (batch, head) and streams Q / dO blocks; everything is held
//                    TRANSPOSED (rows = kv, columns = q) so that P^T and dS^T are the register A operands of the two
//                    accumulating MMAs;
//   MODE 1 (dQ):     a CTA owns 128 query rows and streams K / V blocks.
// X = the stationary tiles, Y = the streamed 64-row blocks; MODE 0: X = (K, V), Y = (Q, dO);  MODE 1: X = (Q, dO),
// Y = (K, V).  Per block and consumer warpgroup (64 stationary rows):
//                        S~  = X0 . Y0^T   (wgmma, smem x smem, 64 x 64 in registers)
//                        dP~ = X1 . Y1^T
//                        P~, dS~ -> bf16 register fragments
//                        G1 += P~ . Y1     (MODE 0 only: dV)     Y blocks re-read as MN-major B operands
//                        G0 += dS~ . Y0    (dK or dQ)
//   warpgroup 0 (1 lane)   TMA producer: X tiles once, (Y0, Y1, lse2, delta) through a 2-stage ring
//   warpgroups 1, 2        consumers, 64 stationary rows each; G0 / G1 accumulate in registers
//
// Replaces the autograd of F.scaled_dot_product_attention / flash_attn backward reached by
// accelerator.backward(loss) in the reference (train_denoiser.py:1172) for every FLUX block.
#include <cmath>

#include "attention_common.cuh"

namespace b2f {

using namespace attn;

namespace {

constexpr int BWD_THREADS = 384;
constexpr int BWD_STAGES = 2;
constexpr int BS = 64;                          // streamed rows per block
constexpr int Y_BYTES = BS * DH * 2;            // 16 KB: two [64][64] swizzled halves
constexpr int Y_HALF = Y_BYTES / 2;
constexpr int BWD_VEC_FLOATS = 2 * BS;          // lse2[64], delta[64] of one stage
constexpr int BWD_SMEM = 2 * TILE_BYTES + BWD_STAGES * 2 * Y_BYTES + BWD_STAGES * BWD_VEC_FLOATS * 4 + 256 + 1024;

struct AttnBwdParams {
  int B, H, S, S_pad;
  float scale, scale_log2;
  const float* lse;     // [B, H, S_pad], base-2
  const float* delta;   // [B, H, S_pad]
  __nv_bfloat16* g0;    // MODE 0: dK, MODE 1: dQ     token-major [B, S, ld]
  __nv_bfloat16* g1;    // MODE 0: dV
  long long ld0, ld1;
};

template <int MODE>
__global__ void __launch_bounds__(BWD_THREADS, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tmX0, const __grid_constant__ CUtensorMap tmX1,
                const __grid_constant__ CUtensorMap tmY0, const __grid_constant__ CUtensorMap tmY1,
                const AttnBwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* x_smem = smem;                                  // X0, X1
  uint8_t* y_smem = smem + 2 * TILE_BYTES;                 // per stage: Y0, Y1
  float* vec_smem = reinterpret_cast<float*>(y_smem + BWD_STAGES * 2 * Y_BYTES);   // per stage: lse2[64], delta[64]
  uint64_t* bars = reinterpret_cast<uint64_t*>(vec_smem + BWD_STAGES * BWD_VEC_FLOATS);
  uint64_t* x_full = bars;                   // 1
  uint64_t* y_full = bars + 1;               // BWD_STAGES
  uint64_t* y_empty = y_full + BWD_STAGES;   // BWD_STAGES

  const int wg = __shfl_sync(0xffffffffu, int(threadIdx.x >> 7), 0);   // warp-uniform for the compiler
  const int h = blockIdx.y, b = blockIdx.z;
  const int row0_cta = blockIdx.x * 128;         // first stationary row (kv in MODE 0, q in MODE 1)
  const int n_it = (p.S + BS - 1) / BS;          // streamed blocks

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmX0);
    tma_prefetch_desc(&tmX1);
    tma_prefetch_desc(&tmY0);
    tma_prefetch_desc(&tmY1);
    mbar_init(x_full, 1);
    for (int i = 0; i < BWD_STAGES; ++i) {
      mbar_init(&y_full[i], 1);
      mbar_init(&y_empty[i], 8);   // one arrive per consumer warp: its MMAs and its reads of lse2 / delta are done
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      // ---------------------------------------------------------------- TMA producer
      mbar_expect_tx(x_full, 2 * TILE_BYTES);
      for (int half = 0; half < 2; ++half) {
        tma_load_3d(x_smem + half * HALF_BYTES, &tmX0, x_full, h * DH + half * 64, row0_cta, b);
        tma_load_3d(x_smem + TILE_BYTES + half * HALF_BYTES, &tmX1, x_full, h * DH + half * 64, row0_cta, b);
      }
      const float* lse_row = p.lse + ((long long)b * p.H + h) * p.S_pad;
      const float* dl_row = p.delta + ((long long)b * p.H + h) * p.S_pad;
      for (int i = 0; i < n_it; ++i) {
        const int stage = i % BWD_STAGES;
        mbar_wait(&y_empty[stage], ((i / BWD_STAGES) & 1) ^ 1);
        uint8_t* y0 = y_smem + stage * 2 * Y_BYTES;
        uint8_t* y1 = y0 + Y_BYTES;
        mbar_expect_tx(&y_full[stage], 2 * Y_BYTES + (MODE == 0 ? BWD_VEC_FLOATS * 4 : 0));
        for (int half = 0; half < 2; ++half) {
          tma_load_3d(y0 + half * Y_HALF, &tmY0, &y_full[stage], h * DH + half * 64, i * BS, b);
          tma_load_3d(y1 + half * Y_HALF, &tmY1, &y_full[stage], h * DH + half * 64, i * BS, b);
        }
        if (MODE == 0) {
          // the streamed index is the query index: its lse2 / delta rows ride along with the blocks
          bulk_load_1d(vec_smem + stage * BWD_VEC_FLOATS, lse_row + i * BS, BS * 4, &y_full[stage]);
          bulk_load_1d(vec_smem + stage * BWD_VEC_FLOATS + BS, dl_row + i * BS, BS * 4, &y_full[stage]);
        }
      }
    }
    return;
  }

  // ------------------------------------------------------------------ consumer warpgroups
  setmaxnreg_inc<CONSUMER_REGS>();
  const auto [c, w, lane, row0, colq] = consumer_pos(wg, row0_cta);   // stationary rows row0, row0 + 8
  const uint64_t dx0 = make_sdesc_sw128(smem_u32(x_smem) + c * 8192, 16, 1024);
  const uint64_t dx1 = dx0 + uint64_t(TILE_BYTES >> 4);
  const uint64_t dyk = make_sdesc_sw128(smem_u32(y_smem), 16, 1024);        // K-major view of a Y block
  const uint64_t dym = make_sdesc_sw128(smem_u32(y_smem), Y_HALF, 1024);    // MN-major view
  float my_lse[2] = {0.f, 0.f}, my_delta[2] = {0.f, 0.f};
  if (MODE == 1) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      // rows beyond S read the padding (lse = +inf, delta = 0): P = 0 there
      my_lse[r] = p.lse[((long long)b * p.H + h) * p.S_pad + row0 + 8 * r];
      my_delta[r] = p.delta[((long long)b * p.H + h) * p.S_pad + row0 + 8 * r];
    }
  }
  float g0[64], g1[64];   // g1 (dV) is used in MODE 0 only; the compiler drops it from MODE 1
#pragma unroll
  for (int i = 0; i < 64; ++i) g0[i] = g1[i] = 0.f;
  mbar_wait(x_full, 0);
  for (int it = 0; it < n_it; ++it) {
    const int stage = it % BWD_STAGES;
    mbar_wait(&y_full[stage], (it / BWD_STAGES) & 1);
    const uint64_t y0_off = uint64_t((stage * 2 * Y_BYTES) >> 4), y1_off = uint64_t((stage * 2 * Y_BYTES + Y_BYTES) >> 4);
    float st[32], dpt[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < DH / 16; ++k) {
      const uint32_t xo = (k >> 2) * HALF_BYTES + (k & 3) * 32, yo = (k >> 2) * Y_HALF + (k & 3) * 32;
      wgmma_m64n64_ss<0, 0>(st, dx0 + uint64_t(xo >> 4), dyk + y0_off + uint64_t(yo >> 4), k != 0 ? 1u : 0u);
    }
#pragma unroll
    for (int k = 0; k < DH / 16; ++k) {
      const uint32_t xo = (k >> 2) * HALF_BYTES + (k & 3) * 32, yo = (k >> 2) * Y_HALF + (k & 3) * 32;
      wgmma_m64n64_ss<0, 0>(dpt, dx1 + uint64_t(xo >> 4), dyk + y1_off + uint64_t(yo >> 4), k != 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(st);
    reg_fence(dpt);
    const float* lse_s = vec_smem + stage * BWD_VEC_FLOATS;
    const float* dl_s = lse_s + BS;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int r = acc_row(i) / 8;
      const int lc = acc_col(i, colq);   // streamed index inside the block
      float l, d;
      if (MODE == 0) {
        l = lse_s[lc];
        d = dl_s[lc];
      } else {
        l = my_lse[r];
        d = my_delta[r];
      }
      float pv = ex2(fmaf(st[i], p.scale_log2, -l));
      if (MODE == 0) {
        if (row0 + 8 * r >= p.S) pv = 0.f;            // K/V rows beyond the sequence (zero-filled tiles)
      } else {
        if (it * BS + lc >= p.S) pv = 0.f;            // K/V columns beyond the sequence
      }
      st[i] = pv;
      dpt[i] = pv * (dpt[i] - d);
    }
    uint32_t pf[BS / 16][4], df[BS / 16][4];
#pragma unroll
    for (int kk = 0; kk < BS / 16; ++kk) {
      pack_a_frag(st, kk, pf[kk]);
      pack_a_frag(dpt, kk, df[kk]);
    }
    reg_fence(g0);
    if (MODE == 0) reg_fence(g1);
    wgmma_fence();
    if (MODE == 0) {
      // dV += P~ . dO      (B = Y1 as [K = q rows, N = dh], MN-major)
#pragma unroll
      for (int kk = 0; kk < BS / 16; ++kk)
        wgmma_m64n128_rs<1>(g1, pf[kk], dym + y1_off + uint64_t((kk * 2048) >> 4), 1u);
    }
    // dK / dQ += dS~ . Y0
#pragma unroll
    for (int kk = 0; kk < BS / 16; ++kk)
      wgmma_m64n128_rs<1>(g0, df[kk], dym + y0_off + uint64_t((kk * 2048) >> 4), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(g0);
    if (MODE == 0) reg_fence(g1);
    consumer_release(&y_empty[stage], lane);
  }

  // ---------------------------------------------------------------- epilogue: accumulators -> bf16 -> global
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = row0 + 8 * r;
    if (row >= p.S) continue;
    store_row_bf16(p.g0 + ((long long)b * p.S + row) * p.ld0 + (long long)h * DH, g0, r, colq, p.scale);
    if (MODE == 0) store_row_bf16(p.g1 + ((long long)b * p.S + row) * p.ld1 + (long long)h * DH, g1, r, colq, 1.0f);
  }
}

}  // namespace

// q/k/v/dout: token-major [B, S, H*128] views (pitches ld*); lse, delta: fp32 [B, H, S_pad] with S_pad a multiple of
// 128, lse = +inf and delta = 0 in the padding (attn_delta writes both); dq/dk/dv: [B, S, H*128] views.
extern "C" int b2f_attention_bwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv,
                                 const void* dout, int64_t lddo, const float* lse, const float* delta, int64_t S_pad,
                                 void* dq, int64_t lddq, void* dk, int64_t lddk, void* dv, int64_t lddv, int B, int H,
                                 int S, int head_dim, float scale, b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (!q || !k || !v || !dout || !lse || !delta || !dq || !dk || !dv || B <= 0 || H <= 0 || S <= 0) return B2F_ERR_INVALID;
  if (head_dim != DH) return B2F_ERR_UNSUPPORTED;
  if (S_pad < S || (S_pad & 127)) return B2F_ERR_INVALID;
  if ((ldq | ldk | ldv | lddo | lddq | lddk | lddv) & 7) return B2F_ERR_ALIGN;
  if ((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v) |
       reinterpret_cast<uintptr_t>(dout) | reinterpret_cast<uintptr_t>(dq) | reinterpret_cast<uintptr_t>(dk) |
       reinterpret_cast<uintptr_t>(dv) | reinterpret_cast<uintptr_t>(lse) | reinterpret_cast<uintptr_t>(delta)) & 15)
    return B2F_ERR_ALIGN;
  static bool attr_set = false;
  if (int rc = set_max_smem_once(attr_set, BWD_SMEM, "attention bwd smem attribute", attn_bwd_kernel<0>,
                                 attn_bwd_kernel<1>))
    return rc;
  // every operand as a stationary tile (128-row boxes) and as a streamed block (64-row boxes)
  CUtensorMap tQ, tK, tV, tO, sQ, sK, sV, sO;
  const void* src[4] = {q, k, v, dout};
  const int64_t lds[4] = {ldq, ldk, ldv, lddo};
  CUtensorMap* tiles[4] = {&tQ, &tK, &tV, &tO};
  CUtensorMap* blocks[4] = {&sQ, &sK, &sV, &sO};
  for (int i = 0; i < 4; ++i) {
    int rc = make_tmap_3d_rows(tiles[i], src[i], (uint64_t)H * DH, S, B, lds[i], (uint64_t)S * lds[i]);
    if (rc) return rc;
    rc = make_tmap_3d_rows(blocks[i], src[i], (uint64_t)H * DH, S, B, lds[i], (uint64_t)S * lds[i], BS);
    if (rc) return rc;
  }
  AttnBwdParams p{};
  p.B = B;
  p.H = H;
  p.S = S;
  p.S_pad = (int)S_pad;
  p.scale = scale;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.lse = lse;
  p.delta = delta;
  dim3 grid((S + 127) / 128, H, B);
  const double unit = 2.0 * B * H * (double)S * S * DH;
  p.g0 = static_cast<__nv_bfloat16*>(dk);
  p.ld0 = lddk;
  p.g1 = static_cast<__nv_bfloat16*>(dv);
  p.ld1 = lddv;
  prof_begin(KC_ATTN, stream);
  attn_bwd_kernel<0><<<grid, BWD_THREADS, BWD_SMEM, stream>>>(tK, tV, sQ, sO, p);
  prof_end(KC_ATTN, stream, 4.0 * unit, 2.0 * DH * B * H * 6.0 * S);
  B2F_LAUNCHED("attn_bwd_kernel<dKdV>", 1);
  p.g0 = static_cast<__nv_bfloat16*>(dq);
  p.ld0 = lddq;
  p.g1 = nullptr;
  prof_begin(KC_ATTN, stream);
  attn_bwd_kernel<1><<<grid, BWD_THREADS, BWD_SMEM, stream>>>(tQ, tO, sK, sV, p);
  prof_end(KC_ATTN, stream, 3.0 * unit, 2.0 * DH * B * H * 5.0 * S);
  B2F_LAUNCHED("attn_bwd_kernel<dQ>", 1);
  return B2F_OK;
}

}  // namespace b2f
