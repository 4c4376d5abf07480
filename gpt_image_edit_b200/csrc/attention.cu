// Fused non-causal / causal softmax attention for sm_90a, head_dim 128, bf16 in/out.
//
//   O[b, q, h, :] = softmax(Q[b, q, h, :] · K[b, :, hk, :]^T * scale) · V[b, :, hk, :]
//
// One CTA owns a 128-row query tile of one (batch, head) and streams K/V in 128-row blocks:
//   warpgroup 0 (1 lane)   TMA producer: Q once, K_j and V_j through two double-buffered 32 KB slots
//   warpgroups 1, 2        64 query rows each:  S = Q·K_j^T (wgmma, both operands in smem, S in registers),
//                          online softmax in registers (base 2), P packed to bf16 in registers,
//                          O += P·V_j (wgmma with A = P from registers, B = V_j MN-major in smem)
// The two consumer warpgroups run independently, so one warpgroup's softmax overlaps the other's MMAs.
// Causal calls (Sq == Skv) stop streaming at the tile's last query row; GQA maps head h to K/V head h / (H / Hkv);
// the BIAS kernel adds a bf16 score bias (T5 relative positions) before the softmax.
// The WIN kernel (b2f_attention_fwd_window) gives every batch item a text window: keys [lo, hi) of the first S_txt
// and every key from S_txt on are valid, the rest are never loaded or, in a block that straddles them, get p = 0 and
// zeroed V rows.
//
// Replaces F.scaled_dot_product_attention as reached by diffusers FluxAttnProcessor2_0
// (SURVEY.md A.2; reference call site univa/utils/flux_pipeline.py:1067) and flash_attn as reached
// through transformers' attn_implementation="flash_attention_2" (univa/serve/cli.py:40).
#include <cmath>

#include "attention_common.cuh"

namespace b2f {

using namespace attn;

namespace {

constexpr int ATTN_SMEM = FwdSmem<TILE_BYTES>::BYTES;

// BIAS: additive bf16 score bias; the bias kernel folds the score scale into the bias step and runs with
// scale_log2 = log2(e).
// WIN: per-item text window p.win[b] = (lo, hi) over the first p.S_txt keys (non-causal, no bias).  The K/V blocks
// start at lo instead of 0: one run of blocks over [lo, end0) and, when the window stops short of the image rows
// (hi < S_txt), a second run over [S_txt, Skv).  With end0 = Skv for hi == S_txt (left-padded text, the full window)
// there is one run and no pad row is ever loaded; the full window (0, S_txt) streams exactly the blocks of the kernel
// without WIN.
template <bool BIAS, bool WIN>
__global__ void __launch_bounds__(ATTN_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  const FwdSmem<TILE_BYTES> sm(smem_raw);

  const int wg = __shfl_sync(0xffffffffu, int(threadIdx.x >> 7), 0);   // warp-uniform for the compiler
  const int h = blockIdx.y, b = blockIdx.z;
  const int hk = h / (p.H / p.Hkv);
  const int q0 = blockIdx.x * BQ;
  // K/V blocks this CTA needs (causal: only up to its last query row; Sq == Skv then)
  int kv_len = p.Skv;
  if (p.causal) kv_len = min(p.Skv, q0 + BQ);
  int n_kv = (kv_len + BKV - 1) / BKV;
  // WIN: block j < n0 covers keys [lo + j BKV, ..) of the run ending at end0, block j >= n0 [S_txt + (j - n0) BKV, ..)
  int lo = 0, hi = 0, end0 = 0, n0 = 0;
  if (WIN) {
    const int2 tw = text_window(p.win, b, p.S_txt);
    lo = tw.x;
    hi = tw.y;
    end0 = hi == p.S_txt ? p.Skv : hi;
    n0 = (end0 - lo + BKV - 1) / BKV;
    n_kv = n0 + (hi == p.S_txt ? 0 : (p.Skv - p.S_txt + BKV - 1) / BKV);
  }
  auto kv_start = [&](int j) { return !WIN ? j * BKV : j < n0 ? lo + j * BKV : p.S_txt + (j - n0) * BKV; };

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    sm.init_barriers();
  }
  __syncthreads();

  if (wg == 0) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      // ---------------------------------------------------------------- TMA producer
      mbar_expect_tx(sm.q_full, TILE_BYTES);
      for (int half = 0; half < 2; ++half)
        tma_load_3d(sm.q + half * HALF_BYTES, &tmQ, sm.q_full, h * DH + half * 64, q0, b);
      // K / V block j: two 64-column halves of the 128 rows from kv_start(j)
      sm.produce_kv(
          n_kv,
          [&](int j, uint8_t* dst, uint64_t* bar) {
            for (int half = 0; half < 2; ++half)
              tma_load_3d(dst + half * HALF_BYTES, &tmK, bar, hk * DH + half * 64, kv_start(j), b);
          },
          [&](int j, uint8_t* dst, uint64_t* bar) {
            for (int half = 0; half < 2; ++half)
              tma_load_3d(dst + half * HALF_BYTES, &tmV, bar, hk * DH + half * 64, kv_start(j), b);
          });
    }
    return;
  }

  // ------------------------------------------------------------------ consumer warpgroups
  setmaxnreg_inc<CONSUMER_REGS>();
  const auto [c, w, lane, row0, colq] = consumer_pos(wg, q0);
  const uint64_t dq0 = make_sdesc_sw128(smem_u32(sm.q) + c * 8192, 16, 1024);
  const uint64_t dk0 = make_sdesc_sw128(smem_u32(sm.k), 16, 1024);
  const uint64_t dv0 = make_sdesc_sw128(smem_u32(sm.v), HALF_BYTES, 1024);
  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};   // l: this thread's partial row sums
  mbar_wait(sm.q_full, 0);
  for (int j = 0; j < n_kv; ++j) {
    const int slot = j % KV_SLOTS;
    const uint32_t phase = (j / KV_SLOTS) & 1;
    float s[64];
    mbar_wait(&sm.k_full[slot], phase);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < DH / 16; ++k) {
      const uint64_t off = uint64_t(((k >> 2) * HALF_BYTES + (k & 3) * 32) >> 4);
      wgmma_m64n128_ss<0, 0>(s, dq0 + off, dk0 + uint64_t((slot * TILE_BYTES) >> 4) + off, k != 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);
    consumer_release(&sm.k_empty[slot], lane);

    const int kv0 = kv_start(j);
    if (BIAS) {
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        const int row = row0 + acc_row(i);
        const int col = kv0 + acc_col(i, colq);
        if (row < p.Sq && col < p.Skv)
          s[i] = fmaf(s[i], p.bias_scale,
                      __bfloat162float(p.bias[(long long)h * p.bias_h_stride + (long long)row * p.bias_row_stride + col]));
      }
    }
    if (WIN) {
      const int kv_end = j < n0 ? end0 : p.Skv;   // keys [kv_end, kv0 + BKV) of this block are masked
      if (kv0 + BKV > kv_end) {
#pragma unroll
        for (int i = 0; i < 64; ++i)
          if (kv0 + acc_col(i, colq) >= kv_end) s[i] = -INFINITY;
      }
    } else if (kv0 + BKV > p.Skv || p.causal) {
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        const int limit = p.causal ? min(p.Skv, row0 + acc_row(i) + 1) : p.Skv;
        if (kv0 + acc_col(i, colq) >= limit) s[i] = -INFINITY;
      }
    }
    float alpha[2];
    softmax_step<0>(s, m, l, p.scale_log2, alpha);
#pragma unroll
    for (int i = 0; i < 64; ++i) o[i] *= alpha[acc_row(i) / 8];

    uint32_t pa[BKV / 16][4];
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) pack_a_frag(s, kk, pa[kk]);
    if (WIN && j == n0 - 1 && hi < p.S_txt && hi - kv0 < BKV) {
      // The last block of the text run holds pad rows [hi, S_txt) (any content, NaN included): p = 0 there, but
      // 0 * NaN is NaN in P.V, so both consumer warpgroups zero those V rows (all 128 channels, whole 128-byte rows
      // of both swizzled halves) before either multiplies.  Rows from S_txt on are image rows (finite) and rows past
      // Skv arrive as TMA zero fill.
      const int z0 = hi - kv0, z1 = min(p.S_txt - kv0, BKV);
      mbar_wait(&sm.v_full[slot], phase);
      uint8_t* vt = sm.v + slot * TILE_BYTES;
      for (int i = z0 * 16 + (int(threadIdx.x) - 128); i < z1 * 16; i += 256)
        *reinterpret_cast<uint4*>(vt + (i & 8) / 8 * HALF_BYTES + (i >> 4) * 128 + (i & 7) * 16) = make_uint4(0, 0, 0, 0);
      fence_proxy_async_smem();
      named_bar_sync(1, 256);
    }
    mbar_wait(&sm.v_full[slot], phase);
    reg_fence(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk)
      wgmma_m64n128_rs<1>(o, pa[kk], dv0 + uint64_t((slot * TILE_BYTES + kk * 2048) >> 4), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(o);
    consumer_release(&sm.v_empty[slot], lane);
  }

  // ---------------------------------------------------------------- epilogue: O / l -> bf16
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = row0 + 8 * r;
    const float lt = quad_sum(l[r]);
    const float inv_l = 1.0f / lt;
    if (row >= p.Sq) continue;
    if (p.lse && (lane & 3) == 0) p.lse[((long long)b * p.H + h) * p.lse_stride + row] = m[r] + log2f(lt);
    store_row_bf16(p.out + ((long long)b * p.Sq + row) * p.ldo + (long long)h * DH, o, r, colq, inv_l);
  }
}

}  // namespace

static int attention_impl(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v,
                          int64_t ldv, void* out, int64_t ldo, int B, int H, int Hkv, int Sq, int Skv,
                          int head_dim, float scale, int causal, const void* bias, int64_t bias_h_stride,
                          int64_t bias_row_stride, float* lse, int64_t lse_stride, const int32_t* win, int S_txt,
                          cudaStream_t stream) {
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (lse && lse_stride < Sq) return B2F_ERR_INVALID;
  if (!q || !k || !v || !out || B <= 0 || H <= 0 || Hkv <= 0 || Sq <= 0 || Skv <= 0)
    return B2F_ERR_INVALID;
  if (head_dim != DH) return B2F_ERR_UNSUPPORTED;
  if (H % Hkv) return B2F_ERR_INVALID;
  if (causal && Sq != Skv) return B2F_ERR_UNSUPPORTED;
  if ((ldq & 7) || (ldk & 7) || (ldv & 7) || (ldo & 7)) return B2F_ERR_ALIGN;
  if ((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) |
       reinterpret_cast<uintptr_t>(v) | reinterpret_cast<uintptr_t>(out)) & 15)
    return B2F_ERR_ALIGN;
  static bool attr_set = false;
  if (int rc = set_max_smem_once(attr_set, ATTN_SMEM, "attention smem attribute", attn_fwd_kernel<false, false>,
                                 attn_fwd_kernel<true, false>, attn_fwd_kernel<false, true>))
    return rc;
  CUtensorMap tmQ, tmK, tmV;
  int rc = make_tmap_3d_rows(&tmQ, q, (uint64_t)H * DH, Sq, B, ldq, (uint64_t)Sq * ldq);
  if (rc) return rc;
  rc = make_tmap_3d_rows(&tmK, k, (uint64_t)Hkv * DH, Skv, B, ldk, (uint64_t)Skv * ldk);
  if (rc) return rc;
  rc = make_tmap_3d_rows(&tmV, v, (uint64_t)Hkv * DH, Skv, B, ldv, (uint64_t)Skv * ldv);
  if (rc) return rc;
  AttnParams p{};
  p.B = B;
  p.H = H;
  p.Hkv = Hkv;
  p.Sq = Sq;
  p.Skv = Skv;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.causal = causal;
  p.out = static_cast<__nv_bfloat16*>(out);
  p.ldo = ldo;
  p.lse = lse;
  p.lse_stride = lse_stride;
  if (bias) {
    // score = scale * q.k + bias, evaluated before the base-2 conversion
    p.bias = static_cast<const __nv_bfloat16*>(bias);
    p.bias_h_stride = bias_h_stride;
    p.bias_row_stride = bias_row_stride;
    p.bias_scale = scale;
    p.scale_log2 = 1.4426950408889634f;
    dim3 grid_b((Sq + BQ - 1) / BQ, H, B);
    prof_begin(KC_ATTN, stream);
    attn_fwd_kernel<true, false><<<grid_b, ATTN_THREADS, ATTN_SMEM, stream>>>(tmQ, tmK, tmV, p);
    prof_end(KC_ATTN, stream, (causal ? 2.0 : 4.0) * B * H * (double)Sq * Skv * DH,
             2.0 * DH * B * (2.0 * H * Sq + 2.0 * Hkv * Skv) + 2.0 * H * (double)Sq * Skv);
    B2F_LAUNCHED("attn_fwd_kernel<bias>", 1);
    return B2F_OK;
  }
  dim3 grid((Sq + BQ - 1) / BQ, H, B);
  if (win) {
    p.win = win;
    p.S_txt = S_txt;
    prof_begin(KC_ATTN, stream);
    attn_fwd_kernel<false, true><<<grid, ATTN_THREADS, ATTN_SMEM, stream>>>(tmQ, tmK, tmV, p);
    // the full-window bound: blocks outside the windows are skipped
    prof_end(KC_ATTN, stream, 4.0 * B * H * (double)Sq * Skv * DH, 2.0 * DH * B * (2.0 * H * Sq + 2.0 * Hkv * Skv));
    B2F_LAUNCHED("attn_fwd_kernel<window>", 1);
    return B2F_OK;
  }
  prof_begin(KC_ATTN, stream);
  attn_fwd_kernel<false, false><<<grid, ATTN_THREADS, ATTN_SMEM, stream>>>(tmQ, tmK, tmV, p);
  prof_end(KC_ATTN, stream, (causal ? 2.0 : 4.0) * B * H * (double)Sq * Skv * DH,
           2.0 * DH * B * (2.0 * H * Sq + 2.0 * Hkv * Skv));
  B2F_LAUNCHED("attn_fwd_kernel", 1);
  return B2F_OK;
}

extern "C" int b2f_attention_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv,
                                 void* out, int64_t ldo, int B, int H, int Hkv, int Sq, int Skv, int head_dim,
                                 float scale, int causal, b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  return attention_impl(q, ldq, k, ldk, v, ldv, out, ldo, B, H, Hkv, Sq, Skv, head_dim, scale, causal,
                        nullptr, 0, 0, nullptr, 0, nullptr, 0, stream);
}

extern "C" int b2f_attention_fwd_window(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v,
                                        int64_t ldv, void* out, int64_t ldo, int B, int H, int Hkv, int Sq, int Skv,
                                        int head_dim, float scale, const int32_t* win, int S_txt,
                                        b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!win || S_txt < 0 || S_txt > Skv) return B2F_ERR_INVALID;
  return attention_impl(q, ldq, k, ldk, v, ldv, out, ldo, B, H, Hkv, Sq, Skv, head_dim, scale, 0, nullptr, 0, 0,
                        nullptr, 0, win, S_txt, stream);
}

// forward that also emits the base-2 log-sum-exp rows the backward kernels need (attention_bwd.cu)
extern "C" int b2f_attention_fwd_lse(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv,
                                     void* out, int64_t ldo, int B, int H, int Hkv, int Sq, int Skv, int head_dim,
                                     float scale, int causal, float* lse, int64_t lse_stride, b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!lse) return B2F_ERR_INVALID;
  return attention_impl(q, ldq, k, ldk, v, ldv, out, ldo, B, H, Hkv, Sq, Skv, head_dim, scale, causal, nullptr, 0, 0,
                        lse, lse_stride, nullptr, 0, stream);
}

extern "C" int b2f_attention_bias_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v,
                                      int64_t ldv, void* out, int64_t ldo, int B, int H, int Hkv, int Sq, int Skv,
                                      int head_dim, float scale, int causal, const void* bias, int64_t bias_h_stride,
                                      int64_t bias_row_stride, b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!bias || bias_row_stride < Skv || bias_h_stride < 0) return B2F_ERR_INVALID;
  return attention_impl(q, ldq, k, ldk, v, ldv, out, ldo, B, H, Hkv, Sq, Skv, head_dim, scale, causal,
                        bias, bias_h_stride, bias_row_stride, nullptr, 0, nullptr, 0, stream);
}

}  // namespace b2f
