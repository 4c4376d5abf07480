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
//
// Replaces F.scaled_dot_product_attention as reached by diffusers FluxAttnProcessor2_0
// (SURVEY.md A.2; reference call site univa/utils/flux_pipeline.py:1067) and flash_attn as reached
// through transformers' attn_implementation="flash_attention_2" (univa/serve/cli.py:40).
#include <cmath>

#include "attention_common.cuh"

namespace b2f {

using namespace attn;

namespace {

// BIAS: additive bf16 score bias; the bias kernel folds the score scale into the bias step and runs with
// scale_log2 = log2(e).
template <bool BIAS>
__global__ void __launch_bounds__(ATTN_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~uintptr_t(1023));
  uint8_t* q_smem = smem;
  uint8_t* k_smem = smem + TILE_BYTES;                      // KV_SLOTS tiles
  uint8_t* v_smem = k_smem + KV_SLOTS * TILE_BYTES;         // KV_SLOTS tiles
  uint64_t* bars = reinterpret_cast<uint64_t*>(v_smem + KV_SLOTS * TILE_BYTES);
  uint64_t* q_full = bars;                 // 1
  uint64_t* k_full = bars + 1;             // KV_SLOTS
  uint64_t* k_empty = k_full + KV_SLOTS;
  uint64_t* v_full = k_empty + KV_SLOTS;
  uint64_t* v_empty = v_full + KV_SLOTS;

  const int wg = __shfl_sync(0xffffffffu, int(threadIdx.x >> 7), 0);   // warp-uniform for the compiler
  const int h = blockIdx.y, b = blockIdx.z;
  const int hk = h / (p.H / p.Hkv);
  const int q0 = blockIdx.x * BQ;
  // K/V blocks this CTA needs (causal: only up to its last query row; Sq == Skv then)
  int kv_len = p.Skv;
  if (p.causal) kv_len = min(p.Skv, q0 + BQ);
  const int n_kv = (kv_len + BKV - 1) / BKV;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(q_full, 1);
    for (int i = 0; i < KV_SLOTS; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&v_full[i], 1);
      mbar_init(&k_empty[i], 8);   // one arrive per consumer warp
      mbar_init(&v_empty[i], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 24;");
    if (threadIdx.x == 0) {
      // ---------------------------------------------------------------- TMA producer
      mbar_expect_tx(q_full, TILE_BYTES);
      for (int half = 0; half < 2; ++half)
        tma_load_3d(q_smem + half * HALF_BYTES, &tmQ, q_full, h * DH + half * 64, q0, b);
      for (int j = 0; j < n_kv; ++j) {
        const int slot = j % KV_SLOTS;
        const uint32_t phase = (j / KV_SLOTS) & 1;
        mbar_wait(&k_empty[slot], phase ^ 1);
        mbar_expect_tx(&k_full[slot], TILE_BYTES);
        for (int half = 0; half < 2; ++half)
          tma_load_3d(k_smem + slot * TILE_BYTES + half * HALF_BYTES, &tmK, &k_full[slot], hk * DH + half * 64, j * BKV, b);
        mbar_wait(&v_empty[slot], phase ^ 1);
        mbar_expect_tx(&v_full[slot], TILE_BYTES);
        for (int half = 0; half < 2; ++half)
          tma_load_3d(v_smem + slot * TILE_BYTES + half * HALF_BYTES, &tmV, &v_full[slot], hk * DH + half * 64, j * BKV, b);
      }
    }
    return;
  }

  // ------------------------------------------------------------------ consumer warpgroups
  asm volatile("setmaxnreg.inc.sync.aligned.u32 240;");
  const int c = wg - 1;
  const int w = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int row0 = q0 + c * 64 + w * 16 + (lane >> 2);   // this thread's rows: row0 and row0 + 8
  const int colq = 2 * (lane & 3);                       // first of its two columns in every 8-column group
  const uint64_t dq0 = make_sdesc_sw128(smem_u32(q_smem) + c * 8192, 16, 1024);
  const uint64_t dk0 = make_sdesc_sw128(smem_u32(k_smem), 16, 1024);
  const uint64_t dv0 = make_sdesc_sw128(smem_u32(v_smem), HALF_BYTES, 1024);
  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};   // l: this thread's partial row sums
  mbar_wait(q_full, 0);
  for (int j = 0; j < n_kv; ++j) {
    const int slot = j % KV_SLOTS;
    const uint32_t phase = (j / KV_SLOTS) & 1;
    float s[64];
    mbar_wait(&k_full[slot], phase);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < DH / 16; ++k) {
      const uint64_t off = uint64_t(((k >> 2) * HALF_BYTES + (k & 3) * 32) >> 4);
      wgmma_m64n128_ss<0, 0>(s, dq0 + off, dk0 + uint64_t((slot * TILE_BYTES) >> 4) + off, k != 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);
    __syncwarp();
    if (lane == 0) mbar_arrive(&k_empty[slot]);

    const int kv0 = j * BKV;
    if (BIAS) {
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        const int row = row0 + 8 * ((i >> 1) & 1);
        const int col = kv0 + 8 * (i >> 2) + colq + (i & 1);
        if (row < p.Sq && col < p.Skv)
          s[i] = fmaf(s[i], p.bias_scale,
                      __bfloat162float(p.bias[(long long)h * p.bias_h_stride + (long long)row * p.bias_row_stride + col]));
      }
    }
    if (kv0 + BKV > p.Skv || p.causal) {
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        const int row = row0 + 8 * ((i >> 1) & 1);
        const int col = kv0 + 8 * (i >> 2) + colq + (i & 1);
        const int limit = p.causal ? min(p.Skv, row + 1) : p.Skv;
        if (col >= limit) s[i] = -INFINITY;
      }
    }
    float alpha[2], neg_m[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < 64; ++i)
        if (((i >> 1) & 1) == r) mx = fmaxf(mx, s[i]);
      mx = quad_max(mx);
      const float m_new = fmaxf(m[r], mx * p.scale_log2);
      alpha[r] = m[r] == -INFINITY ? 0.f : ex2(m[r] - m_new);
      neg_m[r] = m_new == -INFINITY ? 0.f : -m_new;   // fully masked row so far
      m[r] = m_new;
    }
    float sum[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 64; ++i) {
      const int r = (i >> 1) & 1;
      s[i] = ex2(fmaf(s[i], p.scale_log2, neg_m[r]));
      sum[r] += s[i];
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) l[r] = l[r] * alpha[r] + sum[r];
#pragma unroll
    for (int i = 0; i < 64; ++i) o[i] *= alpha[(i >> 1) & 1];

    uint32_t pa[BKV / 16][4];
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) pack_a_frag(s, kk, pa[kk]);
    mbar_wait(&v_full[slot], phase);
    reg_fence(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk)
      wgmma_m64n128_rs<1>(o, pa[kk], dv0 + uint64_t((slot * TILE_BYTES + kk * 2048) >> 4), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(o);
    __syncwarp();
    if (lane == 0) mbar_arrive(&v_empty[slot]);
  }

  // ---------------------------------------------------------------- epilogue: O / l -> bf16
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = row0 + 8 * r;
    const float lt = quad_sum(l[r]);
    const float inv_l = 1.0f / lt;
    if (row >= p.Sq) continue;
    if (p.lse && (lane & 3) == 0) p.lse[((long long)b * p.H + h) * p.lse_stride + row] = m[r] + log2f(lt);
    __nv_bfloat16* out_row = p.out + ((long long)b * p.Sq + row) * p.ldo + (long long)h * DH;
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
      const int i = 4 * jj + 2 * r;
      *reinterpret_cast<uint32_t*>(out_row + 8 * jj + colq) = pack_bf16x2(o[i] * inv_l, o[i + 1] * inv_l);
    }
  }
}

}  // namespace

static int attention_impl(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v,
                          int64_t ldv, void* out, int64_t ldo, int B, int H, int Hkv, int Sq, int Skv,
                          int head_dim, float scale, int causal, const void* bias, int64_t bias_h_stride,
                          int64_t bias_row_stride, float* lse, int64_t lse_stride, cudaStream_t stream) {
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
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(attn_fwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATTN_SMEM);
    if (e != cudaSuccess) return cuda_err(e, "attention smem attribute");
    e = cudaFuncSetAttribute(attn_fwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATTN_SMEM);
    if (e != cudaSuccess) return cuda_err(e, "attention smem attribute");
    attr_set = true;
  }
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
    attn_fwd_kernel<true><<<grid_b, ATTN_THREADS, ATTN_SMEM, stream>>>(tmQ, tmK, tmV, p);
    prof_end(KC_ATTN, stream, (causal ? 2.0 : 4.0) * B * H * (double)Sq * Skv * DH,
             2.0 * DH * B * (2.0 * H * Sq + 2.0 * Hkv * Skv) + 2.0 * H * (double)Sq * Skv);
    B2F_LAUNCHED("attn_fwd_kernel<bias>", 1);
    return B2F_OK;
  }
  dim3 grid((Sq + BQ - 1) / BQ, H, B);
  prof_begin(KC_ATTN, stream);
  attn_fwd_kernel<false><<<grid, ATTN_THREADS, ATTN_SMEM, stream>>>(tmQ, tmK, tmV, p);
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
                        nullptr, 0, 0, nullptr, 0, stream);
}

// forward that also emits the base-2 log-sum-exp rows the backward kernels need (attention_bwd.cu)
extern "C" int b2f_attention_fwd_lse(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv,
                                     void* out, int64_t ldo, int B, int H, int Hkv, int Sq, int Skv, int head_dim,
                                     float scale, int causal, float* lse, int64_t lse_stride, b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!lse) return B2F_ERR_INVALID;
  return attention_impl(q, ldq, k, ldk, v, ldv, out, ldo, B, H, Hkv, Sq, Skv, head_dim, scale, causal, nullptr, 0, 0,
                        lse, lse_stride, stream);
}

extern "C" int b2f_attention_bias_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v,
                                      int64_t ldv, void* out, int64_t ldo, int B, int H, int Hkv, int Sq, int Skv,
                                      int head_dim, float scale, int causal, const void* bias, int64_t bias_h_stride,
                                      int64_t bias_row_stride, b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!bias || bias_row_stride < Skv || bias_h_stride < 0) return B2F_ERR_INVALID;
  return attention_impl(q, ldq, k, ldk, v, ldv, out, ldo, B, H, Hkv, Sq, Skv, head_dim, scale, causal,
                        bias, bias_h_stride, bias_row_stride, nullptr, 0, stream);
}

}  // namespace b2f
