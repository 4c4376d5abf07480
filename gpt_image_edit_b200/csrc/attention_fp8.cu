// FP8 (e4m3) softmax attention for sm_90a, head_dim 128, non-causal (include/b2f.h, "FP8 attention").
//
//   b2f_attn_quant_fp8   bf16 Q / K / V (the pitched views of b2f_attention_fwd) -> q8, k8 [B, S, H*128] with one
//                        scale per (batch item, head), and v8t [B, H, 128, S_pad] (tokens contiguous, in the P-fragment
//                        order of b2f.h) with one scale per (batch item, head, channel);
//   b2f_attention_fp8    the online softmax of attention.cu on those operands: S = Q8 K8^T and O += P8 V8 on the FP8
//                        tensor cores (wgmma m64n128k32 e4m3, fp32 accumulators), P8 = e4m3(256 p) packed in registers
//                        (the factor 256 is folded into the exponent, which saves one multiply per score in a kernel
//                        bound by its softmax).
//
// The attention kernel has the structure of attn_fwd_kernel with 16 KB tiles and shares its shared-memory layout, K / V
// ring and online-softmax step (attention_common.cuh): one TMA producer warpgroup streams K8 / V8t blocks of 128 tokens
// through two slots, two consumer warpgroups own 64 query rows each.  V8t is K-major for the P.V product (FP8
// wgmma takes no MN-major operand), and its token order within every 32-token group makes the m64n128 accumulator
// layout of S the register A fragment of the k32 P.V wgmma, so P converts in place without shuffles.
//
// With a per-item text window (b2f_attn_quant_fp8_window / b2f_attention_fp8_window) the quantizer takes its amaxes
// over the valid tokens only and writes masked tokens as +0 in q8, k8 and v8t; the attention kernel skips the 128-token
// blocks that hold no valid key and masks the scores of the others, so p = 0 meets V = +0 there.
#include <cmath>

#include "attention_common.cuh"

namespace b2f {

using namespace attn;

namespace {

constexpr int F8_TILE = 128 * 128;   // [128 rows][128 bytes], one 128-byte-swizzled TMA box
constexpr int F8_SMEM = FwdSmem<F8_TILE>::BYTES;
constexpr int QTOK = 128;            // tokens per CTA of the quantizer passes

// k-position of token r (0..31) of a 32-token group in v8t: the inverse of
//   token(p) = (p & 16) + 2 ((p & 15) >> 2) + (p & 1) + 8 ((p >> 1) & 1)
__device__ __forceinline__ int v8t_pos(int r) {
  const int lo = r & 15;
  return (r & 16) + 4 * ((lo & 7) >> 1) + (lo & 1) + 2 * (lo >> 3);
}

struct QuantAttnParams {
  const __nv_bfloat16 *q, *k, *v;
  long long ldq, ldk, ldv;
  uint8_t *q8, *k8, *v8t;
  float *sq, *sk, *sv;
  int H, S, S_pad;
  // optional per-item text window int32 [B, 2] (lo, hi): token t < S_txt is valid iff lo <= t < hi
  const int32_t* win;
  int S_txt;
};

// Thread t of a 256-thread CTA covers channels 8 (t % 16) .. + 7 of tokens t / 16 + 16 i (i < 8) of the CTA's block.
__device__ __forceinline__ const __nv_bfloat16* head_row(const __nv_bfloat16* x, long long ld, int b, int S, int tok,
                                                         int h) {
  return x + ((long long)b * S + tok) * ld + (long long)h * DH;
}

// Pass 1: amax of every Q / K head and every V channel, atomicMax on the bits of non-negative floats (order-independent).
__global__ void __launch_bounds__(256) attn_amax_kernel(const QuantAttnParams p) {
  __shared__ float red[8][DH];
  __shared__ float redqk[2][8];
  const int h = blockIdx.y, b = blockIdx.z, t = threadIdx.x;
  const int cc = t & 15, r0 = t >> 4, warp = t >> 5;
  float mq = 0.f, mk = 0.f, mv[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  const int2 tw = p.win ? text_window(p.win, b, p.S_txt) : make_int2(0, 0);
#pragma unroll 4
  for (int i = 0; i < QTOK / 16; ++i) {
    const int tok = blockIdx.x * QTOK + r0 + 16 * i;
    if (tok >= p.S) break;
    if (p.win && in_text_gap(tok, tw, p.S_txt)) continue;
    // Q, K and V as three 16-byte loads issued together, before any of them is used
    const uint4 qv = *reinterpret_cast<const uint4*>(head_row(p.q, p.ldq, b, p.S, tok, h) + 8 * cc);
    const uint4 kv = *reinterpret_cast<const uint4*>(head_row(p.k, p.ldk, b, p.S, tok, h) + 8 * cc);
    const uint4 vv = *reinterpret_cast<const uint4*>(head_row(p.v, p.ldv, b, p.S, tok, h) + 8 * cc);
    mq = amax8(qv, mq);
    mk = amax8(kv, mk);
    float f[8];
    unpack8(vv, f);
#pragma unroll
    for (int j = 0; j < 8; ++j) mv[j] = fmaxf(mv[j], fabsf(f[j]));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mq = fmaxf(mq, __shfl_xor_sync(0xffffffffu, mq, o));
    mk = fmaxf(mk, __shfl_xor_sync(0xffffffffu, mk, o));
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) mv[j] = fmaxf(mv[j], __shfl_xor_sync(0xffffffffu, mv[j], 16));
  if ((t & 31) == 0) {
    redqk[0][warp] = mq;
    redqk[1][warp] = mk;
  }
  if ((t & 31) < 16) {
#pragma unroll
    for (int j = 0; j < 8; ++j) red[warp][8 * cc + j] = mv[j];
  }
  __syncthreads();
  if (t < DH) {
    float m = red[0][t];
#pragma unroll
    for (int w = 1; w < 8; ++w) m = fmaxf(m, red[w][t]);
    atomicMax(reinterpret_cast<int*>(p.sv) + ((long long)b * p.H + h) * DH + t, __float_as_int(m));
  } else if (t < DH + 2) {
    float m = redqk[t - DH][0];
#pragma unroll
    for (int w = 1; w < 8; ++w) m = fmaxf(m, redqk[t - DH][w]);
    atomicMax(reinterpret_cast<int*>(t == DH ? p.sq : p.sk) + (long long)b * p.H + h, __float_as_int(m));
  }
}

// Byte offset of k-position `pos` in row c of the transposed V tile.  The 4-byte words of a row are XOR-swizzled with a
// key that differs between the 16 channel blocks a warp writes at once (channel c = 8 cc + j, j fixed per store), so
// the byte stores of one warp fall into different banks; the read-out below undoes it word by word.
__device__ __forceinline__ int vt_off(int c, int pos) {
  return c * QTOK + (pos ^ ((((c >> 3) ^ (c & 7)) & 15) << 2));
}

// Pass 2: the row rule with the amaxes of pass 1 (still in sq / sk / sv); V is transposed through shared memory.
__global__ void __launch_bounds__(256) attn_quant_kernel(const QuantAttnParams p) {
  __shared__ __align__(16) uint8_t vt[DH * QTOK];   // [channel][k-position], swizzled by vt_off
  const int h = blockIdx.y, b = blockIdx.z, t = threadIdx.x;
  const int cc = t & 15, r0 = t >> 4;
  const long long bh = (long long)b * p.H + h;
  float s_, inv_q, inv_k, inv_v[8];
  row_scale_of(p.sq[bh], s_, inv_q);
  row_scale_of(p.sk[bh], s_, inv_k);
#pragma unroll
  for (int j = 0; j < 8; ++j) row_scale_of(p.sv[bh * DH + 8 * cc + j], s_, inv_v[j]);
  const int2 tw = p.win ? text_window(p.win, b, p.S_txt) : make_int2(0, 0);
#pragma unroll 2
  for (int i = 0; i < QTOK / 16; ++i) {
    const int tl = r0 + 16 * i;
    const int tok = blockIdx.x * QTOK + tl;
    const int pos = (tl & ~31) + v8t_pos(tl & 31);
    const bool masked = p.win && in_text_gap(tok, tw, p.S_txt);
    if (tok >= p.S || masked) {   // padding and masked tokens of v8t are +0 (and masked ones of q8 / k8 too)
#pragma unroll
      for (int j = 0; j < 8; ++j) vt[vt_off(8 * cc + j, pos)] = 0;
      if (masked) {
        const long long o8 = (((long long)b * p.S + tok) * p.H + h) * DH + 8 * cc;
        *reinterpret_cast<uint2*>(p.q8 + o8) = make_uint2(0, 0);
        *reinterpret_cast<uint2*>(p.k8 + o8) = make_uint2(0, 0);
      }
      continue;
    }
    const long long o8 = (((long long)b * p.S + tok) * p.H + h) * DH + 8 * cc;
    float f[8];
    // uint4(...): one 16-byte load each; unpack8's reference argument would let the compiler split it into two 8-byte
    // loads
    unpack8(uint4(*reinterpret_cast<const uint4*>(head_row(p.q, p.ldq, b, p.S, tok, h) + 8 * cc)), f);
    *reinterpret_cast<uint2*>(p.q8 + o8) = inv_q > 0.f ? quant_e4m3x8(f, inv_q) : make_uint2(0, 0);
    unpack8(uint4(*reinterpret_cast<const uint4*>(head_row(p.k, p.ldk, b, p.S, tok, h) + 8 * cc)), f);
    *reinterpret_cast<uint2*>(p.k8 + o8) = inv_k > 0.f ? quant_e4m3x8(f, inv_k) : make_uint2(0, 0);
    unpack8(uint4(*reinterpret_cast<const uint4*>(head_row(p.v, p.ldv, b, p.S, tok, h) + 8 * cc)), f);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint16_t e = cvt_e4m3x2(f[2 * j] * inv_v[2 * j], f[2 * j + 1] * inv_v[2 * j + 1]);
      vt[vt_off(8 * cc + 2 * j, pos)] = inv_v[2 * j] > 0.f ? uint8_t(e & 0xff) : 0;
      vt[vt_off(8 * cc + 2 * j + 1, pos)] = inv_v[2 * j + 1] > 0.f ? uint8_t(e >> 8) : 0;
    }
  }
  __syncthreads();
  uint8_t* dst = p.v8t + bh * DH * p.S_pad + (long long)blockIdx.x * QTOK;
#pragma unroll
  for (int i = 0; i < DH * QTOK / 16 / 256; ++i) {
    const int idx = t + 256 * i;
    const int c = idx >> 3, x = idx & 7;
    uint32_t w[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) w[k] = *reinterpret_cast<const uint32_t*>(&vt[vt_off(c, 16 * x + 4 * k)]);
    *reinterpret_cast<uint4*>(dst + (long long)c * p.S_pad + 16 * x) = make_uint4(w[0], w[1], w[2], w[3]);
  }
}

// Pass 3: the amaxes in sq / sk / sv become the scales of the row rule.
__global__ void __launch_bounds__(256) attn_scale_kernel(float* sq, float* sk, float* sv, int n_heads) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= n_heads * (2 + DH)) return;
  float* x = i < n_heads ? sq + i : i < 2 * n_heads ? sk + (i - n_heads) : sv + (i - 2 * n_heads);
  float s, inv;
  row_scale_of(*x, s, inv);
  *x = s;
}

struct AttnFp8Params {
  int H, S;
  const float *sq, *sk, *sv;
  float scale_log2;
  __nv_bfloat16* out;
  long long ldo;
  const int32_t* win;   // WIN kernel: per-item text window over the first S_txt tokens
  int S_txt;
};

// WIN: the kernel streams the 128-token blocks [lo / BKV, ceil(hi / BKV)) of the text window and then the blocks from
// max(that end, S_txt / BKV) on, at the block positions of the kernel without WIN (v8t's token order lives in 32-token
// groups from token 0, so blocks cannot start at lo); blocks that are not wholly valid mask their invalid scores.  The
// full window (0, S_txt) streams every block and masks exactly the tail the kernel without WIN masks.
template <bool WIN>
__global__ void __launch_bounds__(ATTN_THREADS, 1)
attn_fp8_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const AttnFp8Params p) {
  extern __shared__ uint8_t smem_raw[];
  const FwdSmem<F8_TILE> sm(smem_raw);

  const int wg = __shfl_sync(0xffffffffu, int(threadIdx.x >> 7), 0);
  const int h = blockIdx.y, b = blockIdx.z;
  const int q0 = blockIdx.x * BQ;
  int n_kv = (p.S + BKV - 1) / BKV;
  int2 tw = make_int2(0, 0);
  int n_txt = 0, j_img = 0;   // WIN: blocks [lo / BKV, + n_txt), then [j_img, n_kv) of the unwindowed numbering
  if (WIN) {
    tw = text_window(p.win, b, p.S_txt);
    n_txt = tw.y > tw.x ? (tw.y + BKV - 1) / BKV - tw.x / BKV : 0;
    j_img = max(tw.x / BKV + n_txt, p.S_txt / BKV);
    n_kv = n_txt + max(n_kv - j_img, 0);
  }
  auto kv_block = [&](int j) { return !WIN ? j : j < n_txt ? tw.x / BKV + j : j_img + (j - n_txt); };

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
      mbar_expect_tx(sm.q_full, F8_TILE);
      tma_load_3d(sm.q, &tmQ, sm.q_full, h * DH, q0, b);
      // K8 block j: one box of 128 tokens; V8t block j: the same tokens' columns of the head's [128][S_pad] item
      sm.produce_kv(
          n_kv, [&](int j, uint8_t* dst, uint64_t* bar) { tma_load_3d(dst, &tmK, bar, h * DH, kv_block(j) * BKV, b); },
          [&](int j, uint8_t* dst, uint64_t* bar) { tma_load_3d(dst, &tmV, bar, kv_block(j) * BKV, 0, b * p.H + h); });
    }
    return;
  }

  // ------------------------------------------------------------------ consumer warpgroups
  setmaxnreg_inc<CONSUMER_REGS>();
  const auto [c, w, lane, row0, colq] = consumer_pos(wg, q0);
  const long long bh = (long long)b * p.H + h;
  // score scale of this head: fp32(fp32(sq * sk) * fp32(scale * log2 e))
  const float cl = p.sq[bh] * p.sk[bh] * p.scale_log2;
  const uint64_t dq0 = make_sdesc_sw128(smem_u32(sm.q) + c * 8192, 16, 1024);
  const uint64_t dk0 = make_sdesc_sw128(smem_u32(sm.k), 16, 1024);
  const uint64_t dv0 = make_sdesc_sw128(smem_u32(sm.v), 16, 1024);
  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  // m: running max of the base-2 scores t; l: this thread's partial row sums of p' = 256 p
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  const uint32_t one = uint32_t(n_kv > 0);   // scale-d in a register: a constant is materialized between the wgmmas
  mbar_wait(sm.q_full, 0);
  for (int j = 0; j < n_kv; ++j) {
    const int slot = j % KV_SLOTS;
    const uint32_t phase = (j / KV_SLOTS) & 1;
    float s[64];
    mbar_wait(&sm.k_full[slot], phase);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < DH / 32; ++k)
      wgmma_m64n128k32_e4m3_ss(s, dq0 + uint64_t(k * 2), dk0 + uint64_t((slot * F8_TILE) >> 4) + uint64_t(k * 2),
                               k != 0 ? one : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);
    consumer_release(&sm.k_empty[slot], lane);

    const int kv0 = kv_block(j) * BKV;
    if (WIN) {
      const int kv1 = kv0 + BKV;
      const bool whole = (kv0 >= tw.x && kv1 <= tw.y) || (kv0 >= (tw.y == p.S_txt ? tw.x : p.S_txt) && kv1 <= p.S);
      if (!whole) {   // masked text columns and the tail give p = 0
#pragma unroll
        for (int i = 0; i < 64; ++i) {
          const int col = kv0 + acc_col(i, colq);
          if (col >= p.S || in_text_gap(col, tw, p.S_txt)) s[i] = -INFINITY;
        }
      }
    } else if (kv0 + BKV > p.S) {   // masked tail columns give p = 0
#pragma unroll
      for (int i = 0; i < 64; ++i)
        if (kv0 + acc_col(i, colq) >= p.S) s[i] = -INFINITY;
    }
    float alpha[2];
    softmax_step<8>(s, m, l, cl, alpha);   // p' = ex2(t - m + 8) = 256 p
    if (__any_sync(0xffffffffu, alpha[0] != 1.f || alpha[1] != 1.f)) {   // exact: skipping a multiply by 1
#pragma unroll
      for (int i = 0; i < 64; ++i) o[i] *= alpha[acc_row(i) / 8];
    }

    // P8 = e4m3(p') as the A fragments of the four k32 steps (ptx.cuh, wgmma_m64n128k32_e4m3_rs): step kk covers
    // accumulator elements [16 kk, 16 kk + 16), whose columns are v8t's k-positions of that 32-token group
    uint32_t pa[BKV / 32][4];
#pragma unroll
    for (int kk = 0; kk < BKV / 32; ++kk) {
      const float* e = s + 16 * kk;
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int i0 = 8 * (r >> 1) + 2 * (r & 1);   // r: row g / g + 8 (bit 0), k 4t.. / 16 + 4t.. (bit 1)
        pa[kk][r] = uint32_t(cvt_e4m3x2(e[i0], e[i0 + 1])) |
                    (uint32_t(cvt_e4m3x2(e[i0 + 4], e[i0 + 5])) << 16);
      }
    }
    mbar_wait(&sm.v_full[slot], phase);
    reg_fence(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BKV / 32; ++kk)
      wgmma_m64n128k32_e4m3_rs(o, pa[kk], dv0 + uint64_t((slot * F8_TILE + kk * 32) >> 4), one);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(o);
    consumer_release(&sm.v_empty[slot], lane);
  }

  // ---------------------------------------------------------------- epilogue: bf16((O * sv) * (1 / l'))
  // sv is applied here, not by scaling o in place for store_row_bf16: that form changed the consumer loop's register
  // allocation and took 1.25-1.29 ms instead of 1.15-1.20 ms at B 1, H 24, S 8736 (H100 80GB HBM3, 700 W)
  const float* svh = p.sv + bh * DH;
  float fv[32];
#pragma unroll
  for (int jj = 0; jj < 16; ++jj) {
    fv[2 * jj] = svh[8 * jj + colq];
    fv[2 * jj + 1] = svh[8 * jj + colq + 1];
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = row0 + 8 * r;
    const float inv_l = 1.0f / quad_sum(l[r]);
    if (row >= p.S) continue;
    __nv_bfloat16* out_row = p.out + ((long long)b * p.S + row) * p.ldo + (long long)h * DH;
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
      const int i = 4 * jj + 2 * r;
      *reinterpret_cast<uint32_t*>(out_row + 8 * jj + colq) =
          pack_bf16x2(o[i] * fv[2 * jj] * inv_l, o[i + 1] * fv[2 * jj + 1] * inv_l);
    }
  }
}

bool misaligned16(const void* a) { return reinterpret_cast<uintptr_t>(a) & 15; }

}  // namespace

static int attn_quant_fp8_impl(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv,
                               void* q8, void* k8, float* sq, float* sk, void* v8t, float* sv, int B, int H, int S,
                               int head_dim, const int32_t* win, int S_txt, cudaStream_t stream) {
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (!q || !k || !v || !q8 || !k8 || !sq || !sk || !v8t || !sv || B <= 0 || H <= 0 || S <= 0) return B2F_ERR_INVALID;
  if (head_dim != DH) return B2F_ERR_UNSUPPORTED;
  if ((ldq & 7) || (ldk & 7) || (ldv & 7)) return B2F_ERR_ALIGN;
  if (misaligned16(q) || misaligned16(k) || misaligned16(v) || misaligned16(q8) || misaligned16(k8) ||
      misaligned16(v8t))
    return B2F_ERR_ALIGN;
  const int nblk = (S + QTOK - 1) / QTOK;
  QuantAttnParams p{static_cast<const __nv_bfloat16*>(q), static_cast<const __nv_bfloat16*>(k),
                    static_cast<const __nv_bfloat16*>(v), ldq, ldk, ldv, static_cast<uint8_t*>(q8),
                    static_cast<uint8_t*>(k8), static_cast<uint8_t*>(v8t), sq, sk, sv, H, S, nblk * QTOK, win, S_txt};
  const size_t heads = (size_t)B * H;
  cudaError_t e = cudaMemsetAsync(sq, 0, heads * sizeof(float), stream);
  if (e == cudaSuccess) e = cudaMemsetAsync(sk, 0, heads * sizeof(float), stream);
  if (e == cudaSuccess) e = cudaMemsetAsync(sv, 0, heads * DH * sizeof(float), stream);
  if (e != cudaSuccess) return cuda_err(e, "attn_quant_fp8 memset");
  const dim3 grid(nblk, H, B);
  const double elems = (double)B * S * H * DH;
  prof_begin(KC_OTHER, stream);
  attn_amax_kernel<<<grid, 256, 0, stream>>>(p);
  attn_quant_kernel<<<grid, 256, 0, stream>>>(p);
  const int n = (int)(heads * (2 + DH));
  attn_scale_kernel<<<(n + 255) / 256, 256, 0, stream>>>(sq, sk, sv, (int)heads);
  // both passes read Q, K and V; the second writes q8, k8 and v8t
  prof_end(KC_OTHER, stream, 0.0, 12.0 * elems + 2.0 * elems + (double)B * H * DH * nblk * QTOK);
  B2F_LAUNCHED("attn_quant_fp8 kernels", 3);
  return B2F_OK;
}

extern "C" int b2f_attn_quant_fp8(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv,
                                  void* q8, void* k8, float* sq, float* sk, void* v8t, float* sv, int B, int H, int S,
                                  int head_dim, b2f_stream_t stream) {
  return attn_quant_fp8_impl(q, ldq, k, ldk, v, ldv, q8, k8, sq, sk, v8t, sv, B, H, S, head_dim, nullptr, 0,
                             static_cast<cudaStream_t>(stream));
}

extern "C" int b2f_attn_quant_fp8_window(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v,
                                         int64_t ldv, void* q8, void* k8, float* sq, float* sk, void* v8t, float* sv,
                                         int B, int H, int S, int head_dim, const int32_t* win, int S_txt,
                                         b2f_stream_t stream) {
  if (!win || S_txt < 0 || S_txt > S) return B2F_ERR_INVALID;
  return attn_quant_fp8_impl(q, ldq, k, ldk, v, ldv, q8, k8, sq, sk, v8t, sv, B, H, S, head_dim, win, S_txt,
                             static_cast<cudaStream_t>(stream));
}

static int attention_fp8_impl(const void* q8, const void* k8, const float* sq, const float* sk, const void* v8t,
                              const float* sv, void* out, int64_t ldo, int B, int H, int S, int head_dim, float scale,
                              int causal, const int32_t* win, int S_txt, cudaStream_t stream) {
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (!q8 || !k8 || !sq || !sk || !v8t || !sv || !out || B <= 0 || H <= 0 || S <= 0) return B2F_ERR_INVALID;
  if (head_dim != DH || causal) return B2F_ERR_UNSUPPORTED;
  if (ldo & 7) return B2F_ERR_ALIGN;
  if (misaligned16(q8) || misaligned16(k8) || misaligned16(v8t) || misaligned16(out)) return B2F_ERR_ALIGN;
  static bool attr_set = false;
  if (int rc = set_max_smem_once(attr_set, F8_SMEM, "attention fp8 smem attribute", attn_fp8_kernel<false>,
                                 attn_fp8_kernel<true>))
    return rc;
  const uint64_t width = (uint64_t)H * DH;
  const uint64_t S_pad = (uint64_t)(S + BKV - 1) / BKV * BKV;
  CUtensorMap tmQ, tmK, tmV;
  int rc = make_tmap_u8_rows(&tmQ, q8, 3, width, S, B, width, (uint64_t)S * width);
  if (rc) return rc;
  rc = make_tmap_u8_rows(&tmK, k8, 3, width, S, B, width, (uint64_t)S * width);
  if (rc) return rc;
  // v8t [B, H, 128, S_pad] as B*H items of [128 channels][S_pad tokens]
  rc = make_tmap_u8_rows(&tmV, v8t, 3, S_pad, DH, (uint64_t)B * H, S_pad, DH * S_pad);
  if (rc) return rc;
  // fp32(scale * log2 e) with the product of the fp32 scale taken in double
  AttnFp8Params p{H, S, sq, sk, sv, float((double)scale * 1.4426950408889634), static_cast<__nv_bfloat16*>(out), ldo,
                  win, S_txt};
  const dim3 grid((S + BQ - 1) / BQ, H, B);
  prof_begin(KC_ATTN, stream);
  if (win)
    attn_fp8_kernel<true><<<grid, ATTN_THREADS, F8_SMEM, stream>>>(tmQ, tmK, tmV, p);
  else
    attn_fp8_kernel<false><<<grid, ATTN_THREADS, F8_SMEM, stream>>>(tmQ, tmK, tmV, p);
  char tag[64];
  snprintf(tag, sizeof tag, "attn fp8 B%d H%d S%d", B, H, S);
  prof_end_tagged(KC_ATTN, stream, 4.0 * B * H * (double)S * S * DH,
                  (double)DH * B * H * (2.0 * S + S_pad) + 2.0 * DH * B * H * (double)S, tag);
  B2F_LAUNCHED(win ? "attn_fp8_kernel<window>" : "attn_fp8_kernel", 1);
  return B2F_OK;
}

extern "C" int b2f_attention_fp8(const void* q8, const void* k8, const float* sq, const float* sk, const void* v8t,
                                 const float* sv, void* out, int64_t ldo, int B, int H, int S, int head_dim,
                                 float scale, int causal, b2f_stream_t stream) {
  return attention_fp8_impl(q8, k8, sq, sk, v8t, sv, out, ldo, B, H, S, head_dim, scale, causal, nullptr, 0,
                            static_cast<cudaStream_t>(stream));
}

extern "C" int b2f_attention_fp8_window(const void* q8, const void* k8, const float* sq, const float* sk,
                                        const void* v8t, const float* sv, void* out, int64_t ldo, int B, int H, int S,
                                        int head_dim, float scale, const int32_t* win, int S_txt,
                                        b2f_stream_t stream) {
  if (!win || S_txt < 0 || S_txt > S) return B2F_ERR_INVALID;
  return attention_fp8_impl(q8, k8, sq, sk, v8t, sv, out, ldo, B, H, S, head_dim, scale, 0, win, S_txt,
                            static_cast<cudaStream_t>(stream));
}

}  // namespace b2f
