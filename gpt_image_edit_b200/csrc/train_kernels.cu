// HBM-bound kernels of the stage-2 training step (reference train_denoiser.py:829-1181): the backward of every
// fused row kernel of the MMDiT block, the flow-matching loss, gradient-norm and AdamW.  The reference reaches all
// of these through torch.autograd over diffusers' eager ops, DeepSpeed's fused Adam and accelerate's
// clip_grad_norm_ (train_denoiser.py:596-602, 1172-1181).
//
// Conventions: activations and activation gradients are bf16 (what autograd produces for bf16 modules), all
// arithmetic is fp32, parameter gradients and every reduction over tokens are fp32.  Column reductions over tokens
// (bias / gate / scale / shift / RMSNorm-weight gradients) are two-stage and deterministic: each block writes a
// partial row into a caller-provided fp32 scratch, `col_reduce` sums the partial rows in a fixed order.
#include "host_common.h"
#include "ptx.cuh"

namespace b2f {

namespace {

constexpr int CHUNK_ROWS = 32;   // token rows per block of the column-reduction kernels

// ------------------------------------------------------------------------------------------------
// x + gate * y  (forward, training mode: y is kept for the gate gradient) and its backward
//   fwd:  out = bf16(x + bf16(gate[b] * y))                       (the GEMM's GATE_RESID epilogue, unfused)
//   bwd:  dy = bf16(gate[b] * dout);  dgate[b, c] = sum_rows dout * y;   (y == null: plain column sum of dout)
// Rows [0, split_row) use `gate`, the others `gate_b` (text / image stream of a double block).
// Partial sums cover rows >= part_row0 only (the image stream, whose AdaLN linear is trainable).
struct GateParams {
  const __nv_bfloat16* x;     // fwd: residual; bwd: dout
  const __nv_bfloat16* y;
  const __nv_bfloat16* gate;
  const __nv_bfloat16* gate_b;
  __nv_bfloat16* out;         // fwd: x + gate*y; bwd: dy (may be null)
  float* partial;             // bwd: [batch, nchunks, D]
  long long ldx, x_bs, ldy, y_bs, ldo, o_bs, gate_ld;
  int batch, rows, D, split_row, part_row0;
};

__global__ void __launch_bounds__(128) gate_resid_fwd_kernel(const GateParams p) {
  const int c = (blockIdx.y * 128 + threadIdx.x) * 8;
  if (c >= p.D) return;
  const int b = blockIdx.z;
  const int r0 = blockIdx.x * CHUNK_ROWS;
  float g[8], gb[8];
  unpack8(__ldg(reinterpret_cast<const uint4*>(p.gate + (long long)b * p.gate_ld + c)), g);
  if (p.split_row > 0) unpack8(__ldg(reinterpret_cast<const uint4*>(p.gate_b + (long long)b * p.gate_ld + c)), gb);
  for (int r = r0; r < min(r0 + CHUNK_ROWS, p.rows); ++r) {
    float x[8], y[8], o[8];
    unpack8(*reinterpret_cast<const uint4*>(p.x + b * p.x_bs + r * p.ldx + c), x);
    unpack8(*reinterpret_cast<const uint4*>(p.y + b * p.y_bs + r * p.ldy + c), y);
    const bool second = p.split_row > 0 && r >= p.split_row;
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = x[j] + bf16r((second ? gb[j] : g[j]) * y[j]);
    *reinterpret_cast<uint4*>(p.out + b * p.o_bs + r * p.ldo + c) = pack8(o);
  }
}

__global__ void __launch_bounds__(128) gate_bwd_kernel(const GateParams p) {
  const int c = (blockIdx.y * 128 + threadIdx.x) * 8;
  if (c >= p.D) return;
  const int b = blockIdx.z;
  const int r0 = blockIdx.x * CHUNK_ROWS;
  float g[8], gb[8], acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f, g[j] = 1.f, gb[j] = 1.f;
  if (p.gate) {
    unpack8(__ldg(reinterpret_cast<const uint4*>(p.gate + (long long)b * p.gate_ld + c)), g);
    if (p.split_row > 0) unpack8(__ldg(reinterpret_cast<const uint4*>(p.gate_b + (long long)b * p.gate_ld + c)), gb);
  }
  for (int r = r0; r < min(r0 + CHUNK_ROWS, p.rows); ++r) {
    float d[8];
    unpack8(*reinterpret_cast<const uint4*>(p.x + b * p.x_bs + r * p.ldx + c), d);
    if (p.partial && r >= p.part_row0) {
      if (p.y) {
        float y[8];
        unpack8(*reinterpret_cast<const uint4*>(p.y + b * p.y_bs + r * p.ldy + c), y);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = fmaf(d[j], y[j], acc[j]);
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += d[j];
      }
    }
    if (p.out) {
      const bool second = p.split_row > 0 && r >= p.split_row;
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (second ? gb[j] : g[j]) * d[j];
      *reinterpret_cast<uint4*>(p.out + b * p.o_bs + r * p.ldo + c) = pack8(o);
    }
  }
  if (p.partial) {
    float* dst = p.partial + ((long long)b * gridDim.x + blockIdx.x) * p.D + c;
    *reinterpret_cast<float4*>(dst) = make_float4(acc[0], acc[1], acc[2], acc[3]);
    *reinterpret_cast<float4*>(dst + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
  }
}

// out[b, c] (+)= sum_chunk partial[b, chunk, c]   (fixed summation order)
__global__ void __launch_bounds__(256) col_reduce_kernel(const float* partial, int nchunks, int D, float* out,
                                                         long long out_ld, int accumulate) {
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c >= D) return;
  const int b = blockIdx.y;
  const float* src = partial + (long long)b * nchunks * D + c;
  float s = 0.f;
  for (int k = 0; k < nchunks; ++k) s += src[(long long)k * D];
  float* o = out + (long long)b * out_ld + c;
  *o = accumulate ? *o + s : s;
}

// ------------------------------------------------------------------------------------------------
// Backward of AdaLN modulate  y = LN(x) * (1 + scale[b]) + shift[b]   (ln_modulate_kernel, elementwise.cu):
//   xhat = (x - mean) * rstd;  g = dy * bf16(1 + scale);  dx = rstd * (g - mean(g) - xhat * mean(g * xhat))
//   dres_out = bf16(dres_in + bf16(dx))        (the LN branch joins the residual-stream gradient)
//   dscale[b, c] = sum_rows dy * xhat;   dshift[b, c] = sum_rows dy            (rows >= part_row0)
// One block per CHUNK_LN rows: phase 1, a warp per row computes (mean, rstd, mean(g), mean(g xhat)) into smem;
// phase 2, a thread per 8 columns walks the rows, writes dx and accumulates the column sums in registers.
constexpr int CHUNK_LN = 16;
struct LnBwdParams {
  const __nv_bfloat16* x;
  const __nv_bfloat16* dy;
  const __nv_bfloat16* scale;
  const __nv_bfloat16* scale_b;
  const __nv_bfloat16* dres_in;   // may be null (no residual gradient yet)
  __nv_bfloat16* dres_out;
  float* partial;                 // [batch, nchunks, 2*D]: dscale | dshift  (may be null)
  long long ldx, x_bs, ldy, dy_bs, ldr, r_bs, ldo, o_bs, mod_ld;
  int batch, rows, D, split_row, part_row0;
  float eps;
};

__global__ void __launch_bounds__(256) ln_modulate_bwd_kernel(const LnBwdParams p) {
  __shared__ float st[CHUNK_LN][4];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.y;
  const int r0 = blockIdx.x * CHUNK_LN;
  const int nrows = min(CHUNK_LN, p.rows - r0);
  const float inv_d = 1.0f / float(p.D);
  for (int i = warp; i < nrows; i += 8) {
    const int r = r0 + i;
    const __nv_bfloat16* xr = p.x + b * p.x_bs + r * p.ldx;
    const __nv_bfloat16* dr = p.dy + b * p.dy_bs + r * p.ldy;
    const bool second = p.split_row > 0 && r >= p.split_row;
    const __nv_bfloat16* sc = (second ? p.scale_b : p.scale) + (long long)b * p.mod_ld;
    float s = 0.f;
    for (int c = lane * 8; c < p.D; c += 256) {
      float v[8];
      unpack8(*reinterpret_cast<const uint4*>(xr + c), v);
#pragma unroll
      for (int j = 0; j < 8; ++j) s += v[j];
    }
    const float mean = warp_sum(s) * inv_d;
    float ss = 0.f;
    for (int c = lane * 8; c < p.D; c += 256) {
      float v[8];
      unpack8(*reinterpret_cast<const uint4*>(xr + c), v);
#pragma unroll
      for (int j = 0; j < 8; ++j) ss += (v[j] - mean) * (v[j] - mean);
    }
    const float rstd = rsqrtf(warp_sum(ss) * inv_d + p.eps);
    float c1 = 0.f, c2 = 0.f;
    for (int c = lane * 8; c < p.D; c += 256) {
      float v[8], d[8], a[8];
      unpack8(*reinterpret_cast<const uint4*>(xr + c), v);
      unpack8(*reinterpret_cast<const uint4*>(dr + c), d);
      unpack8(__ldg(reinterpret_cast<const uint4*>(sc + c)), a);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float g = d[j] * bf16r(1.0f + a[j]);
        c1 += g;
        c2 = fmaf(g, (v[j] - mean) * rstd, c2);
      }
    }
    c1 = warp_sum(c1) * inv_d;
    c2 = warp_sum(c2) * inv_d;
    if (lane == 0) {
      st[i][0] = mean;
      st[i][1] = rstd;
      st[i][2] = c1;
      st[i][3] = c2;
    }
  }
  __syncthreads();
  for (int c = threadIdx.x * 8; c < p.D; c += 2048) {
    float a0[8], a1[8], t0[8], t1[8], ds[8], dh[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(p.scale + (long long)b * p.mod_ld + c)), a0);
    if (p.split_row > 0) unpack8(__ldg(reinterpret_cast<const uint4*>(p.scale_b + (long long)b * p.mod_ld + c)), a1);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      t0[j] = bf16r(1.0f + a0[j]);
      t1[j] = p.split_row > 0 ? bf16r(1.0f + a1[j]) : t0[j];
      ds[j] = dh[j] = 0.f;
    }
    for (int i = 0; i < nrows; ++i) {
      const int r = r0 + i;
      const float mean = st[i][0], rstd = st[i][1], c1 = st[i][2], c2 = st[i][3];
      const bool second = p.split_row > 0 && r >= p.split_row;
      float v[8], d[8], o[8];
      unpack8(*reinterpret_cast<const uint4*>(p.x + b * p.x_bs + r * p.ldx + c), v);
      unpack8(*reinterpret_cast<const uint4*>(p.dy + b * p.dy_bs + r * p.ldy + c), d);
      if (p.dres_in)
        unpack8(*reinterpret_cast<const uint4*>(p.dres_in + b * p.r_bs + r * p.ldr + c), o);
      else {
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = 0.f;
      }
      const bool part = p.partial && r >= p.part_row0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float xh = (v[j] - mean) * rstd;
        const float g = d[j] * (second ? t1[j] : t0[j]);
        const float dx = rstd * (g - c1 - xh * c2);
        o[j] += bf16r(dx);
        if (part) {
          ds[j] = fmaf(d[j], bf16r(xh), ds[j]);
          dh[j] += d[j];
        }
      }
      *reinterpret_cast<uint4*>(p.dres_out + b * p.o_bs + r * p.ldo + c) = pack8(o);
    }
    if (p.partial) {
      float* dst = p.partial + ((long long)b * gridDim.x + blockIdx.x) * 2 * p.D;
      *reinterpret_cast<float4*>(dst + c) = make_float4(ds[0], ds[1], ds[2], ds[3]);
      *reinterpret_cast<float4*>(dst + c + 4) = make_float4(ds[4], ds[5], ds[6], ds[7]);
      *reinterpret_cast<float4*>(dst + p.D + c) = make_float4(dh[0], dh[1], dh[2], dh[3]);
      *reinterpret_cast<float4*>(dst + p.D + c + 4) = make_float4(dh[4], dh[5], dh[6], dh[7]);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Backward of per-head RMSNorm + interleaved-pair RoPE (rmsnorm_rope_out_kernel / the QKV GEMM epilogue):
//   fwd: r = rsqrt(mean(x^2) + eps); y = x r w; o = rope(y)
//   bwd: dy0 = do0 c0 + do1 s1, dy1 = do1 c1 - do0 s0;  dw += dy x r;  g = dy w;
//        dx = r (g - x r^2 mean(g x))
// In place on the Q and K column blocks of the gradient buffer; x is read from the saved pre-norm projections.
// Each block of 8 warps (8 tokens) writes one partial row [wq_a | wk_a | wq_b | wk_b] x 128 of weight gradients.
struct NormRopeBwdParams {
  __nv_bfloat16* dq;
  __nv_bfloat16* dk;
  const __nv_bfloat16* xq;
  const __nv_bfloat16* xk;
  long long ld, batch_stride, ldx, x_batch_stride;
  const __nv_bfloat16 *wq_a, *wk_a, *wq_b, *wk_b;
  const float* cos;
  const float* sin;
  float* partial;   // [nblocks, 512]
  int batch, S, H, n_a;
  float eps;
};

__global__ void __launch_bounds__(256) rmsnorm_rope_bwd_kernel(const NormRopeBwdParams p) {
  // per-warp weight-gradient rows, summed in a fixed order afterwards (no atomics: bit-reproducible)
  __shared__ float acc_sm[8][256];
  __shared__ int set_sm[8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long tok = (long long)blockIdx.x * 8 + warp;
  const int is_k = lane >> 4;
  const int l16 = lane & 15;
  float dw[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) dw[j] = 0.f;
  int my_set = -1;   // -1: no token, 0: weight set a (text rows), 1: set b
  if (tok < (long long)p.batch * p.S) {
    const int b = int(tok / p.S);
    const int s = int(tok - (long long)b * p.S);
    __nv_bfloat16* gbase = (is_k ? p.dk : p.dq) + b * p.batch_stride + s * p.ld + l16 * 8;
    const __nv_bfloat16* xbase = (is_k ? p.xk : p.xq) + b * p.x_batch_stride + s * p.ldx + l16 * 8;
    const bool set_a = s < p.n_a;
    my_set = set_a ? 0 : 1;
    const __nv_bfloat16* wptr = is_k ? (set_a ? p.wk_a : p.wk_b) : (set_a ? p.wq_a : p.wq_b);
    float w[8], cs[8], sn[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(wptr + l16 * 8)), w);
    {
      const float4* c4 = reinterpret_cast<const float4*>(p.cos + (long long)s * 128 + l16 * 8);
      const float4* s4 = reinterpret_cast<const float4*>(p.sin + (long long)s * 128 + l16 * 8);
      const float4 c0 = __ldg(c4), c1 = __ldg(c4 + 1), s0 = __ldg(s4), s1 = __ldg(s4 + 1);
      cs[0] = c0.x; cs[1] = c0.y; cs[2] = c0.z; cs[3] = c0.w;
      cs[4] = c1.x; cs[5] = c1.y; cs[6] = c1.z; cs[7] = c1.w;
      sn[0] = s0.x; sn[1] = s0.y; sn[2] = s0.z; sn[3] = s0.w;
      sn[4] = s1.x; sn[5] = s1.y; sn[6] = s1.z; sn[7] = s1.w;
    }
#pragma unroll 2
    for (int h = 0; h < p.H; ++h) {
      float x[8], d[8], dy[8], o[8];
      unpack8(*reinterpret_cast<const uint4*>(xbase + h * 128), x);
      unpack8(*reinterpret_cast<const uint4*>(gbase + h * 128), d);
      float ss = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) ss += x[j] * x[j];
#pragma unroll
      for (int o2 = 8; o2 > 0; o2 >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o2);
      const float r = rsqrtf(ss * (1.0f / 128.0f) + p.eps);
      float gx = 0.f;
#pragma unroll
      for (int j = 0; j < 8; j += 2) {
        dy[j] = d[j] * cs[j] + d[j + 1] * sn[j + 1];
        dy[j + 1] = d[j + 1] * cs[j + 1] - d[j] * sn[j];
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        dw[j] = fmaf(dy[j], bf16r(x[j] * r), dw[j]);
        gx = fmaf(dy[j] * w[j], x[j], gx);
      }
#pragma unroll
      for (int o2 = 8; o2 > 0; o2 >>= 1) gx += __shfl_xor_sync(0xffffffffu, gx, o2);
      const float k2 = r * r * gx * (1.0f / 128.0f);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = r * (dy[j] * w[j] - x[j] * k2);
      *reinterpret_cast<uint4*>(gbase + h * 128) = pack8(o);
    }
  }
  if (!p.partial) return;
  float* dst = &acc_sm[warp][is_k * 128 + l16 * 8];
#pragma unroll
  for (int j = 0; j < 8; ++j) dst[j] = dw[j];
  if (lane == 0) set_sm[warp] = my_set;
  __syncthreads();
  for (int i = threadIdx.x; i < 512; i += 256) {
    const int set = i >> 8, c = i & 255;
    float sum = 0.f;
#pragma unroll
    for (int wi = 0; wi < 8; ++wi)
      if (set_sm[wi] == set) sum += acc_sm[wi][c];
    p.partial[(long long)blockIdx.x * 512 + i] = sum;
  }
}

// ------------------------------------------------------------------------------------------------
// y = gelu_tanh(x) over a [rows, D] view (training forward keeps the pre-activation for B2F_EPI_DGELU)
__global__ void __launch_bounds__(256) gelu_rows_kernel(const __nv_bfloat16* x, long long ldx, __nv_bfloat16* y,
                                                        long long ldy, long long rows, int D) {
  const long long per_row = D / 8;
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= rows * per_row) return;
  const long long r = i / per_row;
  const int c = int(i - r * per_row) * 8;
  float v[8];
  unpack8(*reinterpret_cast<const uint4*>(x + r * ldx + c), v);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float u = v[j];
    const float inner = 0.7978845608028654f * (u + 0.044715f * u * u * u);
    v[j] = 0.5f * u * (1.0f + tanhf(inner));
  }
  *reinterpret_cast<uint4*>(y + r * ldy + c) = pack8(v);
}

// ------------------------------------------------------------------------------------------------
// dW[n, k] (+)= sum_b dmod[b, n] * act[b, k]   — weight gradient of an AdaLN linear (its input is one row per
// batch item, so the gradient is a sum of B outer products); dmod fp32, act = silu(temb) bf16, dW fp32.
__global__ void __launch_bounds__(256) outer_acc_kernel(const float* dmod, long long dmod_ld, const __nv_bfloat16* act,
                                                        long long act_ld, float* dW, long long ldw, int B, int N, int K,
                                                        int accumulate) {
  const int k = (blockIdx.x * 256 + threadIdx.x) * 4;
  const int n = blockIdx.y;
  if (k >= K) return;
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int b = 0; b < B; ++b) {
    const float g = __ldg(dmod + (long long)b * dmod_ld + n);
    const uint2 q = __ldg(reinterpret_cast<const uint2*>(act + (long long)b * act_ld + k));
    const float2 lo = unpack_bf16x2(q.x), hi = unpack_bf16x2(q.y);
    a.x = fmaf(g, lo.x, a.x);
    a.y = fmaf(g, lo.y, a.y);
    a.z = fmaf(g, hi.x, a.z);
    a.w = fmaf(g, hi.y, a.w);
  }
  float4* o = reinterpret_cast<float4*>(dW + (long long)n * ldw + k);
  if (accumulate) {
    const float4 old = *o;
    a.x += old.x; a.y += old.y; a.z += old.z; a.w += old.w;
  }
  *o = a;
}

// ------------------------------------------------------------------------------------------------
// Attention backward preprocessing: delta[b, h, s] = sum_c dO[b, s, h, c] * O[b, s, h, c]; rows s in [S, S_pad)
// get delta = 0 and lse = +inf so that the backward kernels see P = 0 there.  Half a warp per head vector.
__global__ void __launch_bounds__(256) attn_delta_kernel(const __nv_bfloat16* o, long long ldo, const __nv_bfloat16* dout,
                                                         long long lddo, float* delta, float* lse, int B, int H, int S,
                                                         int S_pad) {
  const long long hv = ((long long)blockIdx.x * 256 + threadIdx.x) >> 4;   // head-vector index
  const int l16 = threadIdx.x & 15;
  const long long total = (long long)B * H * S_pad;
  if (hv >= total) return;
  const int s = int(hv % S_pad);
  const int h = int((hv / S_pad) % H);
  const int b = int(hv / ((long long)S_pad * H));
  float acc = 0.f;
  if (s < S) {
    float a[8], d[8];
    unpack8(*reinterpret_cast<const uint4*>(o + ((long long)b * S + s) * ldo + h * 128 + l16 * 8), a);
    unpack8(*reinterpret_cast<const uint4*>(dout + ((long long)b * S + s) * lddo + h * 128 + l16 * 8), d);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc = fmaf(a[j], d[j], acc);
  }
#pragma unroll
  for (int off = 8; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  if (l16 == 0) {
    delta[hv] = acc;
    if (s >= S) lse[hv] = __int_as_float(0x7f800000);
  }
}

// ------------------------------------------------------------------------------------------------
// Flow-matching loss (reference train_denoiser.py:1105-1167, default weighting = 1):
//   loss = mean_over_all( w * (pred - target)^2 );   dpred = bf16( 2 w (pred - target) * grad_scale / n )
// target fp32 (= noise - x0), pred bf16, w: optional fp32 per-element weights.
__global__ void __launch_bounds__(256) mse_loss_kernel(const __nv_bfloat16* pred, const float* target, const float* w,
                                                       __nv_bfloat16* dpred, float* partial, long long n, float gscale,
                                                       float inv_n) {
  __shared__ float red[8];
  float acc = 0.f;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const float d = __bfloat162float(pred[i]) - target[i];
    const float wi = w ? w[i] : 1.0f;
    acc = fmaf(wi * d, d, acc);
    if (dpred) dpred[i] = __float2bfloat16_rn(2.0f * wi * d * gscale);
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < 8; ++i) s += red[i];
    partial[blockIdx.x] = s * inv_n;
  }
}

// ------------------------------------------------------------------------------------------------
// Gradient norm and AdamW on flat fp32 shards (reference: accelerator.clip_grad_norm_ + torch/DeepSpeed AdamW,
// train_denoiser.py:596-602, 1174-1181).
// 16-byte accesses, four independent ones in flight per thread and array: the optimizer kernels are pure streams over the
// trainable set (4.04 B fp32 values at stage 2), scalar 4-byte grid-stride loops left them at ~4.6 TB/s
__global__ void __launch_bounds__(256) sumsq_kernel(const float* g, long long n, float* partial) {
  __shared__ float red[8];
  float acc = 0.f;
  const bool vec = (reinterpret_cast<uintptr_t>(g) & 15) == 0;
  const long long n4 = vec ? n >> 2 : 0;
  const float4* g4 = reinterpret_cast<const float4*>(g);
  float a4[4] = {0.f, 0.f, 0.f, 0.f};
  const long long stride = (long long)gridDim.x * 256;
  long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  for (; i + 3 * stride < n4; i += 4 * stride) {
    float4 x[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) x[u] = __ldcs(g4 + i + u * stride);
#pragma unroll
    for (int u = 0; u < 4; ++u) a4[u] = fmaf(x[u].x, x[u].x, fmaf(x[u].y, x[u].y, fmaf(x[u].z, x[u].z, fmaf(x[u].w, x[u].w, a4[u]))));
  }
  for (; i < n4; i += stride) {
    const float4 x = __ldcs(g4 + i);
    a4[0] = fmaf(x.x, x.x, fmaf(x.y, x.y, fmaf(x.z, x.z, fmaf(x.w, x.w, a4[0]))));
  }
  acc = (a4[0] + a4[1]) + (a4[2] + a4[3]);
  for (long long k = (n4 << 2) + (long long)blockIdx.x * 256 + threadIdx.x; k < n; k += stride) acc = fmaf(g[k], g[k], acc);
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int k = 0; k < 8; ++k) s += red[k];
    partial[blockIdx.x] = s;
  }
}
// coef = min(1, max_norm / (sqrt(sumsq) + 1e-6)) * pre_scale;  norm_out = sqrt(sumsq)
__global__ void clip_coef_kernel(const float* sumsq, float max_norm, float pre_scale, float* coef, float* norm_out) {
  const float nrm = sqrtf(*sumsq) * pre_scale;
  float c = max_norm > 0.f ? max_norm / (nrm + 1e-6f) : 1.0f;
  *coef = fminf(c, 1.0f) * pre_scale;
  if (norm_out) *norm_out = nrm;
}
struct AdamParams {
  float* p32;
  float* m;
  float* v;
  const float* g;
  __nv_bfloat16* p16;
  long long n;
  float lr, beta1, beta2, eps, wd, bc1, bc2;
  const float* gscale;   // device scalar (clip coefficient x 1/world), may be null
};
__device__ __forceinline__ float adamw_one(const AdamParams& a, float gs, float g, float& m, float& v, float p) {
  g *= gs;
  m = a.beta1 * m + (1.0f - a.beta1) * g;
  v = a.beta2 * v + (1.0f - a.beta2) * g * g;
  p *= 1.0f - a.lr * a.wd;
  p -= (a.lr / a.bc1) * m / (sqrtf(v) / sqrtf(a.bc2) + a.eps);
  return p;
}
__global__ void __launch_bounds__(256) adamw_kernel(const AdamParams a) {
  const float gs = a.gscale ? *a.gscale : 1.0f;
  const bool vec = ((reinterpret_cast<uintptr_t>(a.g) | reinterpret_cast<uintptr_t>(a.m) | reinterpret_cast<uintptr_t>(a.v) |
                     reinterpret_cast<uintptr_t>(a.p32)) & 15) == 0 && (reinterpret_cast<uintptr_t>(a.p16) & 7) == 0;
  const long long n4 = vec ? a.n >> 2 : 0;
  const long long stride = (long long)gridDim.x * 256;
  for (long long i0 = (long long)blockIdx.x * 256 + threadIdx.x; i0 < n4; i0 += 2 * stride) {
    float4 g[2], m[2], v[2], p[2];
    bool on[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const long long i = i0 + u * stride;
      on[u] = i < n4;
      if (on[u]) {
        g[u] = __ldcs(reinterpret_cast<const float4*>(a.g) + i);      // gradients are dead after this kernel: stream them
        m[u] = reinterpret_cast<const float4*>(a.m)[i];
        v[u] = reinterpret_cast<const float4*>(a.v)[i];
        p[u] = reinterpret_cast<const float4*>(a.p32)[i];
      }
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      if (!on[u]) continue;
      const long long i = i0 + u * stride;
      p[u].x = adamw_one(a, gs, g[u].x, m[u].x, v[u].x, p[u].x);
      p[u].y = adamw_one(a, gs, g[u].y, m[u].y, v[u].y, p[u].y);
      p[u].z = adamw_one(a, gs, g[u].z, m[u].z, v[u].z, p[u].z);
      p[u].w = adamw_one(a, gs, g[u].w, m[u].w, v[u].w, p[u].w);
      reinterpret_cast<float4*>(a.m)[i] = m[u];
      reinterpret_cast<float4*>(a.v)[i] = v[u];
      reinterpret_cast<float4*>(a.p32)[i] = p[u];
      if (a.p16) {
        uint2 o;
        o.x = pack_bf16x2(p[u].x, p[u].y);
        o.y = pack_bf16x2(p[u].z, p[u].w);
        reinterpret_cast<uint2*>(a.p16)[i] = o;
      }
    }
  }
  for (long long i = (n4 << 2) + (long long)blockIdx.x * 256 + threadIdx.x; i < a.n; i += stride) {
    float m = a.m[i], v = a.v[i];
    const float p = adamw_one(a, gs, a.g[i], m, v, a.p32[i]);
    a.m[i] = m;
    a.v[i] = v;
    a.p32[i] = p;
    if (a.p16) a.p16[i] = __float2bfloat16_rn(p);
  }
}
__global__ void __launch_bounds__(256) cast_kernel(const void* src, void* dst, long long n, int to_f32) {
  const bool vec = ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0;
  const long long n8 = vec ? n >> 3 : 0;
  const long long stride = (long long)gridDim.x * 256;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n8; i += stride) {
    if (to_f32) {
      float f[8];
      unpack8(static_cast<const uint4*>(src)[i], f);
      static_cast<float4*>(dst)[2 * i] = make_float4(f[0], f[1], f[2], f[3]);
      static_cast<float4*>(dst)[2 * i + 1] = make_float4(f[4], f[5], f[6], f[7]);
    } else {
      const float4 x = static_cast<const float4*>(src)[2 * i], y = static_cast<const float4*>(src)[2 * i + 1];
      const float f[8] = {x.x, x.y, x.z, x.w, y.x, y.y, y.z, y.w};
      static_cast<uint4*>(dst)[i] = pack8(f);
    }
  }
  for (long long i = (n8 << 3) + (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += stride) {
    if (to_f32)
      static_cast<float*>(dst)[i] = __bfloat162float(static_cast<const __nv_bfloat16*>(src)[i]);
    else
      static_cast<__nv_bfloat16*>(dst)[i] = __float2bfloat16_rn(static_cast<const float*>(src)[i]);
  }
}

// out = bf16( bf16(a * wa) + bf16(b * wb) ): `old * (1 - f) + image_embeds * f` of the reference's
// vlm_residual_image_factor branch (modeling_univa_qwen2p5vl.py:504-506) with torch's bf16 rounding points
__global__ void __launch_bounds__(256) blend_kernel(const __nv_bfloat16* a, const __nv_bfloat16* b, float wa, float wb,
                                                    __nv_bfloat16* out, long long n8) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= n8) return;
  float x[8], y[8];
  unpack8(reinterpret_cast<const uint4*>(a)[i], x);
  unpack8(reinterpret_cast<const uint4*>(b)[i], y);
  // a Python scalar multiplying a bf16 CUDA tensor enters the kernel as an fp32 (opmath) value, NOT rounded to bf16
  // (checked on the GPU against torch's own expression; a 0-dim TENSOR operand, as in the Euler step, is cast to bf16 first)
#pragma unroll
  for (int j = 0; j < 8; ++j) x[j] = bf16r(x[j] * wa) + bf16r(y[j] * wb);
  reinterpret_cast<uint4*>(out)[i] = pack8(x);
}

inline bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

extern "C" int b2f_train_chunks(int rows) { return (rows + CHUNK_ROWS - 1) / CHUNK_ROWS; }
extern "C" int b2f_train_ln_chunks(int rows) { return (rows + CHUNK_LN - 1) / CHUNK_LN; }

extern "C" int b2f_gate_resid_fwd(const void* x, int64_t ldx, int64_t x_bs, const void* y, int64_t ldy, int64_t y_bs,
                                  const void* gate, const void* gate_b, int64_t gate_ld, void* out, int64_t ldo,
                                  int64_t o_bs, int batch, int rows, int D, int split_row, b2f_stream_t stream_) {
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  if (!x || !y || !gate || !out || batch <= 0 || rows <= 0 || D <= 0 || (D & 7)) return B2F_ERR_INVALID;
  if (split_row > 0 && !gate_b) return B2F_ERR_INVALID;
  if ((ldx | x_bs | ldy | y_bs | ldo | o_bs | gate_ld) & 7) return B2F_ERR_ALIGN;
  if (!al16(x) || !al16(y) || !al16(gate) || !al16(gate_b) || !al16(out)) return B2F_ERR_ALIGN;
  GateParams p{};
  p.x = static_cast<const __nv_bfloat16*>(x);
  p.y = static_cast<const __nv_bfloat16*>(y);
  p.gate = static_cast<const __nv_bfloat16*>(gate);
  p.gate_b = static_cast<const __nv_bfloat16*>(gate_b);
  p.out = static_cast<__nv_bfloat16*>(out);
  p.ldx = ldx; p.x_bs = x_bs; p.ldy = ldy; p.y_bs = y_bs; p.ldo = ldo; p.o_bs = o_bs; p.gate_ld = gate_ld;
  p.batch = batch; p.rows = rows; p.D = D; p.split_row = split_row;
  dim3 grid(b2f_train_chunks(rows), (D + 1023) / 1024, batch);
  prof_begin(KC_OTHER, st);
  gate_resid_fwd_kernel<<<grid, 128, 0, st>>>(p);
  prof_end(KC_OTHER, st, 0, 6.0 * batch * rows * D);
  B2F_LAUNCHED("gate_resid_fwd_kernel", 1);
  return B2F_OK;
}

// partial: fp32 scratch of batch * b2f_train_chunks(rows) * D floats (may be null: no column sums)
extern "C" int b2f_gate_bwd(const void* dout, int64_t ldd, int64_t d_bs, const void* y, int64_t ldy, int64_t y_bs,
                            const void* gate, const void* gate_b, int64_t gate_ld, void* dy, int64_t ldo, int64_t o_bs,
                            float* partial, int batch, int rows, int D, int split_row, int part_row0,
                            b2f_stream_t stream_) {
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  if (!dout || batch <= 0 || rows <= 0 || D <= 0 || (D & 7)) return B2F_ERR_INVALID;
  if (dy && !gate) return B2F_ERR_INVALID;
  if (gate && split_row > 0 && !gate_b) return B2F_ERR_INVALID;
  if ((ldd | d_bs | ldy | y_bs | ldo | o_bs | gate_ld) & 7) return B2F_ERR_ALIGN;
  if (!al16(dout) || !al16(y) || !al16(gate) || !al16(gate_b) || !al16(dy) || !al16(partial)) return B2F_ERR_ALIGN;
  GateParams p{};
  p.x = static_cast<const __nv_bfloat16*>(dout);
  p.y = static_cast<const __nv_bfloat16*>(y);
  p.gate = static_cast<const __nv_bfloat16*>(gate);
  p.gate_b = static_cast<const __nv_bfloat16*>(gate_b);
  p.out = static_cast<__nv_bfloat16*>(dy);
  p.partial = partial;
  p.ldx = ldd; p.x_bs = d_bs; p.ldy = ldy; p.y_bs = y_bs; p.ldo = ldo; p.o_bs = o_bs; p.gate_ld = gate_ld;
  p.batch = batch; p.rows = rows; p.D = D; p.split_row = split_row; p.part_row0 = part_row0;
  dim3 grid(b2f_train_chunks(rows), (D + 1023) / 1024, batch);
  prof_begin(KC_OTHER, st);
  gate_bwd_kernel<<<grid, 128, 0, st>>>(p);
  prof_end(KC_OTHER, st, 0, (2.0 + (y ? 2.0 : 0.0) + (dy ? 2.0 : 0.0)) * batch * rows * D);
  B2F_LAUNCHED("gate_bwd_kernel", 1);
  return B2F_OK;
}

extern "C" int b2f_col_reduce(const float* partial, int nchunks, int D, float* out, int64_t out_ld, int batch,
                              int accumulate, b2f_stream_t stream_) {
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  if (!partial || !out || nchunks <= 0 || D <= 0 || batch <= 0) return B2F_ERR_INVALID;
  dim3 grid((D + 255) / 256, batch);
  col_reduce_kernel<<<grid, 256, 0, st>>>(partial, nchunks, D, out, out_ld, accumulate);
  B2F_LAUNCHED("col_reduce_kernel", 1);
  return B2F_OK;
}

// partial: batch * b2f_train_ln_chunks(rows) * 2 * D floats (dscale | dshift per chunk), or null
extern "C" int b2f_ln_modulate_bwd(const void* x, int64_t ldx, int64_t x_bs, const void* dy, int64_t ldy, int64_t dy_bs,
                                   const void* scale, const void* scale_b, int64_t mod_ld, const void* dres_in,
                                   int64_t ldr, int64_t r_bs, void* dres_out, int64_t ldo, int64_t o_bs, float* partial,
                                   int batch, int rows, int D, float eps, int split_row, int part_row0,
                                   b2f_stream_t stream_) {
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  if (!x || !dy || !scale || !dres_out || batch <= 0 || rows <= 0 || D <= 0 || (D & 7)) return B2F_ERR_INVALID;
  if (split_row > 0 && !scale_b) return B2F_ERR_INVALID;
  if ((ldx | x_bs | ldy | dy_bs | ldr | r_bs | ldo | o_bs | mod_ld) & 7) return B2F_ERR_ALIGN;
  if (!al16(x) || !al16(dy) || !al16(scale) || !al16(scale_b) || !al16(dres_in) || !al16(dres_out) || !al16(partial))
    return B2F_ERR_ALIGN;
  LnBwdParams p{};
  p.x = static_cast<const __nv_bfloat16*>(x);
  p.dy = static_cast<const __nv_bfloat16*>(dy);
  p.scale = static_cast<const __nv_bfloat16*>(scale);
  p.scale_b = static_cast<const __nv_bfloat16*>(scale_b);
  p.dres_in = static_cast<const __nv_bfloat16*>(dres_in);
  p.dres_out = static_cast<__nv_bfloat16*>(dres_out);
  p.partial = partial;
  p.ldx = ldx; p.x_bs = x_bs; p.ldy = ldy; p.dy_bs = dy_bs; p.ldr = ldr; p.r_bs = r_bs; p.ldo = ldo; p.o_bs = o_bs;
  p.mod_ld = mod_ld;
  p.batch = batch; p.rows = rows; p.D = D; p.split_row = split_row; p.part_row0 = part_row0; p.eps = eps;
  dim3 grid(b2f_train_ln_chunks(rows), batch);
  prof_begin(KC_LNMOD, st);
  ln_modulate_bwd_kernel<<<grid, 256, 0, st>>>(p);
  prof_end(KC_LNMOD, st, 0, (dres_in ? 8.0 : 6.0) * batch * rows * D);
  B2F_LAUNCHED("ln_modulate_bwd_kernel", 1);
  return B2F_OK;
}

// partial: ((batch*S + 7) / 8) * 512 floats, or null.  dq/dk are updated in place.
extern "C" int b2f_rmsnorm_rope_bwd(void* dq, void* dk, int64_t ld, int64_t bs, const void* xq, const void* xk,
                                    int64_t ldx, int64_t x_bs, const void* wq_a, const void* wk_a, const void* wq_b,
                                    const void* wk_b, const float* cos, const float* sin, float* partial, int batch,
                                    int S, int H, int n_a, float eps, b2f_stream_t stream_) {
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  if (!dq || !dk || !xq || !xk || !wq_b || !wk_b || !cos || !sin || batch <= 0 || S <= 0 || H <= 0) return B2F_ERR_INVALID;
  if (n_a > 0 && (!wq_a || !wk_a)) return B2F_ERR_INVALID;
  if ((ld | bs | ldx | x_bs) & 7) return B2F_ERR_ALIGN;
  NormRopeBwdParams p{};
  p.dq = static_cast<__nv_bfloat16*>(dq);
  p.dk = static_cast<__nv_bfloat16*>(dk);
  p.xq = static_cast<const __nv_bfloat16*>(xq);
  p.xk = static_cast<const __nv_bfloat16*>(xk);
  p.ld = ld; p.batch_stride = bs; p.ldx = ldx; p.x_batch_stride = x_bs;
  p.wq_a = static_cast<const __nv_bfloat16*>(n_a > 0 ? wq_a : wq_b);
  p.wk_a = static_cast<const __nv_bfloat16*>(n_a > 0 ? wk_a : wk_b);
  p.wq_b = static_cast<const __nv_bfloat16*>(wq_b);
  p.wk_b = static_cast<const __nv_bfloat16*>(wk_b);
  p.cos = cos; p.sin = sin; p.partial = partial; p.batch = batch; p.S = S; p.H = H; p.n_a = n_a; p.eps = eps;
  const long long tokens = (long long)batch * S;
  prof_begin(KC_NORMROPE, st);
  rmsnorm_rope_bwd_kernel<<<(unsigned)((tokens + 7) / 8), 256, 0, st>>>(p);
  prof_end(KC_NORMROPE, st, 0, 12.0 * tokens * H * 128);
  B2F_LAUNCHED("rmsnorm_rope_bwd_kernel", 1);
  return B2F_OK;
}

extern "C" int b2f_gelu_rows(const void* x, int64_t ldx, void* y, int64_t ldy, int64_t rows, int D,
                             b2f_stream_t stream_) {
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  if (!x || !y || rows <= 0 || D <= 0 || (D & 7) || (ldx & 7) || (ldy & 7)) return B2F_ERR_INVALID;
  const long long n = rows * (D / 8);
  prof_begin(KC_OTHER, st);
  gelu_rows_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(static_cast<const __nv_bfloat16*>(x), ldx,
                                                               static_cast<__nv_bfloat16*>(y), ldy, rows, D);
  prof_end(KC_OTHER, st, 0, 4.0 * rows * D);
  B2F_LAUNCHED("gelu_rows_kernel", 1);
  return B2F_OK;
}

extern "C" int b2f_outer_acc(const float* dmod, int64_t dmod_ld, const void* act, int64_t act_ld, float* dW,
                             int64_t ldw, int B, int N, int K, int accumulate, b2f_stream_t stream_) {
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  if (!dmod || !act || !dW || B <= 0 || N <= 0 || K <= 0 || (K & 3) || (ldw & 3) || (act_ld & 3)) return B2F_ERR_INVALID;
  dim3 grid((K / 4 + 255) / 256, N);
  prof_begin(KC_OTHER, st);
  outer_acc_kernel<<<grid, 256, 0, st>>>(dmod, dmod_ld, static_cast<const __nv_bfloat16*>(act), act_ld, dW, ldw, B, N, K,
                                        accumulate);
  prof_end(KC_OTHER, st, 0, (accumulate ? 8.0 : 4.0) * N * K);
  B2F_LAUNCHED("outer_acc_kernel", 1);
  return B2F_OK;
}

extern "C" int b2f_attn_delta(const void* o, int64_t ldo, const void* dout, int64_t lddo, float* delta, float* lse,
                              int B, int H, int S, int S_pad, b2f_stream_t stream_) {
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  if (!o || !dout || !delta || !lse || B <= 0 || H <= 0 || S <= 0 || S_pad < S || (ldo & 7) || (lddo & 7)) return B2F_ERR_INVALID;
  const long long threads = (long long)B * H * S_pad * 16;
  prof_begin(KC_OTHER, st);
  attn_delta_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(static_cast<const __nv_bfloat16*>(o), ldo,
                                                                      static_cast<const __nv_bfloat16*>(dout), lddo, delta,
                                                                      lse, B, H, S, S_pad);
  prof_end(KC_OTHER, st, 0, 4.0 * B * H * S * 128);
  B2F_LAUNCHED("attn_delta_kernel", 1);
  return B2F_OK;
}

// loss_out: device scalar; ws: >= 1024 floats of scratch
extern "C" int b2f_mse_loss(const void* pred, const float* target, const float* w, void* dpred, float* loss_out,
                            float* ws, int64_t n, float grad_scale, b2f_stream_t stream_) {
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  if (!pred || !target || !loss_out || !ws || n <= 0) return B2F_ERR_INVALID;
  const int blocks = int(n / 256 < 1 ? 1 : (n / 256 > 1024 ? 1024 : n / 256));
  mse_loss_kernel<<<blocks, 256, 0, st>>>(static_cast<const __nv_bfloat16*>(pred), target, w,
                                          static_cast<__nv_bfloat16*>(dpred), ws, n, grad_scale / float(n),
                                          1.0f / float(n));
  B2F_LAUNCHED("mse_loss_kernel", 1);
  // loss = sum of the per-block partial means
  col_reduce_kernel<<<dim3(1, 1), 256, 0, st>>>(ws, blocks, 1, loss_out, 1, 0);
  B2F_LAUNCHED("col_reduce_kernel", 1);
  return B2F_OK;
}

// sumsq_out (+)= sum(g^2);  ws: >= 1024 floats
extern "C" int b2f_grad_sumsq(const float* g, int64_t n, float* sumsq_out, float* ws, int accumulate,
                              b2f_stream_t stream_) {
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  if (!g || !sumsq_out || !ws || n <= 0) return B2F_ERR_INVALID;
  const int blocks = int(n / 1024 < 1 ? 1 : (n / 1024 > 1024 ? 1024 : n / 1024));
  sumsq_kernel<<<blocks, 256, 0, st>>>(g, n, ws);
  B2F_LAUNCHED("sumsq_kernel", 1);
  col_reduce_kernel<<<dim3(1, 1), 256, 0, st>>>(ws, blocks, 1, sumsq_out, 1, accumulate);
  B2F_LAUNCHED("col_reduce_kernel", 1);
  return B2F_OK;
}

extern "C" int b2f_clip_coef(const float* sumsq, float max_norm, float pre_scale, float* coef, float* norm_out,
                             b2f_stream_t stream_) {
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  if (!sumsq || !coef) return B2F_ERR_INVALID;
  clip_coef_kernel<<<1, 1, 0, st>>>(sumsq, max_norm, pre_scale, coef, norm_out);
  B2F_LAUNCHED("clip_coef_kernel", 1);
  return B2F_OK;
}

extern "C" int b2f_adamw_step(float* p32, float* m, float* v, const float* g, void* p16, int64_t n, float lr,
                              float beta1, float beta2, float eps, float wd, int step, const float* gscale,
                              b2f_stream_t stream_) {
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  if (!p32 || !m || !v || !g || n <= 0 || step <= 0) return B2F_ERR_INVALID;
  AdamParams a{};
  a.p32 = p32; a.m = m; a.v = v; a.g = g; a.p16 = static_cast<__nv_bfloat16*>(p16); a.n = n;
  a.lr = lr; a.beta1 = beta1; a.beta2 = beta2; a.eps = eps; a.wd = wd;
  a.bc1 = 1.0f - powf(beta1, (float)step);
  a.bc2 = 1.0f - powf(beta2, (float)step);
  a.gscale = gscale;
  const long long blocks = (n + 255) / 256;
  prof_begin(KC_OTHER, st);
  adamw_kernel<<<(unsigned)(blocks > 148 * 16 ? 148 * 16 : blocks), 256, 0, st>>>(a);
  prof_end(KC_OTHER, st, 0, 30.0 * n);
  B2F_LAUNCHED("adamw_kernel", 1);
  return B2F_OK;
}

extern "C" int b2f_blend_bf16(const void* a, const void* b, float wa, float wb, void* out, int64_t n,
                              b2f_stream_t stream_) {
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  if (!a || !b || !out || n <= 0 || (n & 7)) return B2F_ERR_INVALID;
  if (!al16(a) || !al16(b) || !al16(out)) return B2F_ERR_ALIGN;
  blend_kernel<<<(unsigned)((n / 8 + 255) / 256), 256, 0, st>>>(static_cast<const __nv_bfloat16*>(a),
                                                             static_cast<const __nv_bfloat16*>(b), wa, wb,
                                                             static_cast<__nv_bfloat16*>(out), n / 8);
  B2F_LAUNCHED("blend_kernel", 1);
  return B2F_OK;
}

extern "C" int b2f_cast_bf16_f32(const void* src, void* dst, int64_t n, int to_f32, b2f_stream_t stream_) {
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  if (!src || !dst || n <= 0) return B2F_ERR_INVALID;
  const long long blocks = (n + 255) / 256;
  cast_kernel<<<(unsigned)(blocks > 148 * 16 ? 148 * 16 : blocks), 256, 0, st>>>(src, dst, n, to_f32);
  B2F_LAUNCHED("cast_kernel", 1);
  return B2F_OK;
}

}  // namespace b2f
