// 3x3 convolution as an implicit GEMM on wgmma (sm_90a), NHWC bf16, fp32 accumulation in registers.
//
//   out[n, y, x, co] = bias[co] + sum_{ky,kx,ci} in[n, y*s + ky - p, x*s + kx - p, ci] * w[co, ky, kx, ci]
//
// GEMM view: M = output pixels (one CTA tile = an 8 x 16 spatial patch = 128 rows), N = Cout,
// K = 9 * Cin walked as (tap, 64-channel chunk).  The A tile of every k-step is ONE 4-D TMA box
// {64 ch, 16 x, 8 y, 1 n} of the NHWC input, shifted by the tap offset: the conv halo and the zero
// padding come from TMA's out-of-bounds zero fill, no im2col buffer and no halo staging code.
// The stride-2 downsample (diffusers Downsample2D: pad right/bottom by 1, stride 2, no other padding)
// uses a second tensor map whose traversal stride is 2 in x and y.
// Weights are OHWI ([Cout, 3, 3, Cin] = K-major [Cout, 9*Cin]).  Warp roles, smem ring and the staged
// epilogue are those of gemm.cu (gemm_sm90.cuh).
//
// Replaces cuDNN conv as reached by diffusers AutoencoderKL (ResnetBlock2D conv1/conv2, Downsample2D,
// Upsample2D conv, conv_in/conv_out; SURVEY.md A.4; reference call sites
// univa/utils/flux_pipeline.py:600-613, 1127-1129).
#include "gemm_sm90.cuh"

namespace b2f {

namespace {

using namespace sm90;

constexpr int TILE_H = 8, TILE_W = 16;   // TILE_H * TILE_W = BLOCK_M

struct ConvParams {
  int N, Ho, Wo, Cin, Cout, stride;
  const __nv_bfloat16* bias;
  __nv_bfloat16* out;
  const __nv_bfloat16* resid;  // same layout as out (NHWC), may be null
  int out_nchw;                // 1: write out[n, co, y, x] for co < Cout (small Cout heads)
                               // 2: uint8 NHWC image out[n, y, x, co] = round(clamp(bf16(conv)/2 + 0.5, 0, 1) * 255):
                               //    VaeImageProcessor.postprocess fused into decoder.conv_out (reference flux_pipeline.py:1130)
  int tiles_y, tiles_x, num_m_blocks, num_n_blocks;
};

__global__ void __launch_bounds__(THREADS, 1)
conv3x3_kernel(const __grid_constant__ CUtensorMap tmIn, const __grid_constant__ CUtensorMap tmW,
               const ConvParams p) {
  extern __shared__ uint8_t smem_raw[];
  const Smem s = carve(smem_raw);
  const int wg = threadIdx.x >> 7;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmIn);
    tma_prefetch_desc(&tmW);
  }
  init_barriers(s);

  const int cchunks = p.Cin / BLOCK_K;
  const int num_kb = 9 * cchunks;
  const int tiles_per_img = p.tiles_y * p.tiles_x;
  // n-block fastest: neighbouring CTAs share the same input patch rows through L2
  const int t = blockIdx.x;
  const int n_blk = t % p.num_n_blocks;
  const int m = t / p.num_n_blocks;
  const int n_img = m / tiles_per_img;
  const int r = m - n_img * tiles_per_img;
  const int y0 = (r / p.tiles_x) * TILE_H;
  const int x0 = (r % p.tiles_x) * TILE_W;

  if (wg == 0) {
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      const int pad = p.stride == 1 ? 1 : 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        const int tap = kb / cchunks;
        const int c0 = (kb - tap * cchunks) * BLOCK_K;
        const int ky = tap / 3, kx = tap - ky * 3;
        mbar_wait(&s.empty[stage], phase ^ 1);
        uint8_t* sa = s.ring + stage * STAGE_BYTES;
        uint8_t* sb = sa + A_BYTES;
        mbar_expect_tx(&s.full[stage], STAGE_BYTES);
        tma_load_4d(sa, &tmIn, &s.full[stage], c0, x0 * p.stride + kx - pad, y0 * p.stride + ky - pad, n_img);
        tma_load_2d(sb, &tmW, &s.full[stage], tap * p.Cin + c0, n_blk * BLOCK_N);
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
    return;
  }
  float acc[64];
  mainloop<0, 0>(s, num_kb, wg - 1, acc);
  stage_accumulators(s, wg - 1, acc);

  const int e = threadIdx.x - 128;
  const int row_in_tile = e & (BLOCK_M - 1), half = e >> 7;
  const int yl = row_in_tile / TILE_W, xl = row_in_tile % TILE_W;
  const int y = y0 + yl, x = x0 + xl;
  if (y >= p.Ho || x >= p.Wo) return;
  const long long pix = ((long long)n_img * p.Ho + y) * p.Wo + x;
  __nv_bfloat16* out_row = p.out + pix * p.Cout;
  const __nv_bfloat16* res_row = p.resid ? p.resid + pix * p.Cout : nullptr;
  const float* crow = s.cbuf + row_in_tile * CROW;
#pragma unroll 1
  for (int c0 = half * (BLOCK_N / 2); c0 < (half + 1) * (BLOCK_N / 2); c0 += 32) {
    const int n0 = n_blk * BLOCK_N + c0;
    if (n0 >= p.Cout) break;
    uint32_t acc32[32];
    load_chunk(crow, c0, acc32);
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const int n = n0 + g * 8;
      if (n >= p.Cout) break;
      float v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = __uint_as_float(acc32[g * 8 + j]);
      if (p.bias) {
        const uint4 bq = __ldg(reinterpret_cast<const uint4*>(p.bias + n));
        const uint32_t bw[4] = {bq.x, bq.y, bq.z, bq.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 b2 = unpack_bf16x2(bw[j]);
          v[2 * j] += b2.x;
          v[2 * j + 1] += b2.y;
        }
      }
      if (p.out_nchw == 2) {
        uint8_t* o8 = reinterpret_cast<uint8_t*>(p.out) + pix * p.Cout;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int co = n + j;
          if (co < p.Cout) {
            const float img = bf16r(v[j]);                                   // the bf16 image the decoder returns
            const float u = fminf(fmaxf(img / 2.0f + 0.5f, 0.0f), 1.0f);     // denormalise + clamp in fp32
            o8[co] = (uint8_t)rintf(u * 255.0f);                             // numpy round (half to even)
          }
        }
        continue;
      }
      if (p.out_nchw) {
        // small heads (Cout <= 32): planar output, one scalar per (pixel, channel)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int co = n + j;
          if (co < p.Cout)
            p.out[(((long long)n_img * p.Cout + co) * p.Ho + y) * p.Wo + x] = __float2bfloat16_rn(v[j]);
        }
        continue;
      }
      if (res_row) {
        const uint4 rq = *reinterpret_cast<const uint4*>(res_row + n);
        const uint32_t rw[4] = {rq.x, rq.y, rq.z, rq.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 r2 = unpack_bf16x2(rw[j]);
          v[2 * j] = r2.x + bf16r(v[2 * j]);
          v[2 * j + 1] = r2.y + bf16r(v[2 * j + 1]);
        }
      }
      uint4 o;
      o.x = pack_bf16x2(v[0], v[1]);
      o.y = pack_bf16x2(v[2], v[3]);
      o.z = pack_bf16x2(v[4], v[5]);
      o.w = pack_bf16x2(v[6], v[7]);
      *reinterpret_cast<uint4*>(out_row + n) = o;
    }
  }
}

int launch_conv(const CUtensorMap& tmIn, const CUtensorMap& tmW, ConvParams p, cudaStream_t stream) {
  static bool attr_set = false;
  if (int rc = set_max_smem_once(attr_set, SMEM_BYTES, "conv smem attribute", conv3x3_kernel)) return rc;
  p.num_n_blocks = (p.Cout + BLOCK_N - 1) / BLOCK_N;
  const int num_tiles = p.num_m_blocks * p.num_n_blocks;
  prof_begin(KC_CONV, stream);
  conv3x3_kernel<<<num_tiles, THREADS, SMEM_BYTES, stream>>>(tmIn, tmW, p);
  const double pix = (double)p.N * p.Ho * p.Wo;
  prof_end(KC_CONV, stream, 2.0 * pix * 9.0 * p.Cin * p.Cout,
           2.0 * (pix * p.stride * p.stride * p.Cin + pix * p.Cout + 9.0 * p.Cin * p.Cout));
  B2F_LAUNCHED("conv3x3_kernel", 1);
  return B2F_OK;
}

}  // namespace

extern "C" int b2f_conv3x3(const void* in, const void* w, const void* bias, void* out, const void* resid, int N,
                           int Hin, int Win, int Cin, int Cout, int stride, int out_nchw, b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (!in || !w || !out || N <= 0 || Hin <= 0 || Win <= 0) return B2F_ERR_INVALID;
  if (Cin % 64 || Cout <= 0 || (stride != 1 && stride != 2)) return B2F_ERR_UNSUPPORTED;
  if (!out_nchw && (Cout & 7)) return B2F_ERR_UNSUPPORTED;
  if (out_nchw && resid) return B2F_ERR_UNSUPPORTED;
  if (out_nchw < 0 || out_nchw > 2) return B2F_ERR_INVALID;
  if ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(w) | reinterpret_cast<uintptr_t>(bias) |
       reinterpret_cast<uintptr_t>(resid)) & 15)
    return B2F_ERR_ALIGN;
  if (out_nchw != 2 && (reinterpret_cast<uintptr_t>(out) & 15)) return B2F_ERR_ALIGN;
  ConvParams p{};
  p.N = N;
  p.stride = stride;
  // stride 2 follows Downsample2D: pad (0,1,0,1) then a valid 3x3/2 conv -> floor((H+1-3)/2)+1 = H/2
  p.Ho = stride == 1 ? Hin : (Hin + 1 - 3) / 2 + 1;
  p.Wo = stride == 1 ? Win : (Win + 1 - 3) / 2 + 1;
  p.Cin = Cin;
  p.Cout = Cout;
  p.bias = static_cast<const __nv_bfloat16*>(bias);
  p.out = static_cast<__nv_bfloat16*>(out);
  p.resid = static_cast<const __nv_bfloat16*>(resid);
  p.out_nchw = out_nchw;
  p.tiles_y = (p.Ho + TILE_H - 1) / TILE_H;
  p.tiles_x = (p.Wo + TILE_W - 1) / TILE_W;
  p.num_m_blocks = N * p.tiles_y * p.tiles_x;
  CUtensorMap tmIn, tmW;
  int rc = make_tmap_4d_bf16(&tmIn, in, N, Hin, Win, Cin, TILE_H, TILE_W, BLOCK_K, stride);
  if (rc) return rc;
  // weights padded by the caller to a multiple of 8 rows when Cout is tiny; OOB rows read as zero
  rc = make_tmap_2d_bf16(&tmW, w, (uint64_t)Cout, (uint64_t)9 * Cin, (uint64_t)9 * Cin,
                         BLOCK_N, BLOCK_K);
  if (rc) return rc;
  return launch_conv(tmIn, tmW, p, stream);
}

}  // namespace b2f
