// LoRA weight merge: W <- bf16(W + sum_k fp32(Bcat[:, k] * s_k) Acat[k, :]),  s_k = fp32(colscale[k] * cs_mul).
//
// One fp32 accumulation per element in ascending k (fmaf), then one rounding of W + acc.  This is what
// diffusers' fuse_lora computes (PEFT LoraLayer.merge: W += scaling * B @ A) up to where it rounds: PEFT forms the
// delta in the weight dtype, here it stays fp32 until the single final rounding.  64 x 64 output tiles, 4 x 4 per
// thread, k in chunks of 32 through shared memory.  A one-off at fuse time, so it is written for clarity.
//
// Replaces: peft.tuners.lora.layer.Linear.merge as reached by diffusers FluxLoraLoaderMixin.fuse_lora
// (reference univa/utils/flux_pipeline.py:30 inherits it).
#include <cuda_bf16.h>

#include "host_common.h"

namespace b2f {

namespace {

constexpr int FT = 64, FK = 32;

__global__ void __launch_bounds__(256) lora_fuse_kernel(uint16_t* W, int64_t ldw, int rows, int cols, const uint16_t* Bc,
                                                        int64_t ldb, const uint16_t* A, int64_t lda, const float* cs,
                                                        float cs_mul, int r) {
  __shared__ float sb[FT][FK + 1];   // scaled B: rows of this tile x k
  __shared__ float sa[FK][FT + 1];   // A: k x columns of this tile
  const int r0 = blockIdx.y * FT, c0 = blockIdx.x * FT;
  const int tr = threadIdx.x / 16, tc = threadIdx.x % 16;   // thread owns rows tr + 16 i, columns tc + 16 j
  float acc[4][4] = {};
  auto bf = [](uint16_t u) { return __uint_as_float((uint32_t)u << 16); };
  for (int k0 = 0; k0 < r; k0 += FK) {
    for (int e = threadIdx.x; e < FT * FK; e += 256) {
      const int i = e / FK, k = e % FK;
      const int row = r0 + i, kk = k0 + k;
      sb[i][k] = (row < rows && kk < r) ? bf(Bc[(int64_t)row * ldb + kk]) * (cs[kk] * cs_mul) : 0.f;
      const int kr = e / FT, j = e % FT;
      const int col = c0 + j, ka = k0 + kr;
      sa[kr][j] = (col < cols && ka < r) ? bf(A[(int64_t)ka * lda + col]) : 0.f;
    }
    __syncthreads();
#pragma unroll 4
    for (int k = 0; k < FK; ++k) {
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(sb[tr + 16 * i][k], sa[k][tc + 16 * j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int row = r0 + tr + 16 * i;
    if (row >= rows) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int col = c0 + tc + 16 * j;
      if (col >= cols) continue;
      uint16_t* w = W + (int64_t)row * ldw + col;
      const __nv_bfloat16 o = __float2bfloat16_rn(bf(*w) + acc[i][j]);
      *w = *reinterpret_cast<const uint16_t*>(&o);
    }
  }
}

}  // namespace

extern "C" int b2f_lora_fuse(void* W, int64_t ldw, int rows, int cols, const void* Bc, int64_t ldb, const void* A,
                             int64_t lda, const float* colscale, float cs_mul, int r, b2f_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!device_info().ok) return B2F_ERR_NODEVICE;
  if (!W || !Bc || !A || !colscale || rows <= 0 || cols <= 0 || r <= 0 || ldw < cols || lda < cols || ldb < r)
    return B2F_ERR_INVALID;
  const dim3 grid((cols + FT - 1) / FT, (rows + FT - 1) / FT);
  if (grid.y > 65535) return B2F_ERR_UNSUPPORTED;
  lora_fuse_kernel<<<grid, 256, 0, stream>>>(static_cast<uint16_t*>(W), ldw, rows, cols,
                                             static_cast<const uint16_t*>(Bc), ldb, static_cast<const uint16_t*>(A),
                                             lda, colscale, cs_mul, r);
  B2F_LAUNCHED("lora_fuse_kernel", 1);
  return B2F_OK;
}

}  // namespace b2f
