// Host-side helpers shared by the launchers: error codes, launch counting, TMA tensor-map encoding through
// the driver entry point (no -lcuda link, so the library loads on a box without a driver).  Every launcher
// is itself the extern "C" b2f_* entry point that include/b2f.h declares.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <atomic>
#include <cstdint>
#include <cstdio>

#include "../../include/b2f.h"

namespace b2f {

struct DeviceInfo {
  int num_sms = 0;
  int max_smem_optin = 0;
  bool ok = false;
};
const DeviceInfo& device_info();

// 2-D bf16 tensor map: global [rows, cols] with row pitch ld_elems, box [box_rows, box_cols],
// SWIZZLE_128B (box_cols * 2 bytes must be 128).
int make_tmap_2d_bf16(CUtensorMap* out, const void* gptr, uint64_t rows, uint64_t cols,
                      uint64_t ld_elems, uint32_t box_rows, uint32_t box_cols);
// 3-D bf16 tensor map over [batch, rows, width] with box [1, 128, 64] (attention Q/K/V tiles):
// out-of-range rows are zero-filled per batch item.
int make_tmap_3d_rows(CUtensorMap* out, const void* gptr, uint64_t width, uint64_t rows,
                      uint64_t batch, uint64_t ld_elems, uint64_t batch_stride_elems, uint32_t box_rows = 128);
// Byte-element (e4m3) tensor map over [rows, width] (rank 2) or [batch, rows, width] (rank 3), pitches in bytes, box
// [1,] 128 rows x 128 bytes, SWIZZLE_128B: the same shared-memory layout as a [128][64] bf16 box.
int make_tmap_u8_rows(CUtensorMap* out, const void* gptr, int rank, uint64_t width, uint64_t rows, uint64_t batch,
                      uint64_t ld_bytes, uint64_t batch_stride_bytes);
// 4-D bf16 tensor map for NHWC activations: global [n, h, w, c], box [1, box_h, box_w, box_c].
// `stride` (1 or 2) is the traversal stride in h and w: the box still delivers box_h x box_w pixels.
int make_tmap_4d_bf16(CUtensorMap* out, const void* gptr, uint64_t n, uint64_t h, uint64_t w,
                      uint64_t c, uint32_t box_h, uint32_t box_w, uint32_t box_c, uint32_t stride);

// Optional per-kernel-class timing with CUDA events on the launching stream (bench.py's roofline
// figures).  Disabled by default: zero overhead on the normal path.
enum KernelClass { KC_GEMM = 0, KC_ATTN = 1, KC_LNMOD = 2, KC_NORMROPE = 3, KC_CONV = 4, KC_OTHER = 5, KC_COUNT = 6 };
bool prof_enabled();
void prof_begin(int kc, cudaStream_t s);
void prof_end(int kc, cudaStream_t s, double flops, double bytes);
// the same, additionally filed under a shape tag ("gemm2 8736x3072x15360 e3"): b2f_prof_shapes() lists the per-shape sums
void prof_end_tagged(int kc, cudaStream_t s, double flops, double bytes, const char* tag);

inline int cuda_err(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return B2F_OK;
  fprintf(stderr, "[b2f] CUDA error in %s: %s\n", what, cudaGetErrorString(e));
  return B2F_ERR_CUDA;
}

// Raises the dynamic shared-memory limit of every kernel in `kernels` to `bytes`, once: `done` is set only when every
// call succeeded, so a launcher whose call failed tries again on its next launch.
template <class... Kernels>
int set_max_smem_once(bool& done, int bytes, const char* what, Kernels*... kernels) {
  if (done) return B2F_OK;
  for (const void* k : {reinterpret_cast<const void*>(kernels)...}) {
    const cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) return cuda_err(e, what);
  }
  done = true;
  return B2F_OK;
}

// Workspace carving: sizes and pointers rounded up to 256 bytes (a null pointer stays null).
inline size_t al256(size_t n) { return (n + 255) & ~size_t(255); }
template <class T = uint8_t>
inline T* al256(void* p) {
  return reinterpret_cast<T*>(al256(reinterpret_cast<uintptr_t>(p)));
}

// Kernels launched since load (b2f_launch_count).
extern std::atomic<uint64_t> g_launch_count;

// After enqueueing n kernels: count them, and return B2F_ERR_CUDA from the launcher if a launch failed.
#define B2F_LAUNCHED(name, n)                                           \
  do {                                                                  \
    b2f::g_launch_count.fetch_add((n), std::memory_order_relaxed);      \
    cudaError_t _e = cudaGetLastError();                                \
    if (_e != cudaSuccess) return b2f::cuda_err(_e, name);              \
  } while (0)

}  // namespace b2f
