// Library-wide entry points (error strings, version, device facts, launch count, profiler) and TMA
// tensor-map encoding (driver entry point fetched at run time).
#include "host_common.h"

#include <cstring>

#include <atomic>
#include <map>
#include <mutex>
#include <string>
#include <vector>

namespace b2f {

std::atomic<uint64_t> g_launch_count{0};

extern "C" uint64_t b2f_launch_count(void) { return g_launch_count.load(); }

extern "C" const char* b2f_strerror(int code) {
  switch (code) {
    case B2F_OK: return "ok";
    case B2F_ERR_INVALID: return "invalid argument or shape";
    case B2F_ERR_CUDA: return "CUDA error (see stderr)";
    case B2F_ERR_UNSUPPORTED: return "unsupported shape or mode";
    case B2F_ERR_ALIGN: return "pointer or pitch not 16-byte aligned";
    case B2F_ERR_NODEVICE: return "no sm_90 device";
    case B2F_ERR_WORKSPACE: return "workspace too small";
    default: return "unknown error";
  }
}

extern "C" int b2f_version(void) { return 5; }

extern "C" int b2f_device_info(int* num_sms, int* cc_major, int* cc_minor, size_t* smem_optin) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
    cudaGetLastError();
    return B2F_ERR_NODEVICE;
  }
  int dev = 0, v = 0;
  cudaGetDevice(&dev);
  if (num_sms) cudaDeviceGetAttribute(num_sms, cudaDevAttrMultiProcessorCount, dev);
  if (cc_major) cudaDeviceGetAttribute(cc_major, cudaDevAttrComputeCapabilityMajor, dev);
  if (cc_minor) cudaDeviceGetAttribute(cc_minor, cudaDevAttrComputeCapabilityMinor, dev);
  if (smem_optin) {
    cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    *smem_optin = (size_t)v;
  }
  return B2F_OK;
}

const DeviceInfo& device_info() {
  static DeviceInfo info;
  static std::once_flag once;
  std::call_once(once, [] {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
      cudaGetLastError();
      return;
    }
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return;
    int major = 0;
    cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
    cudaDeviceGetAttribute(&info.num_sms, cudaDevAttrMultiProcessorCount, dev);
    cudaDeviceGetAttribute(&info.max_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    info.ok = (major == 9) && info.num_sms > 0;
  });
  return info;
}

// ------------------------------------------------------------------ event profiler
namespace {
struct ProfState {
  bool enabled = false;
  std::mutex mu;
  std::vector<cudaEvent_t> pool;
  struct Rec { cudaEvent_t a, b; };
  std::vector<Rec> recs[KC_COUNT];
  double flops[KC_COUNT] = {0}, bytes[KC_COUNT] = {0};
  cudaEvent_t pending[KC_COUNT] = {nullptr};
  struct Shape { std::vector<Rec> recs; double flops = 0; };
  std::map<std::string, Shape> shapes;
  cudaEvent_t get() {
    if (!pool.empty()) {
      cudaEvent_t e = pool.back();
      pool.pop_back();
      return e;
    }
    cudaEvent_t e;
    cudaEventCreate(&e);
    return e;
  }
};
ProfState g_prof;
}  // namespace

bool prof_enabled() { return g_prof.enabled; }
void prof_begin(int kc, cudaStream_t s) {
  if (!g_prof.enabled) return;
  std::lock_guard<std::mutex> lk(g_prof.mu);
  cudaEvent_t e = g_prof.get();
  cudaEventRecord(e, s);
  g_prof.pending[kc] = e;
}
void prof_end(int kc, cudaStream_t s, double flops, double bytes) {
  if (!g_prof.enabled) return;
  std::lock_guard<std::mutex> lk(g_prof.mu);
  cudaEvent_t e = g_prof.get();
  cudaEventRecord(e, s);
  g_prof.recs[kc].push_back({g_prof.pending[kc], e});
  g_prof.flops[kc] += flops;
  g_prof.bytes[kc] += bytes;
}
void prof_end_tagged(int kc, cudaStream_t s, double flops, double bytes, const char* tag) {
  if (!g_prof.enabled) return;
  prof_end(kc, s, flops, bytes);
  std::lock_guard<std::mutex> lk(g_prof.mu);
  auto& sh = g_prof.shapes[tag];
  sh.recs.push_back(g_prof.recs[kc].back());     // the event pair is shared with the class list (freed there)
  sh.flops += flops;
}
extern "C" void b2f_prof_enable(int on) { g_prof.enabled = on != 0; }
// "tag\tlaunches\tms\tTFLOP/s\n" per shape since the last call; call BEFORE b2f_prof_collect (which recycles the events)
extern "C" int b2f_prof_shapes(char* buf, int cap) {
  std::lock_guard<std::mutex> lk(g_prof.mu);
  std::string out;
  for (auto& kv : g_prof.shapes) {
    double ms = 0;
    for (auto& r : kv.second.recs) {
      if (cudaEventSynchronize(r.b) != cudaSuccess) return B2F_ERR_CUDA;
      float t = 0;
      cudaEventElapsedTime(&t, r.a, r.b);
      ms += t;
    }
    char line[256];
    snprintf(line, sizeof line, "%s\t%zu\t%.4f\t%.1f\n", kv.first.c_str(), kv.second.recs.size(), ms,
             ms > 0 ? kv.second.flops / (ms * 1e-3) / 1e12 : 0.0);
    out += line;
  }
  g_prof.shapes.clear();
  if ((int)out.size() + 1 > cap) return B2F_ERR_WORKSPACE;
  memcpy(buf, out.c_str(), out.size() + 1);
  return (int)out.size();
}
extern "C" int b2f_prof_collect(int kc, double* ms, int64_t* launches, double* flops, double* bytes) {
  if (kc < 0 || kc >= KC_COUNT) return B2F_ERR_INVALID;
  std::lock_guard<std::mutex> lk(g_prof.mu);
  double total = 0;
  for (auto& r : g_prof.recs[kc]) {
    if (cudaEventSynchronize(r.b) != cudaSuccess) return B2F_ERR_CUDA;
    float t = 0;
    cudaEventElapsedTime(&t, r.a, r.b);
    total += t;
    g_prof.pool.push_back(r.a);
    g_prof.pool.push_back(r.b);
  }
  if (ms) *ms = total;
  if (launches) *launches = (int64_t)g_prof.recs[kc].size();
  if (flops) *flops = g_prof.flops[kc];
  if (bytes) *bytes = g_prof.bytes[kc];
  g_prof.recs[kc].clear();
  g_prof.flops[kc] = g_prof.bytes[kc] = 0;
  return B2F_OK;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) ==
            cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
    else
      cudaGetLastError();
  });
  return fn;
}

int make_tmap_2d_bf16(CUtensorMap* out, const void* gptr, uint64_t rows, uint64_t cols,
                      uint64_t ld_elems, uint32_t box_rows, uint32_t box_cols) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return B2F_ERR_CUDA;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld_elems * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(gptr), dims, strides,
                  box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "[b2f] cuTensorMapEncodeTiled(2d) failed: %d (rows=%llu cols=%llu ld=%llu)\n",
            int(r), (unsigned long long)rows, (unsigned long long)cols,
            (unsigned long long)ld_elems);
    return B2F_ERR_CUDA;
  }
  return B2F_OK;
}

int make_tmap_3d_rows(CUtensorMap* out, const void* gptr, uint64_t width, uint64_t rows,
                      uint64_t batch, uint64_t ld_elems, uint64_t batch_stride_elems, uint32_t box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return B2F_ERR_CUDA;
  cuuint64_t dims[3] = {width, rows, batch};
  cuuint64_t strides[2] = {ld_elems * 2, batch_stride_elems * 2};
  cuuint32_t box[3] = {64, box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(gptr), dims, strides,
                  box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "[b2f] cuTensorMapEncodeTiled(3d) failed: %d\n", int(r));
    return B2F_ERR_CUDA;
  }
  return B2F_OK;
}

int make_tmap_u8_rows(CUtensorMap* out, const void* gptr, int rank, uint64_t width, uint64_t rows, uint64_t batch,
                      uint64_t ld_bytes, uint64_t batch_stride_bytes) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return B2F_ERR_CUDA;
  if (rank != 2 && rank != 3) return B2F_ERR_INVALID;
  cuuint64_t dims[3] = {width, rows, batch};
  cuuint64_t strides[2] = {ld_bytes, batch_stride_bytes};
  cuuint32_t box[3] = {128, 128, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, rank, const_cast<void*>(gptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "[b2f] cuTensorMapEncodeTiled(u8 %dd) failed: %d\n", rank, int(r));
    return B2F_ERR_CUDA;
  }
  return B2F_OK;
}

int make_tmap_4d_bf16(CUtensorMap* out, const void* gptr, uint64_t n, uint64_t h, uint64_t w,
                      uint64_t c, uint32_t box_h, uint32_t box_w, uint32_t box_c, uint32_t stride) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return B2F_ERR_CUDA;
  cuuint64_t dims[4] = {c, w, h, n};
  cuuint64_t strides[3] = {c * 2, w * c * 2, h * w * c * 2};
  cuuint32_t box[4] = {box_c, box_w * stride, box_h * stride, 1};
  cuuint32_t estr[4] = {1, stride, stride, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(gptr), dims, strides,
                  box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "[b2f] cuTensorMapEncodeTiled(4d) failed: %d\n", int(r));
    return B2F_ERR_CUDA;
  }
  return B2F_OK;
}

}  // namespace b2f
