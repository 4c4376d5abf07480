// extern "C" surface of libb2f.so — thin argument marshalling over the b2f:: launchers.
#include <atomic>

#include "host_common.h"

namespace b2f {
extern std::atomic<uint64_t> g_launch_count;
int gemm_bf16(const void* A, int64_t lda, int64_t a_bs, const void* W, int64_t ldw,
              const void* bias, void* out, int64_t ldc, int64_t out_bs, int batch, int M, int N,
              int K, int epilogue, const void* resid, int64_t ldr, int64_t resid_bs, const void* gate,
              int64_t gate_ld, cudaStream_t stream);
int gemm_qkv_norm_rope(const void* A, int64_t lda, int64_t a_bs, const void* W, int64_t ldw,
                       const void* bias, void* out, int64_t ldc, int64_t out_bs, int batch, int M,
                       int d_model, int K, const void* nw_q, const void* nw_k, const float* cos,
                       const float* sin, int rope_row0, float eps, int n_extra, void* out_extra,
                       int64_t ld_extra, int64_t bs_extra, int epi_extra, cudaStream_t stream);
int ln_modulate(const void* x, int64_t ldx, int64_t x_batch_stride, const void* scale,
                const void* shift, int64_t mod_ld, void* out, int64_t ldo, int64_t out_batch_stride,
                int batch, int rows, int D, float eps, int split_row, const void* scale_b,
                const void* shift_b, cudaStream_t stream);
int rmsnorm_rope(void* q, void* k, int64_t ld, int64_t batch_stride, const void* wq_a,
                 const void* wk_a, const void* wq_b, const void* wk_b, const float* cos,
                 const float* sin, int batch, int S, int H, int head_dim, int n_a, float eps,
                 cudaStream_t stream);
int euler_step(void* x, int64_t ldx, const void* v, int64_t ldv, int64_t rows, int cols, float dt,
               cudaStream_t stream);
int silu(const void* x, void* y, int64_t n, cudaStream_t stream);
int temb_sinusoid(const float* t, void* out, int rows, cudaStream_t stream);
int temb_combine(const void* t, const void* g, const void* txt, void* temb, void* silu_temb, int64_t n,
                 cudaStream_t stream);
void prof_set(bool on);
int rmsnorm(const void* x, int64_t ldx, const void* w, void* y, int64_t ldy, int64_t rows, int D,
            float eps, cudaStream_t stream);
int rope_half(void* x, int64_t ld, int heads, int head_pitch, const float* cos, const float* sin,
              int rot, int64_t tokens, int fp32_math, cudaStream_t stream);
int swiglu(const void* gu, int64_t ld, void* out, int64_t ldo, int64_t rows, int I,
           cudaStream_t stream);
int move_rows(const void* src, int64_t ld_src, void* dst, int64_t ld_dst, const int64_t* idx, int64_t n,
              int D, int scatter, cudaStream_t stream);
int conv3x3(const void* in, const void* w, const void* bias, void* out, const void* resid, int N,
            int Hin, int Win, int Cin, int Cout, int stride, int out_nchw, cudaStream_t stream);
int groupnorm_silu(const void* x, const void* gamma, const void* beta, void* y, double* stats_ws,
                   int N, long long P, int C, float eps, int silu, cudaStream_t stream);
int upsample2x(const void* in, void* out, int N, int H, int W, int C, cudaStream_t stream);
int nchw_to_nhwc_pad(const void* in, int in_is_f32, void* out, int N, int C, int H, int W, int Cpad,
                     cudaStream_t stream);
int softmax_rows(void* s, int64_t ld, int rows, int L, float scale, cudaStream_t stream);
int transpose_bf16(const void* in, int64_t ld_in, void* out, int64_t ld_out, int R, int Cc,
                   cudaStream_t stream);
int prof_collect(int kc, double* ms, int64_t* launches, double* flops, double* bytes);
int prof_shapes(char* buf, int cap);
int rope_tables(const float* ids, int S, const int* axes_dim, double theta, float* cos, float* sin,
                cudaStream_t stream);
int attention_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v,
                  int64_t ldv, void* out, int64_t ldo, int B, int H, int Hkv, int Sq, int Skv,
                  int head_dim, float scale, int causal, cudaStream_t stream);
int attention_bias_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v,
                       int64_t ldv, void* out, int64_t ldo, int B, int H, int Hkv, int Sq, int Skv,
                       int head_dim, float scale, int causal, const void* bias, int64_t bias_h_stride,
                       int64_t bias_row_stride, cudaStream_t stream);
int geglu(const void* gu, int64_t ld, void* out, int64_t ldo, int64_t rows, int I, cudaStream_t stream);
int layernorm(const void* x, int64_t ldx, const void* w, const void* b, void* y, int64_t ldy,
              int64_t rows, int D, float eps, cudaStream_t stream);
int embed(const void* tok, int64_t ld_tok, const int64_t* ids, const void* pos, int64_t ld_pos, int period,
          void* out, int64_t ldo, int64_t n, int D, cudaStream_t stream);
// training step (train_kernels.cu, attention_bwd.cu, gemm.cu)
int gemm_dgrad(const void* dY, int64_t ldy, int64_t dy_bs, const void* W, int64_t ldw, void* dX, int64_t ldx,
               int64_t dx_bs, int batch, int M, int N, int K, int epilogue, const void* aux, int64_t ld_aux,
               int64_t aux_bs, cudaStream_t stream);
int gemm_wgrad(const void* dY, int64_t ldy, int64_t dy_bs, const void* X, int64_t ldx, int64_t x_bs, float* dW,
               int64_t ldw, int batch, int rows, int M, int N, int accumulate, cudaStream_t stream);
int attention_fwd_lse(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* out,
                      int64_t ldo, int B, int H, int Hkv, int Sq, int Skv, int head_dim, float scale, int causal,
                      float* lse, int64_t lse_stride, cudaStream_t stream);
int attention_bwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, const void* dout,
                  int64_t lddo, const float* lse, const float* delta, int64_t S_pad, void* dq, int64_t lddq, void* dk,
                  int64_t lddk, void* dv, int64_t lddv, int B, int H, int S, int head_dim, float scale,
                  cudaStream_t stream);
int train_chunks(int rows);
int train_ln_chunks(int rows);
int gate_resid_fwd(const void* x, int64_t ldx, int64_t x_bs, const void* y, int64_t ldy, int64_t y_bs, const void* gate,
                   const void* gate_b, int64_t gate_ld, void* out, int64_t ldo, int64_t o_bs, int batch, int rows, int D,
                   int split_row, cudaStream_t st);
int gate_bwd(const void* dout, int64_t ldd, int64_t d_bs, const void* y, int64_t ldy, int64_t y_bs, const void* gate,
             const void* gate_b, int64_t gate_ld, void* dy, int64_t ldo, int64_t o_bs, float* partial, int batch,
             int rows, int D, int split_row, int part_row0, cudaStream_t st);
int col_reduce(const float* partial, int nchunks, int D, float* out, int64_t out_ld, int batch, int accumulate,
               cudaStream_t st);
int ln_modulate_bwd(const void* x, int64_t ldx, int64_t x_bs, const void* dy, int64_t ldy, int64_t dy_bs,
                    const void* scale, const void* scale_b, int64_t mod_ld, const void* dres_in, int64_t ldr, int64_t r_bs,
                    void* dres_out, int64_t ldo, int64_t o_bs, float* partial, int batch, int rows, int D, float eps,
                    int split_row, int part_row0, cudaStream_t st);
int rmsnorm_rope_out(const void* xq, const void* xk, int64_t ldx, int64_t x_bs, void* oq, void* ok, int64_t ldo,
                     int64_t o_bs, const void* wq_a, const void* wk_a, const void* wq_b, const void* wk_b,
                     const float* cos, const float* sin, int batch, int S, int H, int n_a, float eps, cudaStream_t st);
int rmsnorm_rope_bwd(void* dq, void* dk, int64_t ld, int64_t bs, const void* xq, const void* xk, int64_t ldx, int64_t x_bs,
                     const void* wq_a, const void* wk_a, const void* wq_b, const void* wk_b, const float* cos,
                     const float* sin, float* partial, int batch, int S, int H, int n_a, float eps, cudaStream_t st);
int gelu_rows(const void* x, int64_t ldx, void* y, int64_t ldy, int64_t rows, int D, cudaStream_t st);
int outer_acc(const float* dmod, int64_t dmod_ld, const void* act, int64_t act_ld, float* dW, int64_t ldw, int B, int N,
              int K, int accumulate, cudaStream_t st);
int attn_delta(const void* o, int64_t ldo, const void* dout, int64_t lddo, float* delta, float* lse, int B, int H, int S,
               int S_pad, cudaStream_t st);
int mse_loss(const void* pred, const float* target, const float* w, void* dpred, float* loss_out, float* ws, int64_t n,
             float grad_scale, cudaStream_t st);
int grad_sumsq(const float* g, int64_t n, float* sumsq_out, float* ws, int accumulate, cudaStream_t st);
int clip_coef(const float* sumsq, float max_norm, float pre_scale, float* coef, float* norm_out, cudaStream_t st);
int adamw_step(float* p32, float* m, float* v, const float* g, void* p16, int64_t n, float lr, float beta1, float beta2,
               float eps, float wd, int step, const float* gscale, cudaStream_t st);
int cast_bf16_f32(const void* src, void* dst, int64_t n, int to_f32, cudaStream_t st);
int blend_bf16(const void* a, const void* b, float wa, float wb, void* out, int64_t n, cudaStream_t st);
// LoRA (gemm.cu, lora.cu)
int gemm_bf16_lora(const void* A, int64_t lda, int64_t a_bs, const void* W, int64_t ldw, const void* bias, void* out,
                   int64_t ldc, int64_t out_bs, int batch, int M, int N, int K, int epilogue, const void* resid,
                   int64_t ldr, int64_t resid_bs, const void* gate, int64_t gate_ld, const void* T, int64_t ldt,
                   int64_t t_bs, const void* Bc, int64_t ldbc, int r_pad, cudaStream_t stream);
int gemm_qkv_norm_rope_lora(const void* A, int64_t lda, int64_t a_bs, const void* W, int64_t ldw, const void* bias,
                            void* out, int64_t ldc, int64_t out_bs, int batch, int M, int d_model, int K,
                            const void* nw_q, const void* nw_k, const float* cos, const float* sin, int rope_row0,
                            float eps, int n_extra, void* out_extra, int64_t ld_extra, int64_t bs_extra,
                            int epi_extra, const void* T, int64_t ldt, int64_t t_bs, const void* Bc, int64_t ldbc,
                            int r_pad, cudaStream_t stream);
int gemm_colscale(const void* A, int64_t lda, int64_t a_bs, const void* W, int64_t ldw, void* out, int64_t ldc,
                  int64_t out_bs, int batch, int M, int N, int K, const float* colscale, float cs_mul,
                  cudaStream_t stream);
int lora_fuse(void* W, int64_t ldw, int rows, int cols, const void* Bc, int64_t ldb, const void* A, int64_t lda,
              const float* colscale, float cs_mul, int r, cudaStream_t stream);
}  // namespace b2f

extern "C" {

const char* b2f_strerror(int code) {
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

int b2f_version(void) { return 2; }

int b2f_device_info(int* num_sms, int* cc_major, int* cc_minor, size_t* smem_optin) {
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

uint64_t b2f_launch_count(void) { return b2f::g_launch_count.load(); }

void b2f_prof_enable(int on) { b2f::prof_set(on != 0); }
int b2f_prof_shapes(char* buf, int cap) { return b2f::prof_shapes(buf, cap); }
int b2f_prof_collect(int kernel_class, double* ms, int64_t* launches, double* flops, double* bytes) {
  return b2f::prof_collect(kernel_class, ms, launches, flops, bytes);
}

int b2f_gemm_bf16(const void* A, int64_t lda, int64_t a_batch_stride, const void* W, int64_t ldw,
                  const void* bias, void* out, int64_t ldc, int64_t out_batch_stride, int batch,
                  int M, int N, int K, int epilogue, const void* resid, int64_t ldr,
                  int64_t resid_batch_stride, const void* gate, int64_t gate_ld,
                  b2f_stream_t stream) {
  return b2f::gemm_bf16(A, lda, a_batch_stride, W, ldw, bias, out, ldc, out_batch_stride, batch, M,
                        N, K, epilogue, resid, ldr, resid_batch_stride, gate, gate_ld,
                        static_cast<cudaStream_t>(stream));
}

int b2f_gemm_qkv_norm_rope(const void* A, int64_t lda, int64_t a_batch_stride, const void* W,
                           int64_t ldw, const void* bias, void* out, int64_t ldc,
                           int64_t out_batch_stride, int batch, int M, int d_model, int K,
                           const void* nw_q, const void* nw_k, const float* cos, const float* sin,
                           int rope_row0, float eps, int n_extra, void* out_extra, int64_t ld_extra,
                           int64_t extra_batch_stride, int epi_extra, b2f_stream_t stream) {
  return b2f::gemm_qkv_norm_rope(A, lda, a_batch_stride, W, ldw, bias, out, ldc, out_batch_stride, batch,
                                 M, d_model, K, nw_q, nw_k, cos, sin, rope_row0, eps, n_extra, out_extra,
                                 ld_extra, extra_batch_stride, epi_extra, static_cast<cudaStream_t>(stream));
}

int b2f_ln_modulate(const void* x, int64_t ldx, int64_t x_batch_stride, const void* scale,
                    const void* shift, int64_t mod_ld, void* out, int64_t ldo,
                    int64_t out_batch_stride, int batch, int rows, int D, float eps, int split_row,
                    const void* scale_b, const void* shift_b, b2f_stream_t stream) {
  return b2f::ln_modulate(x, ldx, x_batch_stride, scale, shift, mod_ld, out, ldo, out_batch_stride,
                          batch, rows, D, eps, split_row, scale_b, shift_b, static_cast<cudaStream_t>(stream));
}

int b2f_rmsnorm_rope(void* q, void* k, int64_t ld, int64_t batch_stride, const void* wq_a,
                     const void* wk_a, const void* wq_b, const void* wk_b, const float* cos,
                     const float* sin, int batch, int S, int H, int head_dim, int n_a, float eps,
                     b2f_stream_t stream) {
  return b2f::rmsnorm_rope(q, k, ld, batch_stride, wq_a, wk_a, wq_b, wk_b, cos, sin, batch, S, H,
                           head_dim, n_a, eps, static_cast<cudaStream_t>(stream));
}

int b2f_euler_step(void* x, int64_t ldx, const void* v, int64_t ldv, int64_t rows, int cols,
                   float dt, b2f_stream_t stream) {
  return b2f::euler_step(x, ldx, v, ldv, rows, cols, dt, static_cast<cudaStream_t>(stream));
}

int b2f_rope_tables(const float* ids, int S, const int* axes_dim, double theta, float* cos,
                    float* sin, b2f_stream_t stream) {
  return b2f::rope_tables(ids, S, axes_dim, theta, cos, sin, static_cast<cudaStream_t>(stream));
}

int b2f_conv3x3(const void* in, const void* w, const void* bias, void* out, const void* resid, int N,
                int Hin, int Win, int Cin, int Cout, int stride, int out_nchw, b2f_stream_t stream) {
  return b2f::conv3x3(in, w, bias, out, resid, N, Hin, Win, Cin, Cout, stride, out_nchw,
                      static_cast<cudaStream_t>(stream));
}
int b2f_groupnorm_silu(const void* x, const void* gamma, const void* beta, void* y, void* stats_ws,
                       int N, int64_t P, int C, float eps, int silu, b2f_stream_t stream) {
  return b2f::groupnorm_silu(x, gamma, beta, y, static_cast<double*>(stats_ws), N, P, C, eps, silu,
                             static_cast<cudaStream_t>(stream));
}
int b2f_upsample2x(const void* in, void* out, int N, int H, int W, int C, b2f_stream_t stream) {
  return b2f::upsample2x(in, out, N, H, W, C, static_cast<cudaStream_t>(stream));
}
int b2f_nchw_to_nhwc_pad(const void* in, int in_is_f32, void* out, int N, int C, int H, int W,
                         int Cpad, b2f_stream_t stream) {
  return b2f::nchw_to_nhwc_pad(in, in_is_f32, out, N, C, H, W, Cpad, static_cast<cudaStream_t>(stream));
}
int b2f_softmax_rows(void* s, int64_t ld, int rows, int L, float scale, b2f_stream_t stream) {
  return b2f::softmax_rows(s, ld, rows, L, scale, static_cast<cudaStream_t>(stream));
}
int b2f_transpose_bf16(const void* in, int64_t ld_in, void* out, int64_t ld_out, int R, int Cc,
                       b2f_stream_t stream) {
  return b2f::transpose_bf16(in, ld_in, out, ld_out, R, Cc, static_cast<cudaStream_t>(stream));
}

int b2f_rmsnorm(const void* x, int64_t ldx, const void* w, void* y, int64_t ldy, int64_t rows, int D,
                float eps, b2f_stream_t stream) {
  return b2f::rmsnorm(x, ldx, w, y, ldy, rows, D, eps, static_cast<cudaStream_t>(stream));
}
int b2f_rope_half(void* x, int64_t ld, int heads, int head_pitch, const float* cos, const float* sin,
                  int rot, int64_t tokens, int fp32_math, b2f_stream_t stream) {
  return b2f::rope_half(x, ld, heads, head_pitch, cos, sin, rot, tokens, fp32_math,
                        static_cast<cudaStream_t>(stream));
}
int b2f_swiglu(const void* gu, int64_t ld, void* out, int64_t ldo, int64_t rows, int I,
               b2f_stream_t stream) {
  return b2f::swiglu(gu, ld, out, ldo, rows, I, static_cast<cudaStream_t>(stream));
}
int b2f_move_rows(const void* src, int64_t ld_src, void* dst, int64_t ld_dst, const int64_t* idx,
                  int64_t n, int D, int scatter, b2f_stream_t stream) {
  return b2f::move_rows(src, ld_src, dst, ld_dst, idx, n, D, scatter, static_cast<cudaStream_t>(stream));
}

int b2f_silu(const void* x, void* y, int64_t n, b2f_stream_t stream) {
  return b2f::silu(x, y, n, static_cast<cudaStream_t>(stream));
}
int b2f_temb_sinusoid(const float* t, void* out, int rows, b2f_stream_t stream) {
  return b2f::temb_sinusoid(t, out, rows, static_cast<cudaStream_t>(stream));
}
int b2f_temb_combine(const void* t, const void* g, const void* txt, void* temb, void* silu_temb, int64_t n,
                     b2f_stream_t stream) {
  return b2f::temb_combine(t, g, txt, temb, silu_temb, n, static_cast<cudaStream_t>(stream));
}

int b2f_attention_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v,
                      int64_t ldv, void* out, int64_t ldo, int B, int H, int Hkv, int Sq, int Skv,
                      int head_dim, float scale, int causal, b2f_stream_t stream) {
  return b2f::attention_fwd(q, ldq, k, ldk, v, ldv, out, ldo, B, H, Hkv, Sq, Skv, head_dim, scale,
                            causal, static_cast<cudaStream_t>(stream));
}

int b2f_attention_bias_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v,
                           int64_t ldv, void* out, int64_t ldo, int B, int H, int Hkv, int Sq, int Skv,
                           int head_dim, float scale, int causal, const void* bias,
                           int64_t bias_h_stride, int64_t bias_row_stride, b2f_stream_t stream) {
  return b2f::attention_bias_fwd(q, ldq, k, ldk, v, ldv, out, ldo, B, H, Hkv, Sq, Skv, head_dim, scale,
                                 causal, bias, bias_h_stride, bias_row_stride,
                                 static_cast<cudaStream_t>(stream));
}
int b2f_geglu(const void* gu, int64_t ld, void* out, int64_t ldo, int64_t rows, int I,
              b2f_stream_t stream) {
  return b2f::geglu(gu, ld, out, ldo, rows, I, static_cast<cudaStream_t>(stream));
}
int b2f_layernorm(const void* x, int64_t ldx, const void* w, const void* b, void* y, int64_t ldy,
                  int64_t rows, int D, float eps, b2f_stream_t stream) {
  return b2f::layernorm(x, ldx, w, b, y, ldy, rows, D, eps, static_cast<cudaStream_t>(stream));
}
int b2f_embed(const void* tok, int64_t ld_tok, const int64_t* ids, const void* pos, int64_t ld_pos,
              int period, void* out, int64_t ldo, int64_t n, int D, b2f_stream_t stream) {
  return b2f::embed(tok, ld_tok, ids, pos, ld_pos, period, out, ldo, n, D,
                    static_cast<cudaStream_t>(stream));
}

// ------------------------------------------------------------------ training step
#define ST static_cast<cudaStream_t>(stream)
int b2f_gemm_dgrad(const void* dY, int64_t ldy, int64_t dy_batch_stride, const void* W, int64_t ldw, void* dX,
                   int64_t ldx, int64_t dx_batch_stride, int batch, int M, int N, int K, int epilogue, const void* aux,
                   int64_t ld_aux, int64_t aux_batch_stride, b2f_stream_t stream) {
  return b2f::gemm_dgrad(dY, ldy, dy_batch_stride, W, ldw, dX, ldx, dx_batch_stride, batch, M, N, K, epilogue, aux,
                         ld_aux, aux_batch_stride, ST);
}
int b2f_gemm_wgrad(const void* dY, int64_t ldy, int64_t dy_batch_stride, const void* X, int64_t ldx,
                   int64_t x_batch_stride, float* dW, int64_t ldw, int batch, int rows, int M, int N, int accumulate,
                   b2f_stream_t stream) {
  return b2f::gemm_wgrad(dY, ldy, dy_batch_stride, X, ldx, x_batch_stride, dW, ldw, batch, rows, M, N, accumulate, ST);
}
int b2f_attention_fwd_lse(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* out,
                          int64_t ldo, int B, int H, int Hkv, int Sq, int Skv, int head_dim, float scale, int causal,
                          float* lse, int64_t lse_stride, b2f_stream_t stream) {
  return b2f::attention_fwd_lse(q, ldq, k, ldk, v, ldv, out, ldo, B, H, Hkv, Sq, Skv, head_dim, scale, causal, lse,
                                lse_stride, ST);
}
int b2f_attention_bwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv,
                      const void* dout, int64_t lddo, const float* lse, const float* delta, int64_t S_pad, void* dq,
                      int64_t lddq, void* dk, int64_t lddk, void* dv, int64_t lddv, int B, int H, int S, int head_dim,
                      float scale, b2f_stream_t stream) {
  return b2f::attention_bwd(q, ldq, k, ldk, v, ldv, dout, lddo, lse, delta, S_pad, dq, lddq, dk, lddk, dv, lddv, B, H, S,
                            head_dim, scale, ST);
}
int b2f_attn_delta(const void* o, int64_t ldo, const void* dout, int64_t lddo, float* delta, float* lse, int B, int H,
                   int S, int S_pad, b2f_stream_t stream) {
  return b2f::attn_delta(o, ldo, dout, lddo, delta, lse, B, H, S, S_pad, ST);
}
int b2f_train_chunks(int rows) { return b2f::train_chunks(rows); }
int b2f_train_ln_chunks(int rows) { return b2f::train_ln_chunks(rows); }
int b2f_gate_resid_fwd(const void* x, int64_t ldx, int64_t x_bs, const void* y, int64_t ldy, int64_t y_bs,
                       const void* gate, const void* gate_b, int64_t gate_ld, void* out, int64_t ldo, int64_t o_bs,
                       int batch, int rows, int D, int split_row, b2f_stream_t stream) {
  return b2f::gate_resid_fwd(x, ldx, x_bs, y, ldy, y_bs, gate, gate_b, gate_ld, out, ldo, o_bs, batch, rows, D, split_row, ST);
}
int b2f_gate_bwd(const void* dout, int64_t ldd, int64_t d_bs, const void* y, int64_t ldy, int64_t y_bs, const void* gate,
                 const void* gate_b, int64_t gate_ld, void* dy, int64_t ldo, int64_t o_bs, float* partial, int batch,
                 int rows, int D, int split_row, int part_row0, b2f_stream_t stream) {
  return b2f::gate_bwd(dout, ldd, d_bs, y, ldy, y_bs, gate, gate_b, gate_ld, dy, ldo, o_bs, partial, batch, rows, D,
                       split_row, part_row0, ST);
}
int b2f_col_reduce(const float* partial, int nchunks, int D, float* out, int64_t out_ld, int batch, int accumulate,
                   b2f_stream_t stream) {
  return b2f::col_reduce(partial, nchunks, D, out, out_ld, batch, accumulate, ST);
}
int b2f_ln_modulate_bwd(const void* x, int64_t ldx, int64_t x_bs, const void* dy, int64_t ldy, int64_t dy_bs,
                        const void* scale, const void* scale_b, int64_t mod_ld, const void* dres_in, int64_t ldr,
                        int64_t r_bs, void* dres_out, int64_t ldo, int64_t o_bs, float* partial, int batch, int rows,
                        int D, float eps, int split_row, int part_row0, b2f_stream_t stream) {
  return b2f::ln_modulate_bwd(x, ldx, x_bs, dy, ldy, dy_bs, scale, scale_b, mod_ld, dres_in, ldr, r_bs, dres_out, ldo,
                              o_bs, partial, batch, rows, D, eps, split_row, part_row0, ST);
}
int b2f_rmsnorm_rope_out(const void* xq, const void* xk, int64_t ldx, int64_t x_bs, void* oq, void* ok, int64_t ldo,
                         int64_t o_bs, const void* wq_a, const void* wk_a, const void* wq_b, const void* wk_b,
                         const float* cos, const float* sin, int batch, int S, int H, int n_a, float eps,
                         b2f_stream_t stream) {
  return b2f::rmsnorm_rope_out(xq, xk, ldx, x_bs, oq, ok, ldo, o_bs, wq_a, wk_a, wq_b, wk_b, cos, sin, batch, S, H, n_a,
                               eps, ST);
}
int b2f_rmsnorm_rope_bwd(void* dq, void* dk, int64_t ld, int64_t bs, const void* xq, const void* xk, int64_t ldx,
                         int64_t x_bs, const void* wq_a, const void* wk_a, const void* wq_b, const void* wk_b,
                         const float* cos, const float* sin, float* partial, int batch, int S, int H, int n_a, float eps,
                         b2f_stream_t stream) {
  return b2f::rmsnorm_rope_bwd(dq, dk, ld, bs, xq, xk, ldx, x_bs, wq_a, wk_a, wq_b, wk_b, cos, sin, partial, batch, S, H,
                               n_a, eps, ST);
}
int b2f_gelu_rows(const void* x, int64_t ldx, void* y, int64_t ldy, int64_t rows, int D, b2f_stream_t stream) {
  return b2f::gelu_rows(x, ldx, y, ldy, rows, D, ST);
}
int b2f_outer_acc(const float* dmod, int64_t dmod_ld, const void* act, int64_t act_ld, float* dW, int64_t ldw, int B,
                  int N, int K, int accumulate, b2f_stream_t stream) {
  return b2f::outer_acc(dmod, dmod_ld, act, act_ld, dW, ldw, B, N, K, accumulate, ST);
}
int b2f_mse_loss(const void* pred, const float* target, const float* w, void* dpred, float* loss_out, float* ws,
                 int64_t n, float grad_scale, b2f_stream_t stream) {
  return b2f::mse_loss(pred, target, w, dpred, loss_out, ws, n, grad_scale, ST);
}
int b2f_grad_sumsq(const float* g, int64_t n, float* sumsq_out, float* ws, int accumulate, b2f_stream_t stream) {
  return b2f::grad_sumsq(g, n, sumsq_out, ws, accumulate, ST);
}
int b2f_clip_coef(const float* sumsq, float max_norm, float pre_scale, float* coef, float* norm_out, b2f_stream_t stream) {
  return b2f::clip_coef(sumsq, max_norm, pre_scale, coef, norm_out, ST);
}
int b2f_adamw_step(float* p32, float* m, float* v, const float* g, void* p16, int64_t n, float lr, float beta1,
                   float beta2, float eps, float weight_decay, int step, const float* gscale, b2f_stream_t stream) {
  return b2f::adamw_step(p32, m, v, g, p16, n, lr, beta1, beta2, eps, weight_decay, step, gscale, ST);
}
int b2f_cast_bf16_f32(const void* src, void* dst, int64_t n, int to_f32, b2f_stream_t stream) {
  return b2f::cast_bf16_f32(src, dst, n, to_f32, ST);
}
int b2f_blend_bf16(const void* a, const void* b, float wa, float wb, void* out, int64_t n, b2f_stream_t stream) {
  return b2f::blend_bf16(a, b, wa, wb, out, n, ST);
}

// ------------------------------------------------------------------ LoRA
int b2f_gemm_bf16_lora(const void* A, int64_t lda, int64_t a_batch_stride, const void* W, int64_t ldw,
                       const void* bias, void* out, int64_t ldc, int64_t out_batch_stride, int batch, int M, int N,
                       int K, int epilogue, const void* resid, int64_t ldr, int64_t resid_batch_stride,
                       const void* gate, int64_t gate_ld, const void* T, int64_t ldt, int64_t t_batch_stride,
                       const void* Bcat, int64_t ldbc, int r_pad, b2f_stream_t stream) {
  return b2f::gemm_bf16_lora(A, lda, a_batch_stride, W, ldw, bias, out, ldc, out_batch_stride, batch, M, N, K,
                             epilogue, resid, ldr, resid_batch_stride, gate, gate_ld, T, ldt, t_batch_stride, Bcat,
                             ldbc, r_pad, ST);
}
int b2f_gemm_qkv_norm_rope_lora(const void* A, int64_t lda, int64_t a_batch_stride, const void* W, int64_t ldw,
                                const void* bias, void* out, int64_t ldc, int64_t out_batch_stride, int batch, int M,
                                int d_model, int K, const void* nw_q, const void* nw_k, const float* cos,
                                const float* sin, int rope_row0, float eps, int n_extra, void* out_extra,
                                int64_t ld_extra, int64_t extra_batch_stride, int epi_extra, const void* T,
                                int64_t ldt, int64_t t_batch_stride, const void* Bcat, int64_t ldbc, int r_pad,
                                b2f_stream_t stream) {
  return b2f::gemm_qkv_norm_rope_lora(A, lda, a_batch_stride, W, ldw, bias, out, ldc, out_batch_stride, batch, M,
                                      d_model, K, nw_q, nw_k, cos, sin, rope_row0, eps, n_extra, out_extra, ld_extra,
                                      extra_batch_stride, epi_extra, T, ldt, t_batch_stride, Bcat, ldbc, r_pad, ST);
}
int b2f_gemm_colscale(const void* A, int64_t lda, int64_t a_batch_stride, const void* W, int64_t ldw, void* out,
                      int64_t ldc, int64_t out_batch_stride, int batch, int M, int N, int K, const float* colscale,
                      float cs_mul, b2f_stream_t stream) {
  return b2f::gemm_colscale(A, lda, a_batch_stride, W, ldw, out, ldc, out_batch_stride, batch, M, N, K, colscale,
                            cs_mul, ST);
}
int b2f_lora_fuse(void* W, int64_t ldw, int rows, int cols, const void* Bcat, int64_t ldb, const void* Acat,
                  int64_t lda, const float* colscale, float cs_mul, int r, b2f_stream_t stream) {
  return b2f::lora_fuse(W, ldw, rows, cols, Bcat, ldb, Acat, lda, colscale, cs_mul, r, ST);
}
#undef ST

}  // extern "C"
