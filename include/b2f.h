/* b2f.h — C ABI of the H100-native FLUX-Kontext denoising engine (libb2f.so).
 *
 * The reference (wyhlovecpp/GPT-Image-Edit) has no FFI: its hot path sits behind Python object
 * protocols whose arithmetic lives in diffusers 0.32.2 / torch (SURVEY.md §8b).  Every entry
 * point below names the reference interface it replaces (path:line under /root/reference).
 *
 * Conventions
 *   - every call returns B2F_OK (0) or a negative error code; nothing throws or aborts;
 *   - all pointers are DEVICE pointers owned by the caller (PyTorch owns storage), row-major,
 *     innermost dimension contiguous, 16-byte aligned; `ld*` arguments are row pitches in
 *     elements;
 *   - all work is enqueued on the caller's stream (a cudaStream_t passed as void*); no call
 *     allocates device memory or synchronises the host unless stated;
 *   - dtype is bf16 (raw uint16 storage) unless a parameter says otherwise.
 */
#ifndef B2F_H_
#define B2F_H_
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2F_OK 0
#define B2F_ERR_INVALID (-1)     /* bad shape / argument */
#define B2F_ERR_CUDA (-2)        /* CUDA runtime/driver error (message on stderr) */
#define B2F_ERR_UNSUPPORTED (-3) /* shape or mode not implemented */
#define B2F_ERR_ALIGN (-4)       /* pointer or pitch not 16-byte aligned */
#define B2F_ERR_NODEVICE (-5)    /* no sm_90 device visible */
#define B2F_ERR_WORKSPACE (-6)   /* workspace too small */

typedef void* b2f_stream_t; /* cudaStream_t */

const char* b2f_strerror(int code);
/* ABI version; bumped on any signature change or addition (2: LoRA entry points, 3: FP8 entry points, 4: FP8
 * attention, 5: first-block cache, 6: GEMM tile override, 7: FP8 GEMMs with unfused LoRA, 8: VAE stop stage, ragged
 * and fp32-input softmax rows, 9: per-item text windows in the joint attention). */
int b2f_version(void);
/* Device facts the host needs for grid sizing / reporting. Returns B2F_ERR_NODEVICE without GPU. */
int b2f_device_info(int* num_sms, int* cc_major, int* cc_minor, size_t* smem_optin);
/* Number of kernels this library has launched since load (bench.py's gpu_launches claim). */
uint64_t b2f_launch_count(void);

/* Per-kernel-class device timing for bench.py's roofline: when enabled, every launch of that class
 * is bracketed by CUDA events on the launching stream.  b2f_prof_collect synchronises those events,
 * returns their summed duration (ms), the launch count and the algorithmic FLOPs / bytes the
 * launches declared, and resets the class.  Classes: 0 gemm, 1 attention, 2 ln_modulate,
 * 3 rmsnorm_rope, 4 conv, 5 other. */
void b2f_prof_enable(int on);
int b2f_prof_collect(int kernel_class, double* ms, int64_t* launches, double* flops, double* bytes);
/* Per-shape breakdown of the GEMM class since the last call: lines "tag<TAB>launches<TAB>ms<TAB>TFLOP/s" written to buf
 * (returns the length, or B2F_ERR_WORKSPACE if cap is too small).  Call BEFORE b2f_prof_collect. */
int b2f_prof_shapes(char* buf, int cap);

/* ------------------------------------------------------------------------------------------
 * Linear layer: out[M,N] = epilogue(A[M,K] · W[N,K]^T + bias[N]).  wgmma (fp32 accumulators in registers), TMA, mbarrier pipeline.
 * Replaces torch.nn.functional.linear → cuBLASLt as reached by diffusers' nn.Linear modules
 * (FluxTransformer2DModel: x_embedder, context_embedder, to_q/k/v, to_out, ff.net.*, proj_mlp,
 * proj_out, norm*.linear — SURVEY.md Appendix A.1/A.6; call site univa/utils/flux_pipeline.py:1067).
 *
 * Batched rows: A is [batch, M, K] (row pitch lda, batch pitch a_batch_stride), out/resid are
 * [batch, M, N] views with their own pitches; gate is [batch, N] (pitch gate_ld).  batch = 1 is
 * the plain 2-D case (batch strides ignored).  This lets one launch process the image rows (or
 * the text rows) of every batch item of a joint [B, S_txt+S_img, d] buffer.
 *
 * epilogue:
 *   B2F_EPI_BIAS        out = bf16(acc + bias)
 *   B2F_EPI_GELU_TANH   out = bf16(gelu_tanh(bf16(acc + bias)))     (ff.net.0 / proj_mlp)
 *   B2F_EPI_SILU        out = bf16(silu(bf16(acc + bias)))          (time_text_embed MLPs, MLP2)
 *   B2F_EPI_GATE_RESID  out = bf16(resid + bf16(gate[b,n] * bf16(acc + bias)))
 *                                                                    (x = x + gate * proj(...))
 * bias may be NULL.  resid may alias out.  K % 8 == 0, N % 8 == 0.
 */
#define B2F_EPI_BIAS 0
#define B2F_EPI_GELU_TANH 1
#define B2F_EPI_SILU 2
#define B2F_EPI_GATE_RESID 3
#define B2F_EPI_RESID 4 /* out = bf16(resid + bf16(acc + bias))  (VAE attention to_out + residual) */
#define B2F_EPI_QKV_NORM_ROPE 6 /* only through b2f_gemm_qkv_norm_rope */
#define B2F_EPI_GELU_ERF 5 /* out = bf16(gelu_erf(bf16(acc + bias)))  (Qwen2.5-VL patch merger, nn.GELU()) */
#define B2F_EPI_QUICK_GELU 7 /* out = bf16(x * bf16(sigmoid(bf16(1.702 x)))), x = bf16(acc + bias)  (CLIP-L MLP) */
/* backward epilogues (b2f_gemm_dgrad / b2f_gemm_wgrad only) */
#define B2F_EPI_DGELU 8   /* out = bf16(bf16(acc) * gelu_tanh'(u)),  u = saved pre-activation */
#define B2F_EPI_DSILU 9   /* out = bf16(bf16(acc) * silu'(u)) */
#define B2F_EPI_F32 10    /* fp32 store (weight gradients) */
#define B2F_EPI_F32_ACC 11 /* fp32 accumulate: out += acc (gradient accumulation steps) */

int b2f_gemm_bf16(const void* A, int64_t lda, int64_t a_batch_stride, const void* W, int64_t ldw,
                  const void* bias, void* out, int64_t ldc, int64_t out_batch_stride, int batch,
                  int M, int N, int K, int epilogue, const void* resid, int64_t ldr,
                  int64_t resid_batch_stride, const void* gate, int64_t gate_ld,
                  b2f_stream_t stream);

/* Tiles: the forward GEMM runs on 128 x 128 tiles (two consumer warpgroups taking turns, so one tile's epilogue overlaps
 * the next tile's MMAs) or, for the large linears of the denoising loop, on 128 x 256 tiles (both warpgroups on one
 * tile, one m64n256k16 each per k16 step: fewer shared-memory and L2 bytes per FLOP).  b2f_gemm_bf16 and
 * b2f_gemm_qkv_norm_rope pick the tile per launch from the shape: the wide tile where its rounds of tiles over the SMs,
 * at the measured cost of a wide tile, finish first (the fused QKV epilogue also needs d_model % 256 == 0).  Both tiles
 * give bit-identical results.  The LoRA, FP8 and backward GEMMs always use 128 x 128.  The profiling tag of a launch
 * (b2f_prof_shapes) ends in " t128" or " t256".
 * b2f_gemm_set_tile_override is for tests and benchmarks only: 0 restores the automatic choice (the default), 128 or
 * 256 forces that tile on every later launch that supports it (process-wide, not thread-safe); anything else returns
 * B2F_ERR_INVALID. */
int b2f_gemm_set_tile_override(int tile_n);

/* Fused QKV projection of an MMDiT attention block: out[.., 3*d] = A · Wqkv^T + b with per-head
 * RMSNorm(eps, weight nw_q / nw_k) and interleaved-pair RoPE applied to the Q and K heads in the GEMM
 * epilogue (V passes through) — diffusers to_q/to_k/to_v + norm_q/norm_k + apply_rotary_emb in one
 * kernel (SURVEY.md A.2, §7.5).  cos/sin: fp32 [S,128]; token `row` of every batch item uses table row
 * rope_row0 + row (the image stream of a double block starts at S_txt).  Same rounding chain as
 * b2f_rmsnorm_rope.  Optional second output block: when n_extra > 0, W has 3*d_model + n_extra rows and
 * the extra columns are written to out_extra (pitch ld_extra) through epilogue epi_extra — the
 * single-stream block's [to_q;to_k;to_v;proj_mlp] runs as ONE launch, its GELU'd MLP part landing in
 * the [attn|mlp] buffer. */
int b2f_gemm_qkv_norm_rope(const void* A, int64_t lda, int64_t a_batch_stride, const void* W,
                           int64_t ldw, const void* bias, void* out, int64_t ldc,
                           int64_t out_batch_stride, int batch, int M, int d_model, int K,
                           const void* nw_q, const void* nw_k, const float* cos, const float* sin,
                           int rope_row0, float eps, int n_extra, void* out_extra, int64_t ld_extra,
                           int64_t extra_batch_stride, int epi_extra, b2f_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * LoRA (low-rank adapters) on the linear layers.  Replaces the PEFT LoraLayer forward / merge that diffusers'
 * FluxLoraLoaderMixin installs on FluxTransformer2DModel (reference univa/utils/flux_pipeline.py:30, 193-195 inherits
 * load_lora_weights / set_adapters / fuse_lora; the per-call scale is joint_attention_kwargs["scale"], :922-924).
 *
 * Adapters i = 1..n on one linear, of ranks r_i, are held concatenated: Acat [r_pad, in] (rows of every A_i),
 * Bcat [out, r_pad] (columns of every B_i), colscale fp32 [r_pad] (alpha_i / r_i x adapter weight_i on adapter i's
 * columns); r_pad = sum r_i rounded up to 64 with zero rows / columns / scales.  An unfused forward is two launches:
 *   down projection  T = bf16(fp32(X Acat^T)[:, k] * fp32(colscale[k] * s))           (b2f_gemm_colscale)
 *   K-extended GEMM  out = epilogue(fp32(X W^T + T Bcat^T) + bias)                    (b2f_gemm_bf16_lora)
 * where s is the call scale and the second launch accumulates both products into the same fp32 accumulators (r_pad/64
 * extra k-blocks per tile) before the unchanged epilogue.  Rounding chain: T is rounded to bf16 once; base and LoRA
 * products share one fp32 accumulation and the epilogue's roundings.  PEFT differs: it rounds the base output
 * bf16(X W^T + b) and the LoRA output bf16(bf16(bf16(X A^T) B^T) * scaling) separately and adds them in bf16 — so
 * outputs agree with PEFT to bf16 rounding, not bit for bit.
 */
/* b2f_gemm_bf16 (every forward epilogue, same arguments) with the contraction extended by T [batch, M, r_pad] (row pitch
 * ldt, batch pitch t_batch_stride) against Bcat [N, r_pad] (pitch ldbc); r_pad % 64 == 0, r_pad > 0. */
int b2f_gemm_bf16_lora(const void* A, int64_t lda, int64_t a_batch_stride, const void* W, int64_t ldw,
                       const void* bias, void* out, int64_t ldc, int64_t out_batch_stride, int batch,
                       int M, int N, int K, int epilogue, const void* resid, int64_t ldr,
                       int64_t resid_batch_stride, const void* gate, int64_t gate_ld, const void* T, int64_t ldt,
                       int64_t t_batch_stride, const void* Bcat, int64_t ldbc, int r_pad, b2f_stream_t stream);
/* b2f_gemm_qkv_norm_rope (including the n_extra second output block) with the same K-extension: the LoRA lands on the
 * projection before RMSNorm / RoPE / GELU, where PEFT adds it. */
int b2f_gemm_qkv_norm_rope_lora(const void* A, int64_t lda, int64_t a_batch_stride, const void* W,
                                int64_t ldw, const void* bias, void* out, int64_t ldc,
                                int64_t out_batch_stride, int batch, int M, int d_model, int K,
                                const void* nw_q, const void* nw_k, const float* cos, const float* sin,
                                int rope_row0, float eps, int n_extra, void* out_extra, int64_t ld_extra,
                                int64_t extra_batch_stride, int epi_extra, const void* T, int64_t ldt,
                                int64_t t_batch_stride, const void* Bcat, int64_t ldbc, int r_pad,
                                b2f_stream_t stream);
/* LoRA down projection: out[batch, M, N] = bf16(fp32(A W^T)[., n] * fp32(colscale[n] * cs_mul)), W = Acat [N, K],
 * colscale fp32 [N] (16-byte aligned).  The forward GEMM with N = r_pad and a per-column scale in its epilogue. */
int b2f_gemm_colscale(const void* A, int64_t lda, int64_t a_batch_stride, const void* W, int64_t ldw, void* out,
                      int64_t ldc, int64_t out_batch_stride, int batch, int M, int N, int K, const float* colscale,
                      float cs_mul, b2f_stream_t stream);
/* Merge in place: W[rows, cols] <- bf16(W + sum_{k<r} fp32(Bcat[:, k] * fp32(colscale[k] * cs_mul)) Acat[k, :]), one
 * fp32 accumulation in ascending k (fmaf) and one rounding (PEFT merge / diffusers fuse_lora).  Bcat [rows, r] (pitch
 * ldb), Acat [r, cols] (pitch lda).  Unfusing is the caller's: restore a saved copy of W. */
int b2f_lora_fuse(void* W, int64_t ldw, int rows, int cols, const void* Bcat, int64_t ldb, const void* Acat,
                  int64_t lda, const float* colscale, float cs_mul, int r, b2f_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * FP8 (e4m3) linear layers: per-token activation scales and per-output-channel weight scales (the scheme torchao calls
 * float8 dynamic activation / float8 weight, per row), computed by the FP8 tensor cores (wgmma ...e4m3.e4m3, fp32
 * accumulators).
 *
 * Row rule.  A bf16 row x[0..K) (a token's activations, or one output channel of a weight) becomes e4m3 bytes q and one
 * fp32 scale s:
 *   amax = max |x_i| (fp32, exact);
 *   amax == 0:  s = 1, every q_i = 0 (+0);
 *   otherwise   inv = 448.0f / amax, s = amax / 448.0f (IEEE fp32 divisions, round to nearest),
 *               q_i = e4m3(x_i * inv): one fp32 multiply, then round to nearest even saturating to +-448
 *               (cvt.rn.satfinite.e4m3x2.f32).
 * So x_i ~ s * q_i.  The CPU equivalent is (x.float() * inv).clamp(-448, 448).to(torch.float8_e4m3fn).
 *
 * GEMM.  acc[m, n] = sum_k qa[m, k] qw[n, k] in fp32 on the tensor cores; the staged value is
 *   x = bf16(fmaf(acc, fp32(sa[m] * sw[n]), bias[n]))      (bf16(acc * fp32(sa[m] * sw[n])) without a bias),
 * and from x on every epilogue is exactly b2f_gemm_bf16's / b2f_gemm_qkv_norm_rope's.  The tensor cores' fp32
 * accumulation of e4m3 products is not IEEE fp32 accumulation: tests/test_fp8_gpu.py states the measured allowance.
 */
/* x [batch, rows, K] bf16 (pitches in elements) -> q [batch, rows, K] e4m3 (pitches in bytes) and scale fp32
 * [batch, rows] (batch pitch scale_batch_stride).  K % 16 == 0; ldq, q_batch_stride multiples of 16. */
int b2f_quant_fp8_rows(const void* x, int64_t ldx, int64_t x_batch_stride, void* q, int64_t ldq, int64_t q_batch_stride,
                       float* scale, int64_t scale_batch_stride, int batch, int rows, int K, b2f_stream_t stream);
/* b2f_gemm_bf16 (every forward epilogue) with A [batch, M, K] e4m3 (pitches in bytes) scaled by a_scale fp32 [batch, M]
 * (batch pitch a_scale_batch_stride) and W [N, K] e4m3 scaled by w_scale fp32 [N] (16-byte aligned).  K, lda, ldw and
 * a_batch_stride are multiples of 16 (TMA). */
int b2f_gemm_fp8(const void* A, int64_t lda, int64_t a_batch_stride, const float* a_scale,
                 int64_t a_scale_batch_stride, const void* W, int64_t ldw, const float* w_scale, const void* bias,
                 void* out, int64_t ldc, int64_t out_batch_stride, int batch, int M, int N, int K, int epilogue,
                 const void* resid, int64_t ldr, int64_t resid_batch_stride, const void* gate, int64_t gate_ld,
                 b2f_stream_t stream);
/* b2f_gemm_qkv_norm_rope (including the n_extra second output block) with the operands of b2f_gemm_fp8. */
int b2f_gemm_qkv_norm_rope_fp8(const void* A, int64_t lda, int64_t a_batch_stride, const float* a_scale,
                               int64_t a_scale_batch_stride, const void* W, int64_t ldw, const float* w_scale,
                               const void* bias, void* out, int64_t ldc, int64_t out_batch_stride, int batch, int M,
                               int d_model, int K, const void* nw_q, const void* nw_k, const float* cos,
                               const float* sin, int rope_row0, float eps, int n_extra, void* out_extra,
                               int64_t ld_extra, int64_t extra_batch_stride, int epi_extra, b2f_stream_t stream);
/* FP8 with an unfused LoRA: b2f_gemm_fp8's operands plus b2f_gemm_bf16_lora's K-extension (T, Bcat in bf16, r_pad % 64
 * == 0, r_pad > 0).  The r_pad / 64 bf16 k-blocks follow the e4m3 ones in the same tile; before the first of them each
 * tile's accumulators are scaled in registers, so the staged value is
 *   x = bf16(fp32(acc8 * fp32(sa[m] * sw[n])) + T Bcat^T + bias[n])
 * with the LoRA products accumulated in fp32 onto the scaled e4m3 accumulator, and the epilogues run from x as
 * everywhere.  This differs from b2f_gemm_fp8's fmaf(acc, s, bias): an adapter with Bcat = 0 gives results within one
 * fp32 rounding of b2f_gemm_fp8's before the bf16 rounding, not bit-identical ones.  The adapter sees T, the bf16 down
 * projection of the linear's bf16 input (b2f_gemm_colscale), so it carries no e4m3 rounding of its own.  128 x 128
 * tiles. */
int b2f_gemm_fp8_lora(const void* A, int64_t lda, int64_t a_batch_stride, const float* a_scale,
                      int64_t a_scale_batch_stride, const void* W, int64_t ldw, const float* w_scale, const void* bias,
                      void* out, int64_t ldc, int64_t out_batch_stride, int batch, int M, int N, int K, int epilogue,
                      const void* resid, int64_t ldr, int64_t resid_batch_stride, const void* gate, int64_t gate_ld,
                      const void* T, int64_t ldt, int64_t t_batch_stride, const void* Bcat, int64_t ldbc, int r_pad,
                      b2f_stream_t stream);
/* b2f_gemm_qkv_norm_rope_fp8 with the K-extension of b2f_gemm_fp8_lora. */
int b2f_gemm_qkv_norm_rope_fp8_lora(const void* A, int64_t lda, int64_t a_batch_stride, const float* a_scale,
                                    int64_t a_scale_batch_stride, const void* W, int64_t ldw, const float* w_scale,
                                    const void* bias, void* out, int64_t ldc, int64_t out_batch_stride, int batch,
                                    int M, int d_model, int K, const void* nw_q, const void* nw_k, const float* cos,
                                    const float* sin, int rope_row0, float eps, int n_extra, void* out_extra,
                                    int64_t ld_extra, int64_t extra_batch_stride, int epi_extra, const void* T,
                                    int64_t ldt, int64_t t_batch_stride, const void* Bcat, int64_t ldbc, int r_pad,
                                    b2f_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * FP8 attention (head_dim 128, non-causal, no bias): b2f_attention_fwd's online softmax with Q / K / V in e4m3 on the
 * FP8 tensor cores (wgmma m64n128k32 e4m3, fp32 accumulators).
 *
 * Scales.  The row rule of "FP8 linear layers" above, unchanged, over a different unit of "row":
 *   Q, K   one scale per (batch item, head): the row is all S x 128 values of that head (after the per-head RMSNorm and
 *          RoPE their range is bounded by the norm weight, well inside e4m3's 2^14.8 normal span);
 *   V      one scale per (batch item, head, channel): the row is that channel's S values.
 * The range costs nothing, but e4m3 keeps 3 mantissa bits: each score carries a relative error of a few percent of
 * sum |q_i k_i|, which moves a peaked softmax row far more than a flat one.  With RMSNorm'd q / k under norm weights of
 * rms 2.5 (median row max p 0.6), S = 4641, the output is 13 % off in rel-L2 (bf16: 0.17 %); see README.
 * Buffers (contiguous): q8, k8 e4m3 [B, S, H*128] (the token-major layout of the bf16 inputs); sq, sk fp32 [B, H];
 * v8t e4m3 [B, H, 128, S_pad] with S_pad = S rounded up to 128 and tokens contiguous (FP8 wgmma takes K-major operands
 * only, and the token is the k dimension of P.V); sv fp32 [B, H, 128].  Padding tokens of v8t are +0.
 *
 * Token order of v8t.  Within every group of 32 tokens, k-position p holds token
 *   token(p) = (p & 16) + 2 ((p & 15) >> 2) + (p & 1) + 8 ((p >> 1) & 1)
 * i.e. with t = lane % 4, k-positions 4t..4t+3 hold tokens {2t, 2t+1, 8+2t, 9+2t} and 16+4t..16+4t+3 hold
 * {16+2t, 17+2t, 24+2t, 25+2t}.  That maps the fp32 accumulator layout of S = Q K^T (m64n128: a thread holds columns
 * 8j + 2t, 8j + 2t + 1) onto the register A fragment of the m64n128k32 e4m3 P.V wgmma (a thread holds k 4t..4t+3 and
 * 16+4t..16+4t+3), so P converts to e4m3 in place, without shuffles.
 *
 * Kernel arithmetic, per 128-token KV block in the order of attention.cu:
 *   c = fp32(fp32(sq * sk) * fp32(scale * log2 e)), the last product of the fp32 scale taken in double;  acc = Q8 K8^T (tensor cores, fp32);  m = running max of c * acc;
 *   p' = ex2(fmaf(acc, c, 8 - m)) = 256 p with p = 2^(t - m), t = c * acc (fp32; masked tail columns give p' = 0);
 *   l' = l' * ex2(m_old - m) + sum(p') (fp32 p', so l' = 256 l);  P8 = e4m3(p') (p' <= 256 never saturates);
 *   O = O * ex2(m_old - m) + P8 V8 (tensor cores, fp32; the rescale is skipped where every factor of a warp is 1),
 * and at the end, per channel c:  out = bf16((O[c] * sv[c]) * (1 / l')).
 * The factor 256 keeps p in e4m3's normal range; it sits in the exponent of ex2 rather than in a multiply, which the
 * softmax-bound kernel needs.  Up to fp32 rounding this is P8 = e4m3(256 p), out = O sv / (256 l).  The e4m3 products
 * are accumulated as the FP8 GEMM's are: tests/test_attn_fp8_gpu.py states the measured allowance.
 */
/* Quantize bf16 q / k / v (the pitched views of b2f_attention_fwd, Sq = Skv = S, H = Hkv heads) into the buffers above:
 * an amax pass (atomicMax on the bits of non-negative floats, so order-independent), a quantize / transpose pass and a
 * pass that turns the amaxes into scales (three launches).  NaN and zero inputs behave as in the row rule.  ldq / ldk /
 * ldv multiples of 8; q, k, v, q8, k8, v8t 16-byte aligned. */
int b2f_attn_quant_fp8(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* q8,
                       void* k8, float* sq, float* sk, void* v8t, float* sv, int B, int H, int S, int head_dim,
                       b2f_stream_t stream);
/* out [B, S, H*128] (row pitch ldo, a multiple of 8) = softmax(Q K^T * scale) V from the buffers of b2f_attn_quant_fp8.
 * head_dim != 128 or causal != 0: B2F_ERR_UNSUPPORTED. */
int b2f_attention_fp8(const void* q8, const void* k8, const float* sq, const float* sk, const void* v8t, const float* sv,
                      void* out, int64_t ldo, int B, int H, int S, int head_dim, float scale, int causal,
                      b2f_stream_t stream);
/* The FP8 pair with the per-item text window of b2f_attention_fwd_window (win int32 DEVICE [B, 2], 0 <= S_txt <= S).
 * The quantizer takes the Q / K amax of every head and the V amax of every channel over the valid tokens only, so an
 * item's sq / sk / sv are bit-equal to those of its valid tokens quantized alone (the amax is order-independent); it
 * writes masked tokens as +0 in q8, k8 and v8t.  The attention streams the 128-token blocks of the unwindowed kernel
 * that hold a valid key, skips the others (no load, no MMA), and gives masked keys p = 0 (against V = +0).  The full
 * window (0, S_txt) is bit-identical to b2f_attn_quant_fp8 + b2f_attention_fp8.  Masked query rows receive finite
 * values that mean nothing. */
int b2f_attn_quant_fp8_window(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv,
                              void* q8, void* k8, float* sq, float* sk, void* v8t, float* sv, int B, int H, int S,
                              int head_dim, const int32_t* win, int S_txt, b2f_stream_t stream);
int b2f_attention_fp8_window(const void* q8, const void* k8, const float* sq, const float* sk, const void* v8t,
                             const float* sv, void* out, int64_t ldo, int B, int H, int S, int head_dim, float scale,
                             const int32_t* win, int S_txt, b2f_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * AdaLN modulate (HBM-bound): out = LayerNorm(x; eps, no affine) * (1 + scale[b]) + shift[b].
 * Replaces nn.LayerNorm + the broadcast multiply/add of diffusers AdaLayerNormZero /
 * AdaLayerNormZeroSingle / AdaLayerNormContinuous and the norm2 modulate inside
 * FluxTransformerBlock (SURVEY.md A.1).  x/out: [batch, rows, D] views; scale/shift: [batch, D]
 * with pitch mod_ld.  D % 256 == 0, D <= 5120.  With split_row > 0, rows [0, split_row) of every batch
 * item use (scale, shift) and the remaining rows (scale_b, shift_b): the text and image streams of a
 * double-stream block share one launch over the joint [txt; img] buffer.
 */
int b2f_ln_modulate(const void* x, int64_t ldx, int64_t x_batch_stride, const void* scale,
                    const void* shift, int64_t mod_ld, void* out, int64_t ldo,
                    int64_t out_batch_stride, int batch, int rows, int D, float eps, int split_row,
                    const void* scale_b, const void* shift_b, b2f_stream_t stream);
/* b2f_ln_modulate whose bf16 result row goes through the FP8 row rule (b2f_quant_fp8_rows) instead of being stored: out
 * receives e4m3 bytes (pitches in bytes, multiples of 16) and row_scale fp32 [batch, rows] (batch pitch
 * row_scale_batch_stride) the row scales.  Bit-identical to b2f_ln_modulate followed by b2f_quant_fp8_rows.
 * D % 256 == 0, D <= 3072. */
int b2f_ln_modulate_fp8(const void* x, int64_t ldx, int64_t x_batch_stride, const void* scale, const void* shift,
                        int64_t mod_ld, void* out, int64_t ldo, int64_t out_batch_stride, float* row_scale,
                        int64_t row_scale_batch_stride, int batch, int rows, int D, float eps, int split_row,
                        const void* scale_b, const void* shift_b, b2f_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Per-head RMSNorm + interleaved-pair RoPE, in place on the Q and K blocks of a fused QKV buffer
 * (HBM-bound).  Replaces diffusers RMSNorm (attn.norm_q/norm_k/norm_added_q/norm_added_k) and
 * apply_rotary_emb(use_real_unbind_dim=-1) in FluxAttnProcessor2_0 (SURVEY.md A.2).
 * q, k: pointers to head 0 of token 0 (token pitch ld, batch pitch batch_stride); H heads of 128.
 * Tokens [0, n_a) of each batch item use weights (wq_a, wk_a) — the text stream's
 * norm_added_q/k — the rest use (wq_b, wk_b).  cos/sin: fp32 [S, 128] (FluxPosEmbed layout).
 */
int b2f_rmsnorm_rope(void* q, void* k, int64_t ld, int64_t batch_stride, const void* wq_a,
                     const void* wk_a, const void* wq_b, const void* wk_b, const float* cos,
                     const float* sin, int batch, int S, int H, int head_dim, int n_a, float eps,
                     b2f_stream_t stream);

/* Flow-matching Euler update x <- bf16(float(x) + bf16(bf16(dt) * v)), in place (replaces
 * FlowMatchEulerDiscreteScheduler.step, reference call site univa/utils/flux_pipeline.py:1099). */
int b2f_euler_step(void* x, int64_t ldx, const void* v, int64_t ldv, int64_t rows, int cols,
                   float dt, b2f_stream_t stream);

/* FluxPosEmbed: 3-axis RoPE tables from token ids.  ids: fp32 DEVICE [S,3] (text ids first, then
 * image ids: (image index, row, col), reference univa/utils/flux_pipeline.py:561-572, 694-698);
 * axes_dim = {16,56,56}; angles in float64, output fp32 [S,128] with each pair value repeated
 * (diffusers get_1d_rotary_pos_embed(repeat_interleave_real=True), SURVEY.md A.2). */
int b2f_rope_tables(const float* ids, int S, const int* axes_dim, double theta, float* cos,
                    float* sin, b2f_stream_t stream);

/* y = silu(x) over n contiguous bf16 elements (n % 8 == 0): the nn.SiLU in front of every AdaLN
 * linear (SURVEY.md A.1). */
int b2f_silu(const void* x, void* y, int64_t n, b2f_stream_t stream);

/* The two row kernels of b2f_flux_temb, exposed on their own so they can be checked element by element.
 * Timestep projection (Timesteps(256, flip_sin_to_cos=True, shift 0)): t fp32 DEVICE [rows] ->
 * out bf16 [rows, 256] = [cos(t f) | sin(t f)], f_j = exp(-ln(10000) j / 128), fp32 math.
 * Combine: temb = bf16(bf16(t + g) + txt) (g may be null: bf16(t + txt)), silu_temb = bf16(silu(temb)),
 * all bf16 contiguous of n elements (n % 8 == 0). */
int b2f_temb_sinusoid(const float* t, void* out, int rows, b2f_stream_t stream);
int b2f_temb_combine(const void* t, const void* g, const void* txt, void* temb, void* silu_temb, int64_t n,
                     b2f_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Fused softmax attention, head_dim 128:  O = softmax(Q K^T * scale [+ causal mask]) V.
 * wgmma QK^T and PV with S/P/O in registers, K/V streamed by TMA, online softmax (FA-style).
 * Replaces F.scaled_dot_product_attention in diffusers' FluxAttnProcessor2_0 (joint [txt;img]
 * attention of FluxTransformerBlock / FluxSingleTransformerBlock, SURVEY.md A.2; reference call
 * site univa/utils/flux_pipeline.py:1067) and flash_attn reached through
 * attn_implementation="flash_attention_2" (univa/serve/cli.py:40) for the Qwen2.5-VL prefill.
 *
 * Layout: token-major.  q points at element [b=0, s=0, head 0, 0]; head h of token s of batch b
 * is at q + (b*Sq + s)*ldq + h*128 (same for k, v with Skv, ldk/ldv and Hkv heads; GQA maps
 * query head h to kv head h / (H/Hkv)).  out is [B, Sq, H*128] with row pitch ldo.  This lets
 * Q/K/V be column slices of one fused QKV projection buffer and lets out be a column slice of
 * the single-stream [attn | mlp] buffer — no transposes or concatenations.
 * causal != 0 requires Sq == Skv.
 */
int b2f_attention_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v,
                      int64_t ldv, void* out, int64_t ldo, int B, int H, int Hkv, int Sq, int Skv,
                      int head_dim, float scale, int causal, b2f_stream_t stream);

/* Non-causal b2f_attention_fwd with a per-item text window: the first S_txt keys of every item are its text (0 <= S_txt
 * <= Skv), win int32 DEVICE [B, 2] holds (lo, hi) per item, and key k of item b is valid iff k >= S_txt or
 * lo <= k < hi (values outside 0 <= lo <= hi <= S_txt are clamped into that range).  Invalid keys never reach an
 * output: the K/V blocks of 128 rows start at lo and cover [lo, Skv) when hi == S_txt, else [lo, hi) and then
 * [S_txt, Skv), so blocks wholly outside the window are never loaded; within a block masked keys get p = 0, and pad
 * V rows [hi, S_txt) sharing a block with valid keys are zeroed in shared memory first, so NaN or Inf there cannot
 * reach P.V.  For hi == S_txt an item sees the blocks, in order and in the same positions, of its valid keys run alone
 * (up to where its query rows sit); the full window (0, S_txt) is bit-identical to b2f_attention_fwd.  Rows of masked
 * queries are computed like any other and mean nothing. */
int b2f_attention_fwd_window(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v,
                             int64_t ldv, void* out, int64_t ldo, int B, int H, int Hkv, int Sq, int Skv,
                             int head_dim, float scale, const int32_t* win, int S_txt, b2f_stream_t stream);

/* Same kernel with an additive score bias: softmax(scale * q.k^T + bias[h]) v, bias bf16 with
 * element [h, s_q, s_kv] at bias + h*bias_h_stride + s_q*bias_row_stride + s_kv (shared by the
 * batch).  Replaces T5Attention's eager `scores += position_bias` path (transformers T5, scale = 1)
 * reached from encode_prompt — reference univa/utils/denoiser_prompt_embedding_flux.py:44. */
int b2f_attention_bias_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v,
                           int64_t ldv, void* out, int64_t ldo, int B, int H, int Hkv, int Sq, int Skv,
                           int head_dim, float scale, int causal, const void* bias,
                           int64_t bias_h_stride, int64_t bias_row_stride, b2f_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Kernels of the T5-XXL / CLIP-L prompt encoders (transformers T5EncoderModel / CLIPTextModel as
 * called by encode_prompt, reference univa/utils/denoiser_prompt_embedding_flux.py:15-104).
 */
/* T5DenseGatedActDense combine: out = bf16(bf16(gelu_tanh(gu[:, :I])) * gu[:, I:2I]). */
int b2f_geglu(const void* gu, int64_t ld, void* out, int64_t ldo, int64_t rows, int I,
              b2f_stream_t stream);
/* nn.LayerNorm with weight and bias, fp32 statistics; D % 256 == 0, D <= 5120. */
int b2f_layernorm(const void* x, int64_t ldx, const void* w, const void* b, void* y, int64_t ldy,
                  int64_t rows, int D, float eps, b2f_stream_t stream);
/* out[i] = bf16(tok[ids[i]] + pos[i % period]) (CLIPTextEmbeddings); pos == NULL: plain lookup
 * (T5 `shared`).  ids: int64 device array, D % 8 == 0. */
int b2f_embed(const void* tok, int64_t ld_tok, const int64_t* ids, const void* pos, int64_t ld_pos,
              int period, void* out, int64_t ldo, int64_t n, int D, b2f_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * FLUX-Kontext MMDiT (diffusers FluxTransformer2DModel) as one object.
 * Replaces `pipe.transformer(...)` — reference call sites univa/utils/flux_pipeline.py:1067-1077,
 * univa/models/modeling_univa_denoise_tower.py:103-110, modeling_univa_qwen2p5vl.py:352-355.
 *
 * Weights are BORROWED device pointers (bf16) bound by name.  Names are the diffusers state-dict
 * keys (SURVEY.md A.6) except that projections which this engine runs as one GEMM are bound as
 * one row-concatenated tensor (the Python side stores them fused and exposes the diffusers names
 * as views, so checkpoints interchange):
 *   transformer_blocks.{i}.attn.qkv.{weight,bias}       rows [to_q; to_k; to_v]               [3d, d]
 *   transformer_blocks.{i}.attn.add_qkv.{weight,bias}   rows [add_q_proj; add_k_proj; add_v_proj]
 *   single_transformer_blocks.{i}.qkv_mlp.{weight,bias} rows [to_q; to_k; to_v; proj_mlp]     [7d, d]
 *   adaln.{weight,bias}   rows, in order: for each double block i [norm1.linear (6d);
 *                         norm1_context.linear (6d)], for each single block [norm.linear (3d)],
 *                         then norm_out.linear (2d)                              [mod_width, d]
 * All other keys keep their diffusers names (x_embedder, context_embedder, time_text_embed.*,
 * attn.to_out.0, attn.to_add_out, attn.norm_*.weight, ff.net.0.proj, ff.net.2, ff_context.*,
 * single proj_out, proj_out).
 */
typedef struct b2f_flux b2f_flux;
typedef struct {
  int num_heads;      /* 24 */
  int head_dim;       /* 128 (only value supported) */
  int num_double;     /* 19 */
  int num_single;     /* 38 */
  int in_channels;    /* 64 */
  int out_channels;   /* 64 */
  int joint_dim;      /* 4096 */
  int pooled_dim;     /* 768 */
  int guidance_embeds;/* 1 */
  int mlp_ratio;      /* 4 */
} b2f_flux_cfg;

int b2f_flux_create(b2f_flux** out, const b2f_flux_cfg* cfg);
void b2f_flux_destroy(b2f_flux* ctx);
int b2f_flux_bind_weight(b2f_flux* ctx, const char* key, const void* dptr, int64_t numel);
/* Checks that every weight is bound with the right element count. */
int b2f_flux_finalize(b2f_flux* ctx);
/* Columns of one modulation row = rows of adaln.weight. */
int64_t b2f_flux_mod_width(const b2f_flux* ctx);
/* RoPE tables (FluxPosEmbed output, fp32 [S_txt+S_img, 128], text rows first); borrowed. */
int b2f_flux_set_rope(b2f_flux* ctx, const float* cos, const float* sin, int S);
size_t b2f_flux_workspace_bytes(const b2f_flux* ctx, int B, int S_img, int S_txt);
size_t b2f_flux_temb_workspace_bytes(const b2f_flux* ctx, int rows);
/* CombinedTimestepGuidanceTextProjEmbeddings (SURVEY.md A.3) for `rows` (step, batch) pairs:
 * timestep/guidance are fp32 DEVICE arrays already multiplied by 1000 in the reference's bf16
 * arithmetic; pooled is bf16 [rows, pooled_dim].  Writes temb and silu(temb), bf16 [rows, d]. */
int b2f_flux_temb(b2f_flux* ctx, const float* timestep, const float* guidance, const void* pooled,
                  int64_t pooled_ld, int rows, void* temb, void* silu_temb, void* ws,
                  size_t ws_bytes, b2f_stream_t stream);
/* Every AdaLN linear of the model in ONE weight-streaming GEMM:
 * mod[rows, mod_width] = silu_temb[rows, d] · adaln.weight^T + adaln.bias.  Hoistable over the
 * whole sampling schedule (rows = steps * batch): the modulation depends only on (t, guidance,
 * pooled), so the 6.46 GB of AdaLN weights are read once per image instead of once per step. */
int b2f_flux_modulation(b2f_flux* ctx, const void* silu_temb, int rows, void* mod,
                        b2f_stream_t stream);
/* Unfused LoRA adapters (diffusers load_lora_weights / set_adapters, see b2f_gemm_bf16_lora): bind (Acat, Bcat, colscale)
 * of r_pad ranks (multiple of 64; borrowed device pointers) to one linear; Acat == NULL unbinds it.  Targets: every
 * linear bound by b2f_flux_bind_weight under its bound name (transformer_blocks.{i}.attn.qkv / attn.add_qkv,
 * single_transformer_blocks.{i}.qkv_mlp, attn.to_out.0, ff.net.2, x_embedder, time_text_embed.*.linear_{1,2},
 * proj_out, ...), and each AdaLN linear under its diffusers name (transformer_blocks.{i}.norm1.linear,
 * norm1_context.linear, single_transformer_blocks.{i}.norm.linear, norm_out.linear): those act on their rows of the
 * fused adaln weight only, through their own K-extended launch in b2f_flux_modulation_ws.  Bindings are dropped by
 * b2f_flux_finalize.  With any adapter bound b2f_flux_workspace_bytes / b2f_flux_temb_workspace_bytes add room for
 * T ([rows, largest r_pad]); without one they are unchanged.  The training step refuses while adapters are bound. */
int b2f_flux_bind_lora(b2f_flux* ctx, const char* target, const void* Acat, const void* Bcat, const float* colscale,
                       int r_pad);
int b2f_flux_clear_lora(b2f_flux* ctx);
/* Call scale s multiplying every colscale (joint_attention_kwargs["scale"]); read when a forward is enqueued. */
int b2f_flux_set_lora_scale(b2f_flux* ctx, float scale);
/* Largest bound r_pad (0: no adapter bound). */
int b2f_flux_lora_rank(const b2f_flux* ctx);
/* b2f_flux_modulation with the AdaLN adapters applied (b2f_flux_modulation itself refuses while one is bound). */
size_t b2f_flux_modulation_workspace_bytes(const b2f_flux* ctx, int rows);
int b2f_flux_modulation_ws(b2f_flux* ctx, const void* silu_temb, int rows, void* mod, void* ws, size_t ws_bytes,
                           b2f_stream_t stream);
/* One MMDiT forward.  hidden [B,S_img,in_channels], enc [B,S_txt,joint_dim], mod: pointer to the
 * first batch item's modulation row (pitch mod_ld between batch items), out
 * [B,n_out_rows,out_channels] (the first n_out_rows image tokens; the pipeline only consumes the
 * target tokens, flux_pipeline.py:1078).  Blocks [first_block, last_block) of the 57 run; pass
 * (0, -1) for the whole model — partial ranges exist for block-level parity tests (the embedders
 * run iff first_block == 0, norm_out/proj_out iff last_block covers the last block; activations
 * persist in ws between calls).  No allocation, no host synchronisation: graph-capturable. */
int b2f_flux_forward(b2f_flux* ctx, const void* hidden, const void* enc, const void* mod,
                     int64_t mod_ld, void* out, int B, int S_img, int S_txt, int n_out_rows,
                     void* ws, size_t ws_bytes, int first_block, int last_block,
                     b2f_stream_t stream);
/* Per-item text windows for batches of instructions of different lengths: win_dev int32 DEVICE [B, 2] (borrowed, read
 * when a forward runs) holds (lo, hi) per batch item; text token k of item b takes part iff lo <= k < hi, and each item
 * then computes what it computes alone on its text rows [lo, hi).  b2f_flux_forward and b2f_flux_forward_cached run
 * every block attention through b2f_attention_fwd_window (or the FP8 window pair) while it is set; the windows are not
 * read on the host, so a forward stays graph-capturable.  Every other stage of a block works row by row, so pad rows
 * need nothing else: their content, NaN included, stays in pad rows.  The first-block cache measures image rows
 * only.  A forward whose B differs from the window's B returns B2F_ERR_INVALID; b2f_flux_train_forward returns
 * B2F_ERR_UNSUPPORTED while a window is set.  win_dev NULL (or B <= 0 with NULL) switches windows off; b2f_flux_finalize
 * does too. */
int b2f_flux_set_text_window(b2f_flux* ctx, const int32_t* win_dev, int B);
/* FP8 block linears (see b2f_gemm_fp8).  b2f_flux_bind_fp8 binds the e4m3 copy w8 [out, in] of one block linear and its
 * fp32 per-channel scales w_scale [out] (borrowed; made by b2f_quant_fp8_rows from the bf16 weight) under the linear's
 * bound name (transformer_blocks.{i}.attn.qkv / attn.add_qkv / attn.to_out.0 / attn.to_add_out / ff.net.0.proj /
 * ff.net.2 / ff_context.net.0.proj / ff_context.net.2, single_transformer_blocks.{i}.qkv_mlp / proj_out); numel =
 * out * in; w8 == NULL unbinds.  b2f_flux_set_fp8(ctx, 1) makes b2f_flux_forward run those ten linears per block in FP8:
 * it requires every one to be bound and no LoRA adapter to be bound (b2f_flux_bind_lora is refused while FP8 is on;
 * fuse adapters first).  b2f_flux_set_fp8(ctx, 2) is the same with unfused adapters accepted: b2f_flux_bind_lora binds,
 * and a block linear with an adapter runs b2f_gemm_colscale on its bf16 input, then b2f_gemm_fp8_lora /
 * b2f_gemm_qkv_norm_rope_fp8_lora.  The bf16 inputs of to_out / to_add_out / ff.net.2 / ff_context.net.2 / proj_out
 * already exist (the cat buffer); for a LayerNorm whose output feeds an adapted linear the block also runs
 * b2f_ln_modulate into xn.  Linears without an adapter run exactly as in mode 1.  Every other linear (embedders, AdaLN, norm_out / proj_out) stays bf16, and so does attention
 * unless b2f_flux_set_fp8_attention is on.  The
 * inputs are quantized per token: the block's modulated LayerNorms by b2f_ln_modulate_fp8, the attention output
 * (input of to_out / to_add_out), the MLP activations (ff.net.2 / ff_context.net.2) and the single block's [attn | mlp]
 * (proj_out) by one b2f_quant_fp8_rows launch each over all tokens.  While FP8 is on b2f_flux_workspace_bytes adds an
 * e4m3 [B, S, 5d] buffer and an fp32 [B, S] scale vector, the blocks leave the workspace's xn rows unwritten, and the
 * training entry points refuse.  b2f_flux_finalize drops the FP8 bindings and switches FP8 off. */
int b2f_flux_bind_fp8(b2f_flux* ctx, const char* name, const void* w8, const float* w_scale, int64_t numel);
int b2f_flux_set_fp8(b2f_flux* ctx, int mode);
/* FP8 attention, independent of b2f_flux_set_fp8: while on, the double and single blocks quantize Q / K / V with
 * b2f_attn_quant_fp8 and run b2f_attention_fp8 where they run b2f_attention_fwd.  b2f_flux_workspace_bytes then adds
 * q8, k8, v8t and their scales, and the training entry points refuse.  Unfused LoRA adapters stay allowed (they act on
 * the linears only).  b2f_flux_finalize switches it off. */
int b2f_flux_set_fp8_attention(b2f_flux* ctx, int on);

/* First-block cache (opt-in; the approach of ParaAttention's FBCache / diffusers' FirstBlockCacheConfig, with this
 * engine's own semantics and rounding points).  Consecutive Euler steps change the hidden states little, so when block
 * 0's residual barely moved since the last step that ran in full, blocks 1..nblk-1 are skipped and their residual from
 * that step is reused.  An approximation: how often it hits and what it does to images depend on the checkpoint.
 *
 * A cached forward on cache state C (full block range only):
 *   1. Head.  The embedders and block 0 run exactly as in b2f_flux_forward.  x0 = the image-stream rows of h after
 *      x_embedder (all S_img rows, target and context, bf16), y0 = the same rows after block 0,
 *      r_k = float(y0) - float(x0) in fp32.
 *   2. Distance.  If C holds a full step with the same (ctx, B, S_img, S_txt, n_out_rows):
 *        dist = sum |r_k - r_prev| / sum |r_prev|   over all B * S_img * d elements, pooled over the batch,
 *      summed in a fixed order: fp32 per thread over its elements, the 256 threads of a CTA (8 rows each) by a fixed
 *      fp64 tree, then the per-CTA partials in fp64 (each thread of one CTA over CTAs t, t + 256, ... in index order,
 *      then a fixed tree), dist = fp32(num / den).  No float atomics: dist is bit-reproducible run to run.
 *   3. Hit iff dist < threshold (strict: threshold 0 never hits).  NaN or infinite dist is a miss, and so is
 *      sum |r_prev| == 0.  A call without a valid state is a miss.
 *   4. Hit.  Blocks 1..nblk-1 are skipped; h' = bf16(float(y0[:n_out]) + R) (round to nearest) is written over the
 *      first n_out_rows image rows of h, and norm_out / proj_out run on it exactly as the uncached tail runs on the final
 *      h (so the sum is rounded to bf16 before the LayerNorm statistics).  C is left unchanged: the next step is
 *      compared with the last FULL step, not with this one.
 *   5. Miss.  Blocks 1..nblk-1 and the tail run unchanged: the output is bit-identical to b2f_flux_forward's.  Then
 *      R = float(h_final[:n_out]) - float(y0[:n_out]) (fp32), r_prev = r_k (fp32), and C records the shapes.
 * The decision is taken for the whole batch: with the cache on, an item's result can depend on its batch-mates.
 *
 * Memory.  The caller owns all of it; nothing is allocated inside the forward.  b2f_flux_cache_bytes gives the size
 * for one shape (0 for an invalid one):
 *   2 x 4 B S_img d (r, two slots) + 4 B n_out d (R) + 16 ceil(B S_img / 8) (partials) + 2 B S_img d (x0 / y0 scratch)
 * plus 256-byte alignment of each region: about 100.7 + 100.7 + 50.3 + 50.3 MB at 1024^2, B = 1 (d 3072, S_img 8192,
 * n_out 4096).  Regions, in order from mem's first 256-aligned byte, each starting 256-aligned: r slot 0, r slot 1, R
 * [B, n_out, d], partials, an 8-byte decision, the scratch (x0, overwritten with y0 by the distance pass).
 * b2f_flux_cache_create makes a state over mem (borrowed) and allocates 8 bytes of pinned host memory for the
 * decision; a state holds shapes up to its bytes.  b2f_flux_cache_reset invalidates it (the next call misses): do so
 * whenever what the blocks compute changes (weights, adapters, LoRA scale, FP8 switches).  A call with other shapes
 * than the state's invalidates it itself.  b2f_flux_cache_state reports whether the state is valid and which r slot
 * holds r_prev (the other one holds the r_k of a call that hit).
 *
 * b2f_flux_forward_cached takes b2f_flux_forward's arguments minus the block range.  It is the one entry point that
 * waits on the device: with a valid state it reads (dist, hit) back, 8 bytes, and synchronises the stream once per
 * call, so it cannot be captured into a CUDA graph (b2f_flux_forward stays capturable).  *hit and *dist receive the
 * decision (dist NaN when there was no valid state).  threshold < 0 or NaN: B2F_ERR_INVALID; +inf is allowed and means
 * "hit whenever there is a state". */
typedef struct b2f_flux_cache b2f_flux_cache;
size_t b2f_flux_cache_bytes(const b2f_flux* ctx, int B, int S_img, int S_txt, int n_out_rows);
int b2f_flux_cache_create(b2f_flux_cache** out, void* mem, size_t bytes);
void b2f_flux_cache_destroy(b2f_flux_cache* cache);
int b2f_flux_cache_reset(b2f_flux_cache* cache);
int b2f_flux_cache_state(const b2f_flux_cache* cache, int* valid, int* r_slot);
int b2f_flux_forward_cached(b2f_flux* ctx, b2f_flux_cache* cache, float threshold, const void* hidden, const void* enc,
                            const void* mod, int64_t mod_ld, void* out, int B, int S_img, int S_txt, int n_out_rows,
                            void* ws, size_t ws_bytes, int* hit, float* dist, b2f_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Kernels of the Qwen2.5-VL conditioning prefill (transformers Qwen2_5_VL*, SURVEY.md Appendix B;
 * reference univa/models/qwen2p5vl/modeling_univa_qwen2p5vl.py:373-399, 481-492, 521-523).
 */
/* Qwen2RMSNorm: y = w * bf16(float(x) * rsqrt(mean(x^2) + eps)); D % 256 == 0, D <= 5120. */
int b2f_rmsnorm(const void* x, int64_t ldx, const void* w, void* y, int64_t ldy, int64_t rows, int D,
                float eps, b2f_stream_t stream);
/* rotate-half RoPE in place on `heads` head vectors per token (slot pitch head_pitch, first `rot`
 * elements rotated; cos/sin fp32 [tokens, rot]).  fp32_math=1: vision tower (one rounding);
 * fp32_math=0: text M-RoPE evaluated in bf16 as transformers' eager code does. */
int b2f_rope_half(void* x, int64_t ld, int heads, int head_pitch, const float* cos, const float* sin,
                  int rot, int64_t tokens, int fp32_math, b2f_stream_t stream);
/* SwiGLU combine: out = bf16(bf16(silu(gu[:, :I])) * gu[:, I:2I]). */
int b2f_swiglu(const void* gu, int64_t ld, void* out, int64_t ldo, int64_t rows, int I,
               b2f_stream_t stream);
/* Row gather (scatter=0: dst[i] = src[idx[i]], embed_tokens) / scatter (scatter=1: dst[idx[i]] =
 * src[i], masked_scatter of the image embeddings); idx: int64 device array, D % 8 == 0. */
int b2f_move_rows(const void* src, int64_t ld_src, void* dst, int64_t ld_dst, const int64_t* idx,
                  int64_t n, int D, int scatter, b2f_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * 3x3 convolution, NHWC bf16, wgmma implicit GEMM (A tiles are shifted 4-D TMA boxes of the
 * input; padding = TMA zero fill).  Replaces cuDNN conv as reached by diffusers AutoencoderKL
 * (SURVEY.md A.4).  in [N,Hin,Win,Cin] (Cin % 64 == 0), w OHWI [Cout,3,3,Cin], bias [>=8] bf16 or
 * NULL, out [N,Ho,Wo,Cout] (NHWC) or, with out_nchw, [N,Cout,Ho,Wo].  stride 1: padding 1.
 * stride 2: diffusers Downsample2D (pad right/bottom by one, no other padding), Ho = Hin/2.
 * resid (NHWC, same shape as out, may alias out): out = bf16(resid + bf16(conv + bias)).
 * out_nchw: 0 NHWC bf16, 1 planar [N,Cout,Ho,Wo] bf16, 2 uint8 pixels [N,Ho,Wo,Cout] = round(clamp(x/2 + 0.5, 0, 1) * 255).
 */
int b2f_conv3x3(const void* in, const void* w, const void* bias, void* out, const void* resid, int N,
                int Hin, int Win, int Cin, int Cout, int stride, int out_nchw, b2f_stream_t stream);

/* GroupNorm(32 groups, eps, affine) [+ SiLU] over x [N, P, C] (P = H*W, NHWC), HBM-bound two-pass.
 * stats_ws: device scratch of 64*N doubles.  Replaces nn.GroupNorm + nn.SiLU in ResnetBlock2D /
 * the mid-block Attention.group_norm / conv_norm_out (SURVEY.md A.4). */
int b2f_groupnorm_silu(const void* x, const void* gamma, const void* beta, void* y, void* stats_ws,
                       int N, int64_t P, int C, float eps, int silu, b2f_stream_t stream);
/* Nearest-neighbour 2x upsample, NHWC (Upsample2D's F.interpolate). */
int b2f_upsample2x(const void* in, void* out, int N, int H, int W, int C, b2f_stream_t stream);
/* NCHW (bf16, or fp32 when in_is_f32) -> NHWC bf16 with channels zero-padded to Cpad. */
int b2f_nchw_to_nhwc_pad(const void* in, int in_is_f32, void* out, int N, int C, int H, int W,
                         int Cpad, b2f_stream_t stream);
/* In-place row softmax p = softmax(scale * s) over rows of length L (bf16, fp32 math).  Any L >= 1; the pitch ld must be
 * a multiple of 8 and at least round_up(L, 8): columns [L, round_up(L, 8)) of every row are written as zeros, columns
 * past that are not touched. */
int b2f_softmax_rows(void* s, int64_t ld, int rows, int L, float scale, b2f_stream_t stream);
/* The same from fp32 scores s [rows, lds] into bf16 p [rows, ldp] (no rounding of the logits); same rules on L and the
 * pitches, 16-byte aligned s and p. */
int b2f_softmax_rows_f32(const void* s, int64_t lds, void* p, int64_t ldp, int rows, int L, float scale,
                         b2f_stream_t stream);
/* out[c, r] = in[r, c] for an [R, Cc] bf16 matrix. */
int b2f_transpose_bf16(const void* in, int64_t ld_in, void* out, int64_t ld_out, int R, int Cc,
                       b2f_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Stage-2 training step (reference train_denoiser.py:829-1181; trainable set :71-119; AdamW :596-602;
 * clip_grad_norm_ :1174-1177; ZeRO-2 sharding scripts/accelerate_configs/zero2.json).  The reference reaches all of
 * this through torch.autograd over diffusers' eager modules; here every backward op is its own kernel.
 * Activations and activation gradients are bf16, weight gradients and token reductions fp32.
 */
/* Backward-data GEMM of nn.Linear: dX[batch, M, N] = epi(dY[batch, M, K] · W[K, N]) with W as stored ([out = K, in = N],
 * read as an MN-major wgmma operand: no transposed copy).  epilogue: B2F_EPI_BIAS (store), B2F_EPI_DGELU /
 * B2F_EPI_DSILU (times act'(aux), aux = saved pre-activation [batch, M, N]), B2F_EPI_RESID (dX = aux + result). */
int b2f_gemm_dgrad(const void* dY, int64_t ldy, int64_t dy_batch_stride, const void* W, int64_t ldw, void* dX,
                   int64_t ldx, int64_t dx_batch_stride, int batch, int M, int N, int K, int epilogue, const void* aux,
                   int64_t ld_aux, int64_t aux_batch_stride, b2f_stream_t stream);
/* Backward-weight GEMM: dW[M, N] (+)= sum_b dY[b, :rows, :M]^T · X[b, :rows, :N], fp32 output (pitch ldw floats); both
 * operands are token-major activations read as MN-major wgmma operands. */
int b2f_gemm_wgrad(const void* dY, int64_t ldy, int64_t dy_batch_stride, const void* X, int64_t ldx,
                   int64_t x_batch_stride, float* dW, int64_t ldw, int batch, int rows, int M, int N, int accumulate,
                   b2f_stream_t stream);
/* b2f_attention_fwd that also writes lse2[b, h, q] = log2(sum_k exp2(scale*log2(e) * q.k)) at
 * lse + (b*H + h)*lse_stride + q (lse_stride >= Sq; use a multiple of 128 for the backward). */
int b2f_attention_fwd_lse(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* out,
                          int64_t ldo, int B, int H, int Hkv, int Sq, int Skv, int head_dim, float scale, int causal,
                          float* lse, int64_t lse_stride, b2f_stream_t stream);
/* delta[b, h, s] = sum_c dO * O for s < S; delta = 0 and lse = +inf for S <= s < S_pad (padding the backward relies on).
 * delta / lse: fp32 [B, H, S_pad]. */
int b2f_attn_delta(const void* o, int64_t ldo, const void* dout, int64_t lddo, float* delta, float* lse, int B, int H,
                   int S, int S_pad, b2f_stream_t stream);
/* Attention backward (non-causal, H == Hkv, head_dim 128): dq, dk, dv from q, k, v, dout, lse2 and delta.  Two
 * wgmma kernels (dK/dV with the scores held transposed in registers; dQ), no atomics: bit-reproducible.  All tensors
 * token-major [B, S, H*128] views.  S_pad: pitch of the lse / delta rows, a multiple of 128. */
int b2f_attention_bwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv,
                      const void* dout, int64_t lddo, const float* lse, const float* delta, int64_t S_pad, void* dq,
                      int64_t lddq, void* dk, int64_t lddk, void* dv, int64_t lddv, int B, int H, int S, int head_dim,
                      float scale, b2f_stream_t stream);
/* Row chunking of the column-reduction kernels below: partial buffers hold one fp32 row per chunk. */
int b2f_train_chunks(int rows);
int b2f_train_ln_chunks(int rows);
/* out = bf16(x + bf16(gate[b] * y)) over [batch, rows, D] views (the GATE_RESID epilogue unfused: training keeps y). */
int b2f_gate_resid_fwd(const void* x, int64_t ldx, int64_t x_bs, const void* y, int64_t ldy, int64_t y_bs,
                       const void* gate, const void* gate_b, int64_t gate_ld, void* out, int64_t ldo, int64_t o_bs,
                       int batch, int rows, int D, int split_row, b2f_stream_t stream);
/* dy = bf16(gate[b] * dout) (dy / gate may be NULL) and per-chunk column sums of dout*y (y NULL: of dout) over rows
 * >= part_row0 into partial[batch, b2f_train_chunks(rows), D] (NULL: none).  Bias, gate gradients. */
int b2f_gate_bwd(const void* dout, int64_t ldd, int64_t d_bs, const void* y, int64_t ldy, int64_t y_bs, const void* gate,
                 const void* gate_b, int64_t gate_ld, void* dy, int64_t ldo, int64_t o_bs, float* partial, int batch,
                 int rows, int D, int split_row, int part_row0, b2f_stream_t stream);
/* out[b, c] (+)= sum_k partial[b, k, c] in a fixed order. */
int b2f_col_reduce(const float* partial, int nchunks, int D, float* out, int64_t out_ld, int batch, int accumulate,
                   b2f_stream_t stream);
/* Backward of b2f_ln_modulate: dres_out = bf16(dres_in + bf16(dx)); per-chunk column sums (dscale | dshift) over rows
 * >= part_row0 into partial[batch, b2f_train_ln_chunks(rows), 2*D] (NULL: none).  dres_in may be NULL or alias dres_out. */
int b2f_ln_modulate_bwd(const void* x, int64_t ldx, int64_t x_bs, const void* dy, int64_t ldy, int64_t dy_bs,
                        const void* scale, const void* scale_b, int64_t mod_ld, const void* dres_in, int64_t ldr,
                        int64_t r_bs, void* dres_out, int64_t ldo, int64_t o_bs, float* partial, int batch, int rows,
                        int D, float eps, int split_row, int part_row0, b2f_stream_t stream);
/* b2f_rmsnorm_rope out of place (training keeps the pre-norm projections); the output may alias the input when the
 * pitches match.  Its backward: in place on the Q / K column blocks of the gradient buffer; partial[(batch*S + 7)/8,
 * 512] receives per-block RMSNorm-weight gradient rows [wq_a | wk_a | wq_b | wk_b] (NULL: none). */
int b2f_rmsnorm_rope_out(const void* xq, const void* xk, int64_t ldx, int64_t x_bs, void* oq, void* ok, int64_t ldo,
                         int64_t o_bs, const void* wq_a, const void* wk_a, const void* wq_b, const void* wk_b,
                         const float* cos, const float* sin, int batch, int S, int H, int n_a, float eps,
                         b2f_stream_t stream);
int b2f_rmsnorm_rope_bwd(void* dq, void* dk, int64_t ld, int64_t bs, const void* xq, const void* xk, int64_t ldx,
                         int64_t x_bs, const void* wq_a, const void* wk_a, const void* wq_b, const void* wk_b,
                         const float* cos, const float* sin, float* partial, int batch, int S, int H, int n_a, float eps,
                         b2f_stream_t stream);
/* y = gelu_tanh(x) over a [rows, D] view. */
int b2f_gelu_rows(const void* x, int64_t ldx, void* y, int64_t ldy, int64_t rows, int D, b2f_stream_t stream);
/* dW[n, k] (+)= sum_b dmod[b, n] * act[b, k]: weight gradient of an AdaLN linear (dmod fp32, act bf16, dW fp32). */
int b2f_outer_acc(const float* dmod, int64_t dmod_ld, const void* act, int64_t act_ld, float* dW, int64_t ldw, int B,
                  int N, int K, int accumulate, b2f_stream_t stream);
/* Flow-matching loss (train_denoiser.py:1105-1167): *loss_out = mean(w * (pred - target)^2); dpred = bf16(2 w (pred -
 * target) * grad_scale / n).  pred bf16, target / w fp32 (w NULL: 1), ws: 1024 floats of scratch. */
int b2f_mse_loss(const void* pred, const float* target, const float* w, void* dpred, float* loss_out, float* ws,
                 int64_t n, float grad_scale, b2f_stream_t stream);
/* *sumsq_out (+)= sum(g^2) over a flat fp32 gradient shard (ws: 1024 floats); coef = min(1, max_norm / (pre_scale *
 * sqrt(sumsq) + 1e-6)) * pre_scale — accelerate's clip_grad_norm_ folded into the gradient scale AdamW applies. */
int b2f_grad_sumsq(const float* g, int64_t n, float* sumsq_out, float* ws, int accumulate, b2f_stream_t stream);
int b2f_clip_coef(const float* sumsq, float max_norm, float pre_scale, float* coef, float* norm_out, b2f_stream_t stream);
/* torch.optim.AdamW on flat fp32 shards (master weights p32, moments m / v), gradient scaled by *gscale (device scalar,
 * NULL: 1), bf16 copy of the new weights written to p16 (NULL: none).  step counts from 1. */
int b2f_adamw_step(float* p32, float* m, float* v, const float* g, void* p16, int64_t n, float lr, float beta1,
                   float beta2, float eps, float weight_decay, int step, const float* gscale, b2f_stream_t stream);
/* out = bf16(bf16(a * wa) + bf16(b * wb)) over n contiguous bf16 elements (n % 8 == 0; wa, wb stay fp32): the
 * `old * (1 - f) + image_embeds * f` blend of vlm_residual_image_factor (modeling_univa_qwen2p5vl.py:504-506). */
int b2f_blend_bf16(const void* a, const void* b, float wa, float wb, void* out, int64_t n, b2f_stream_t stream);
/* bf16 <-> fp32 copies of flat arrays (master-weight initialisation, gradient buckets). */
int b2f_cast_bf16_f32(const void* src, void* dst, int64_t n, int to_f32, b2f_stream_t stream);

/* Training step of the FLUX object (reference train_denoiser.py:829-1181 with enable_gradient_checkpointing, :484-486).
 * b2f_flux_bind_grad binds an fp32 gradient buffer (borrowed) to a trainable tensor; a tensor without a bound
 * gradient is frozen and its weight-gradient GEMM is skipped.  Names (element counts as the weights):
 *   transformer_blocks.{i}.attn.qkv.{weight,bias}            (to_q, to_k, to_v of the image stream, fused)
 *   transformer_blocks.{i}.attn.to_out.0.{weight,bias}
 *   transformer_blocks.{i}.attn.norm_q.weight / norm_k.weight
 *   transformer_blocks.{i}.norm1.linear.{weight,bias}         ([6d, d]: the block's rows of the fused adaln tensor)
 *   single_transformer_blocks.{j}.attn.qkv.{weight,bias}     ([3d, d]: rows [0, 3d) of qkv_mlp)
 *   single_transformer_blocks.{j}.attn.norm_q.weight / norm_k.weight
 *   single_transformer_blocks.{j}.norm.linear.{weight,bias}   ([3d, d])
 * — exactly get_trainable_params(only_img_branch=True), train_denoiser.py:71-119.  dptr == NULL unbinds. */
int b2f_flux_bind_grad(b2f_flux* ctx, const char* key, float* dptr, int64_t numel);
size_t b2f_flux_train_workspace_bytes(const b2f_flux* ctx, int B, int S_img, int S_txt);
/* Forward that keeps the input of every block (activation checkpoints) in ws; same arguments and results as
 * b2f_flux_forward over all blocks. */
int b2f_flux_train_forward(b2f_flux* ctx, const void* hidden, const void* enc, const void* mod, int64_t mod_ld,
                           void* out, int B, int S_img, int S_txt, int n_out_rows, void* ws, size_t ws_bytes,
                           b2f_stream_t stream);
/* Backward over blocks [first_block, last_block) in reverse order, re-running each block from its checkpoint
 * (pass (0, -1) for the whole model; partial ranges let the caller overlap a block's gradient reduction with the
 * next block's backward: the residual-stream gradient persists in ws).  The tail (proj_out, norm_out) runs iff
 * last_block covers the last block and consumes dout [B, n_out_rows, out_channels] bf16; the head runs iff
 * first_block == 0 and writes d_enc [B, S_txt, joint_dim] bf16 (gradient of encoder_hidden_states, NULL: skip).
 * silu_temb: [B, d] bf16 as written by b2f_flux_temb (input of every AdaLN linear).  accumulate != 0 adds to the
 * bound gradient buffers (gradient accumulation steps) instead of overwriting them. */
int b2f_flux_train_backward(b2f_flux* ctx, const void* dout, const void* mod, int64_t mod_ld, const void* silu_temb,
                            int64_t silu_ld, void* d_enc, int B, int S_img, int S_txt, int n_out_rows, int accumulate,
                            void* ws, size_t ws_bytes, int first_block, int last_block, b2f_stream_t stream);
/* Test access: copy of the running residual-stream gradient dh[B, S_txt+S_img, d] bf16. */
int b2f_flux_train_debug_dh(b2f_flux* ctx, void* dst, int B, int S_img, int S_txt, void* ws, b2f_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * FLUX VAE (diffusers AutoencoderKL) as one object.  Replaces `pipe.vae.encode(x)` /
 * `pipe.vae.decode(z)` — reference univa/utils/flux_pipeline.py:609, :1129; train_denoiser.py:887.
 * Weights are borrowed bf16 device pointers bound under their diffusers names (SURVEY.md A.4) with
 * these layout conventions (the Python side converts at load and converts back in state_dict()):
 *   3x3 conv weights   OHWI [Cout,3,3,Cin]; conv_in weights have Cin zero-padded to 64
 *   1x1 conv_shortcut  [Cout,Cin]
 *   biases             zero-padded to a multiple of 8 elements
 *   mid attention      to_q/to_k/to_v bound fused as `<...>.attentions.0.qkv.{weight,bias}` [3C,C]
 */
typedef struct b2f_vae b2f_vae;
typedef struct {
  int block_out[4];     /* 128,256,512,512 */
  int layers_per_block; /* 2 */
  int latent_channels;  /* 16 */
  int in_channels;      /* 3 */
  int out_channels;     /* 3 */
} b2f_vae_cfg;
int b2f_vae_create(b2f_vae** out, const b2f_vae_cfg* cfg);
void b2f_vae_destroy(b2f_vae* ctx);
int b2f_vae_bind_weight(b2f_vae* ctx, const char* key, const void* dptr, int64_t numel);
size_t b2f_vae_workspace_bytes(const b2f_vae* ctx, int N, int H, int W);
/* For tests only: later encode / decode calls on ctx stop after stage `stage` (1-based; 0, the default, runs to the
 * end) and leave that stage's activation, NHWC bf16 [N, h, w, C], at the start of the workspace rounded up to 256 bytes;
 * the output tensor is not written.  Stages, with L = layers_per_block:
 *   encoder  1 conv_in; per down block i = 0..3: L ResnetBlock2D stages, then (i < 3) the downsampler (pad + stride-2
 *            conv); mid_block resnets.0, attentions.0, resnets.1; conv_norm_out + conv_out (the moments).
 *            4L + 8 stages.
 *   decoder  1 conv_in; mid_block resnets.0, attentions.0, resnets.1; per up block i = 0..3: L + 1 ResnetBlock2D
 *            stages, then (i < 3) nearest 2x upsample + conv; conv_norm_out + conv_out (the image).  4L + 12 stages.
 * A stop at or past the last stage is a full run.  The stop is a host-side check between launches. */
int b2f_vae_set_stop_stage(b2f_vae* ctx, int stage);
/* image -> moments [N, 2*latent, H/8, W/8] bf16 (mean | logvar, un-clamped; `latent_dist.mode()` is the first half).
 * image_is_f32 selects the input format: 0 = bf16 [N,3,H,W], 1 = fp32 [N,3,H,W], 2 = uint8 [N,H,W,3] pixels (PIL / numpy
 * layout): the reference's host-side normalisation `(u/255 - 0.5)/0.5` and `.to(bf16)` (univa/serve/cli.py:99-116) run inside
 * the kernel that feeds encoder.conv_in, so a 1024x1024 context image crosses PCIe as 3 MB instead of 12 MB. */
int b2f_vae_encode(b2f_vae* ctx, const void* image_nchw, int image_is_f32, int N, int H, int W,
                   void* moments_nchw, void* ws, size_t ws_bytes, b2f_stream_t stream);
/* z [N,latent,h,w] bf16 -> image [N,3,8h,8w] bf16; b2f_vae_decode_u8 writes uint8 [N,8h,8w,3] pixels instead:
 * VaeImageProcessor.postprocess (`(x/2 + 0.5).clamp(0,1)`, `(. * 255).round()`, reference flux_pipeline.py:1130) fused
 * into the epilogue of decoder.conv_out. */
int b2f_vae_decode(b2f_vae* ctx, const void* z_nchw, int N, int h_lat, int w_lat, void* image_nchw,
                   void* ws, size_t ws_bytes, b2f_stream_t stream);
int b2f_vae_decode_u8(b2f_vae* ctx, const void* z_nchw, int N, int h_lat, int w_lat, void* image_u8_nhwc,
                      void* ws, size_t ws_bytes, b2f_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* B2F_H_ */
