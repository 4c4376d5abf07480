// Stage-2 training step of the FLUX-Kontext MMDiT composed from the libb2f kernels: forward with per-block
// activation checkpoints, backward with per-block recompute, gradients of the reference's trainable set.
//
// Reference: train_denoiser.py:829-1181 (one optimisation step), :484-486 (`enable_gradient_checkpointing`:
// every transformer block is re-run in the backward pass), :71-119 (`get_trainable_params`: per double block
// attn.to_q/k/v, attn.to_out, attn.norm_q/k, norm1.linear; per single block attn.to_q/k/v, attn.norm_q/k,
// norm.linear; image stream only), :1172 (`accelerator.backward`).  The reference gets the backward from
// torch.autograd over diffusers' eager modules; here it is written out op by op:
//
//   forward  (b2f_flux_train_forward):  the inference kernels block by block, the block input h[B,S,d] copied to a
//            checkpoint before each block (57 x B x S x d bf16);
//   backward (b2f_flux_train_backward): for blocks 56..0: re-run the block with the UNFUSED kernels, keeping what
//            the backward needs (pre-norm q/k, pre-GELU u, the gated branch outputs y, LSE), then walk it
//            backwards.  Activation gradients bf16, weight gradients fp32 into caller-bound buffers
//            (b2f_flux_bind_grad; an unbound name = frozen parameter: no weight-gradient GEMM is launched).
// The gradient w.r.t. encoder_hidden_states is returned (it feeds MLP2, which is trainable); x_embedder,
// context_embedder, the FF layers, the text stream's projections and the time/guidance/pooled embedders are
// frozen in stage 2, so only their data gradients are propagated.
#include <cstring>
#include <string>

#include "flux_ctx.h"

namespace b2f {

namespace {

inline size_t al256(size_t n) { return (n + 255) & ~size_t(255); }

// carve-up of the training workspace (all offsets 256-byte aligned)
struct TrainWs {
  size_t infer_bytes;      // workspace of b2f_flux_forward (h | xn | qkv | cat), at offset 0
  bf16_t *ckpt;            // [(nblocks + 1), B, S, d]
  bf16_t *hin, *xn, *pre, *qkv, *cat, *y1, *h1, *xn2, *y2;   // recompute buffers (pre: [B,S,7d], qkv: [B,S,3d], cat: [B,S,5d])
  bf16_t *dh, *dy, *dxn, *dpre, *dattn;                      // gradients (dpre: [B,S,7d])
  float *lse, *delta, *partial, *dmod, *red;
  size_t total;
};

TrainWs carve(const FluxCtx* c, void* ws, int B, int S_img, int S_txt, size_t infer_bytes) {
  const size_t S = (size_t)S_img + S_txt, d = c->d, BS = (size_t)B * S;
  const size_t nblk = (size_t)c->cfg.num_double + c->cfg.num_single;
  const size_t S_pad = (S + 127) / 128 * 128;
  TrainWs w{};
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~uintptr_t(255));
  size_t off = al256(infer_bytes);
  w.infer_bytes = infer_bytes;
  auto take = [&](size_t elems, size_t esz) {
    uint8_t* p = base ? base + off : nullptr;
    off += al256(elems * esz);
    return p;
  };
  w.ckpt = reinterpret_cast<bf16_t*>(take((nblk + 1) * BS * d, 2));
  w.hin = reinterpret_cast<bf16_t*>(take(BS * d, 2));
  w.xn = reinterpret_cast<bf16_t*>(take(BS * d, 2));
  w.pre = reinterpret_cast<bf16_t*>(take(BS * 7 * d, 2));
  w.qkv = reinterpret_cast<bf16_t*>(take(BS * 3 * d, 2));
  w.cat = reinterpret_cast<bf16_t*>(take(BS * 5 * d, 2));
  w.y1 = reinterpret_cast<bf16_t*>(take(BS * d, 2));
  w.h1 = reinterpret_cast<bf16_t*>(take(BS * d, 2));
  w.xn2 = reinterpret_cast<bf16_t*>(take(BS * d, 2));
  w.y2 = reinterpret_cast<bf16_t*>(take(BS * d, 2));
  w.dh = reinterpret_cast<bf16_t*>(take(BS * d, 2));
  w.dy = reinterpret_cast<bf16_t*>(take(BS * d, 2));
  w.dxn = reinterpret_cast<bf16_t*>(take(BS * d, 2));
  w.dpre = reinterpret_cast<bf16_t*>(take(BS * 7 * d, 2));
  w.dattn = reinterpret_cast<bf16_t*>(take(BS * d, 2));
  w.lse = reinterpret_cast<float*>(take((size_t)B * c->cfg.num_heads * S_pad, 4));
  w.delta = reinterpret_cast<float*>(take((size_t)B * c->cfg.num_heads * S_pad, 4));
  // column-sum partials: the largest user is ln_modulate_bwd (B x chunks x 2d); RMSNorm: ceil(B*S/8) x 512
  const size_t p1 = (size_t)B * b2f_train_ln_chunks((int)S) * 2 * d, p2 = (size_t)B * b2f_train_chunks((int)S) * 3 * d,
               p3 = (BS + 7) / 8 * 512;
  w.partial = reinterpret_cast<float*>(take(p1 > p2 ? (p1 > p3 ? p1 : p3) : (p2 > p3 ? p2 : p3), 4));
  w.dmod = reinterpret_cast<float*>(take((size_t)B * 6 * d, 4));
  w.red = reinterpret_cast<float*>(take((size_t)B * 2 * d + 1024, 4));
  w.total = off + 256;
  return w;
}

struct Grad {
  float* p = nullptr;
};
Grad find_grad(FluxCtx* c, const std::string& key, int64_t numel, int* rc) {
  Grad g;
  auto it = c->grads.find(key);
  if (it == c->grads.end()) return g;
  if (it->second.second != numel) {
    fprintf(stderr, "[b2f] gradient '%s' has %lld elements, expected %lld\n", key.c_str(), (long long)it->second.second,
            (long long)numel);
    *rc = B2F_ERR_INVALID;
    return g;
  }
  g.p = it->second.first;
  return g;
}

}  // namespace
}  // namespace b2f

using namespace b2f;

extern "C" {

int b2f_flux_bind_grad(b2f_flux* h, const char* key, float* dptr, int64_t numel) {
  FluxCtx* c = reinterpret_cast<FluxCtx*>(h);
  if (!c || !key) return B2F_ERR_INVALID;
  if (!dptr) {   // unbind: the parameter is frozen again
    c->grads.erase(key);
    return B2F_OK;
  }
  if (numel <= 0) return B2F_ERR_INVALID;
  if (reinterpret_cast<uintptr_t>(dptr) & 15) return B2F_ERR_ALIGN;
  c->grads[key] = {dptr, numel};
  return B2F_OK;
}

size_t b2f_flux_train_workspace_bytes(const b2f_flux* h, int B, int S_img, int S_txt) {
  const FluxCtx* c = reinterpret_cast<const FluxCtx*>(h);
  if (!c || B <= 0 || S_img <= 0 || S_txt <= 0) return 0;
  const size_t infer = b2f_flux_workspace_bytes(h, B, S_img, S_txt);
  return carve(c, nullptr, B, S_img, S_txt, infer).total;
}

int b2f_flux_train_forward(b2f_flux* h, const void* hidden, const void* enc, const void* mod, int64_t mod_ld, void* out,
                           int B, int S_img, int S_txt, int n_out_rows, void* ws, size_t ws_bytes, b2f_stream_t stream_) {
  FluxCtx* c = reinterpret_cast<FluxCtx*>(h);
  if (!c || !c->finalized || !ws) return B2F_ERR_INVALID;
  if (c->lora_rmax() > 0) {   // the backward does not see unfused adapters: fuse or unbind them first
    fprintf(stderr, "[b2f] flux_train_forward: unfused LoRA adapters are bound\n");
    return B2F_ERR_UNSUPPORTED;
  }
  if (c->fp8 || c->fp8_attn) {   // training runs the bf16 weights and attention: switch FP8 off first
    fprintf(stderr, "[b2f] flux_train_forward: FP8 is on\n");
    return B2F_ERR_UNSUPPORTED;
  }
  if (ws_bytes < b2f_flux_train_workspace_bytes(h, B, S_img, S_txt)) return B2F_ERR_WORKSPACE;
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  const size_t infer = b2f_flux_workspace_bytes(h, B, S_img, S_txt);
  TrainWs w = carve(c, ws, B, S_img, S_txt, infer);
  const int nblk = c->cfg.num_double + c->cfg.num_single;
  const size_t S = (size_t)S_img + S_txt, hbytes = (size_t)B * S * c->d * 2;
  // the inference workspace starts with h[B,S,d] (flux_model.cu); same 256-byte alignment rule as there
  bf16_t* hb = reinterpret_cast<bf16_t*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~uintptr_t(255));
  int rc = b2f_flux_forward(h, hidden, enc, mod, mod_ld, out, B, S_img, S_txt, n_out_rows, ws, infer, 0, 0, stream_);
  if (rc) return rc;
  for (int blk = 0; blk < nblk; ++blk) {
    if (cudaMemcpyAsync(w.ckpt + (size_t)blk * B * S * c->d, hb, hbytes, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
      return cuda_err(cudaGetLastError(), "checkpoint copy");
    // blk == 0 re-runs the embedders (first_block == 0): same inputs, same result
    rc = b2f_flux_forward(h, hidden, enc, mod, mod_ld, out, B, S_img, S_txt, n_out_rows, ws, infer, blk, blk + 1, stream_);
    if (rc) return rc;
  }
  if (cudaMemcpyAsync(w.ckpt + (size_t)nblk * B * S * c->d, hb, hbytes, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
    return cuda_err(cudaGetLastError(), "checkpoint copy");
  return B2F_OK;
}

int b2f_flux_train_backward(b2f_flux* h, const void* dout, const void* mod, int64_t mod_ld, const void* silu_temb,
                            int64_t silu_ld, void* d_enc, int B, int S_img, int S_txt, int n_out_rows, int accumulate,
                            void* ws, size_t ws_bytes, int first_block, int last_block, b2f_stream_t stream_) {
  FluxCtx* c = reinterpret_cast<FluxCtx*>(h);
  if (!c || !c->finalized || !mod || !silu_temb || !ws || B <= 0 || S_img <= 0 || S_txt <= 0)
    return B2F_ERR_INVALID;
  if (n_out_rows <= 0 || n_out_rows > S_img) return B2F_ERR_INVALID;
  if (c->fp8 || c->fp8_attn) {
    fprintf(stderr, "[b2f] flux_train_backward: FP8 is on\n");
    return B2F_ERR_UNSUPPORTED;
  }
  if (ws_bytes < b2f_flux_train_workspace_bytes(h, B, S_img, S_txt)) return B2F_ERR_WORKSPACE;
  const int S = S_img + S_txt;
  if (!c->rope_cos || c->rope_S != S) return B2F_ERR_INVALID;
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  const b2f_flux_cfg& g = c->cfg;
  const int64_t d = c->d;
  const int H = g.num_heads, nblk = g.num_double + g.num_single;
  if (first_block < 0) first_block = 0;
  if (last_block < 0 || last_block > nblk) last_block = nblk;
  if (last_block == nblk && !dout) return B2F_ERR_INVALID;
  const float eps = 1e-6f, scale = 1.0f / sqrtf((float)g.head_dim);
  const int64_t S_pad = (S + 127) / 128 * 128;
  TrainWs w = carve(c, ws, B, S_img, S_txt, b2f_flux_workspace_bytes(h, B, S_img, S_txt));
  const int64_t BS = (int64_t)B * S;
  const int64_t bs1 = (int64_t)S * d, bs3 = 3 * bs1, bs5 = 5 * bs1, bs7 = 7 * bs1;
  const bf16_t* modp = static_cast<const bf16_t*>(mod);
  const int acc0 = accumulate ? 1 : 0;
  int rc = B2F_OK;
#define RUN(expr) \
  if ((rc = (expr)) != 0) return rc
  // row-offset helpers into [B, S, width] buffers (text rows first)
  auto img = [&](bf16_t* p, int64_t width) { return p + (int64_t)S_txt * width; };
  const int nch = b2f_train_chunks(S), nlch = b2f_train_ln_chunks(S);

  // column sums of a [B, rows, D] view into a flat fp32 gradient (summed over the batch as well)
  auto bias_grad = [&](const bf16_t* dy, int64_t ld, int64_t bs, int rows, int D, float* dst) -> int {
    const int ch = b2f_train_chunks(rows);
    int r = b2f_gate_bwd(dy, ld, bs, nullptr, 0, 0, nullptr, nullptr, 0, nullptr, 0, 0, w.partial, B, rows, D, 0, 0, st);
    if (r) return r;
    // partial is [B, ch, D]: reduce it as one batch of B*ch chunks
    return b2f_col_reduce(w.partial, B * ch, D, dst, D, 1, acc0, st);
  };
  // AdaLN-linear gradients of one block from dmod[B, n_mod*d] (fp32) and silu(temb)
  auto adaln_grads = [&](const std::string& name, int n_mod) -> int {
    int r = B2F_OK;
    Grad gw = find_grad(c, name + ".weight", (int64_t)n_mod * d * d, &r);
    Grad gb = find_grad(c, name + ".bias", (int64_t)n_mod * d, &r);
    if (r) return r;
    // dmod is [B, n_mod*d] with pitch n_mod*d (6d in a double block, 3d in a single block)
    if (gw.p && (r = b2f_outer_acc(w.dmod, n_mod * d, silu_temb, silu_ld, gw.p, d, B, (int)(n_mod * d), (int)d, acc0, st))) return r;
    if (gb.p && (r = b2f_col_reduce(w.dmod, B, (int)(n_mod * d), gb.p, n_mod * d, 1, acc0, st))) return r;
    return B2F_OK;
  };

  // ---------------------------------------------------------------- tail: proj_out, norm_out
  if (last_block == nblk) {
    RUN(cuda_err(cudaMemsetAsync(w.dh, 0, (size_t)BS * d * 2, st), "memset dh"));
    const bf16_t* mo = modp + (int64_t)g.num_double * 12 * d + (int64_t)g.num_single * 3 * d;
    const bf16_t* hfin = w.ckpt + (int64_t)nblk * BS * d;
    // dxn[img rows < n_out] = dout . proj_out.weight     ([B, n_out, 64] x [64, d])
    RUN(b2f_gemm_dgrad(dout, g.out_channels, (int64_t)n_out_rows * g.out_channels, c->proj_out.w, d, img(w.dxn, d), d, bs1, B,
                       n_out_rows, (int)d, g.out_channels, B2F_EPI_BIAS, nullptr, 0, 0, st));
    RUN(b2f_ln_modulate_bwd(img(const_cast<bf16_t*>(hfin), d), d, bs1, img(w.dxn, d), d, bs1, mo, nullptr, mod_ld, nullptr, 0, 0,
                            img(w.dh, d), d, bs1, nullptr, B, n_out_rows, (int)d, eps, 0, 0, st));
  }

  for (int blk = last_block - 1; blk >= first_block; --blk) {
    const bf16_t* hin = w.ckpt + (int64_t)blk * BS * d;
    if (blk < g.num_double) {
      const DoubleW& wt = c->dbl[blk];
      const std::string pn = "transformer_blocks." + std::to_string(blk) + ".";
      const bf16_t* mi = modp + (int64_t)blk * 12 * d;
      const bf16_t* mt = mi + 6 * d;
      // ------------------------------------------------ recompute, unfused, keeping what the backward reads
      RUN(b2f_ln_modulate(hin, d, bs1, mt + d, mt, mod_ld, w.xn, d, bs1, B, S, (int)d, eps, S_txt, mi + d, mi, st));
      RUN(b2f_gemm_bf16(img(w.xn, d), d, bs1, wt.qkv.w, d, wt.qkv.b, img(w.pre, 3 * d), 3 * d, bs3, B, S_img, (int)(3 * d),
                        (int)d, B2F_EPI_BIAS, nullptr, 0, 0, nullptr, 0, st));
      RUN(b2f_gemm_bf16(w.xn, d, bs1, wt.add_qkv.w, d, wt.add_qkv.b, w.pre, 3 * d, bs3, B, S_txt, (int)(3 * d), (int)d,
                        B2F_EPI_BIAS, nullptr, 0, 0, nullptr, 0, st));
      RUN(b2f_rmsnorm_rope_out(w.pre, w.pre + d, 3 * d, bs3, w.qkv, w.qkv + d, 3 * d, bs3, wt.norm_added_q, wt.norm_added_k,
                               wt.norm_q, wt.norm_k, c->rope_cos, c->rope_sin, B, S, H, S_txt, eps, st));
      RUN(b2f_attention_fwd_lse(w.qkv, 3 * d, w.qkv + d, 3 * d, w.pre + 2 * d, 3 * d, w.cat, 5 * d, B, H, H, S, S, g.head_dim,
                                scale, 0, w.lse, S_pad, st));
      RUN(b2f_gemm_bf16(img(w.cat, 5 * d), 5 * d, bs5, wt.to_out.w, d, wt.to_out.b, img(w.y1, d), d, bs1, B, S_img, (int)d, (int)d,
                        B2F_EPI_BIAS, nullptr, 0, 0, nullptr, 0, st));
      RUN(b2f_gemm_bf16(w.cat, 5 * d, bs5, wt.to_add_out.w, d, wt.to_add_out.b, w.y1, d, bs1, B, S_txt, (int)d, (int)d,
                        B2F_EPI_BIAS, nullptr, 0, 0, nullptr, 0, st));
      RUN(b2f_gate_resid_fwd(hin, d, bs1, w.y1, d, bs1, mt + 2 * d, mi + 2 * d, mod_ld, w.h1, d, bs1, B, S, (int)d, S_txt, st));
      RUN(b2f_ln_modulate(w.h1, d, bs1, mt + 4 * d, mt + 3 * d, mod_ld, w.xn2, d, bs1, B, S, (int)d, eps, S_txt, mi + 4 * d,
                          mi + 3 * d, st));
      // u = pre-GELU MLP activations -> dpre buffer columns [0, 4d) are free until the backward of this block: keep u
      // in `pre` columns... the QKV pre-activations own pre[.., 0:3d]; u lives in pre[.., 3d:7d] (pitch 7d is not
      // shared with the 3d-pitched QKV view, so u gets its own region at the end of the buffer)
      bf16_t* u = w.pre + BS * 3 * d;   // [B, S, 4d], contiguous
      const int64_t bs4 = 4 * bs1;
      RUN(b2f_gemm_bf16(img(w.xn2, d), d, bs1, wt.ff1.w, d, wt.ff1.b, img(u, 4 * d), 4 * d, bs4, B, S_img, (int)(4 * d), (int)d,
                        B2F_EPI_BIAS, nullptr, 0, 0, nullptr, 0, st));
      RUN(b2f_gemm_bf16(w.xn2, d, bs1, wt.ffc1.w, d, wt.ffc1.b, u, 4 * d, bs4, B, S_txt, (int)(4 * d), (int)d, B2F_EPI_BIAS,
                        nullptr, 0, 0, nullptr, 0, st));
      RUN(b2f_gelu_rows(u, 4 * d, w.cat + d, 5 * d, BS, (int)(4 * d), st));
      RUN(b2f_gemm_bf16(img(w.cat, 5 * d) + d, 5 * d, bs5, wt.ff2.w, 4 * d, wt.ff2.b, img(w.y2, d), d, bs1, B, S_img, (int)d,
                        (int)(4 * d), B2F_EPI_BIAS, nullptr, 0, 0, nullptr, 0, st));
      RUN(b2f_gemm_bf16(w.cat + d, 5 * d, bs5, wt.ffc2.w, 4 * d, wt.ffc2.b, w.y2, d, bs1, B, S_txt, (int)d, (int)(4 * d),
                        B2F_EPI_BIAS, nullptr, 0, 0, nullptr, 0, st));
      // ------------------------------------------------ backward
      // h2 = h1 + gate_mlp * y2
      RUN(b2f_gate_bwd(w.dh, d, bs1, w.y2, d, bs1, mt + 5 * d, mi + 5 * d, mod_ld, w.dy, d, bs1, w.partial, B, S, (int)d, S_txt,
                       S_txt, st));
      RUN(b2f_col_reduce(w.partial, nch, (int)d, w.dmod + 5 * d, 6 * d, B, 0, st));
      // y2 = gelu(u) W2^T + b2:  du = (dy . W2) * gelu'(u)   -> dpre[.., 0:4d] viewed with pitch 4d
      bf16_t* du = w.dpre;   // [B, S, 4d]
      RUN(b2f_gemm_dgrad(img(w.dy, d), d, bs1, wt.ff2.w, 4 * d, img(du, 4 * d), 4 * d, bs4, B, S_img, (int)(4 * d), (int)d,
                         B2F_EPI_DGELU, img(u, 4 * d), 4 * d, bs4, st));
      RUN(b2f_gemm_dgrad(w.dy, d, bs1, wt.ffc2.w, 4 * d, du, 4 * d, bs4, B, S_txt, (int)(4 * d), (int)d, B2F_EPI_DGELU, u, 4 * d,
                         bs4, st));
      // u = xn2 W1^T + b1
      RUN(b2f_gemm_dgrad(img(du, 4 * d), 4 * d, bs4, wt.ff1.w, d, img(w.dxn, d), d, bs1, B, S_img, (int)d, (int)(4 * d),
                         B2F_EPI_BIAS, nullptr, 0, 0, st));
      RUN(b2f_gemm_dgrad(du, 4 * d, bs4, wt.ffc1.w, d, w.dxn, d, bs1, B, S_txt, (int)d, (int)(4 * d), B2F_EPI_BIAS, nullptr, 0, 0,
                         st));
      // xn2 = LN(h1) (1 + scale_mlp) + shift_mlp;  dh <- dh + dLN
      RUN(b2f_ln_modulate_bwd(w.h1, d, bs1, w.dxn, d, bs1, mt + 4 * d, mi + 4 * d, mod_ld, w.dh, d, bs1, w.dh, d, bs1, w.partial,
                              B, S, (int)d, eps, S_txt, S_txt, st));
      // partial rows are [dscale | dshift]; dmod columns are [.., shift_mlp (3d), scale_mlp (4d), ..]
      RUN(b2f_col_reduce(w.partial, nlch, (int)(2 * d), w.red, 2 * d, B, 0, st));
      RUN(cuda_err(cudaMemcpy2DAsync(w.dmod + 4 * d, 6 * d * 4, w.red, 2 * d * 4, d * 4, B, cudaMemcpyDeviceToDevice, st),
                   "dscale copy"));
      RUN(cuda_err(cudaMemcpy2DAsync(w.dmod + 3 * d, 6 * d * 4, w.red + d, 2 * d * 4, d * 4, B, cudaMemcpyDeviceToDevice, st),
                   "dshift copy"));
      // h1 = h + gate_msa * y1
      RUN(b2f_gate_bwd(w.dh, d, bs1, w.y1, d, bs1, mt + 2 * d, mi + 2 * d, mod_ld, w.dy, d, bs1, w.partial, B, S, (int)d, S_txt,
                       S_txt, st));
      RUN(b2f_col_reduce(w.partial, nch, (int)d, w.dmod + 2 * d, 6 * d, B, 0, st));
      // y1 = attn W_o^T + b_o   (image stream: to_out is trainable)
      {
        Grad gw = find_grad(c, pn + "attn.to_out.0.weight", d * d, &rc);
        Grad gb = find_grad(c, pn + "attn.to_out.0.bias", d, &rc);
        if (rc) return rc;
        if (gw.p)
          RUN(b2f_gemm_wgrad(img(w.dy, d), d, bs1, img(w.cat, 5 * d), 5 * d, bs5, gw.p, d, B, S_img, (int)d, (int)d, acc0, st));
        if (gb.p) RUN(bias_grad(img(w.dy, d), d, bs1, S_img, (int)d, gb.p));
      }
      RUN(b2f_gemm_dgrad(img(w.dy, d), d, bs1, wt.to_out.w, d, img(w.dattn, d), d, bs1, B, S_img, (int)d, (int)d, B2F_EPI_BIAS,
                         nullptr, 0, 0, st));
      RUN(b2f_gemm_dgrad(w.dy, d, bs1, wt.to_add_out.w, d, w.dattn, d, bs1, B, S_txt, (int)d, (int)d, B2F_EPI_BIAS, nullptr, 0, 0,
                         st));
      // joint attention
      bf16_t* dqkv = w.dpre + BS * 4 * d;   // [B, S, 3d] after the du region
      RUN(b2f_attn_delta(w.cat, 5 * d, w.dattn, d, w.delta, w.lse, B, H, S, (int)S_pad, st));
      RUN(b2f_attention_bwd(w.qkv, 3 * d, w.qkv + d, 3 * d, w.pre + 2 * d, 3 * d, w.dattn, d, w.lse, w.delta, S_pad, dqkv, 3 * d,
                            dqkv + d, 3 * d, dqkv + 2 * d, 3 * d, B, H, S, g.head_dim, scale, st));
      // per-head RMSNorm + RoPE of q, k
      {
        Grad gq = find_grad(c, pn + "attn.norm_q.weight", g.head_dim, &rc);
        Grad gk = find_grad(c, pn + "attn.norm_k.weight", g.head_dim, &rc);
        if (rc) return rc;
        const bool want = gq.p || gk.p;
        RUN(b2f_rmsnorm_rope_bwd(dqkv, dqkv + d, 3 * d, bs3, w.pre, w.pre + d, 3 * d, bs3, wt.norm_added_q, wt.norm_added_k,
                                 wt.norm_q, wt.norm_k, c->rope_cos, c->rope_sin, want ? w.partial : nullptr, B, S, H, S_txt, eps, st));
        if (want) {
          RUN(b2f_col_reduce(w.partial, (int)((BS + 7) / 8), 512, w.red, 512, 1, 0, st));
          // red = [wq_a | wk_a | wq_b | wk_b]: the image stream's norm_q / norm_k are set b
          if (gq.p) RUN(b2f_col_reduce(w.red + 256, 1, 128, gq.p, 128, 1, acc0, st));
          if (gk.p) RUN(b2f_col_reduce(w.red + 384, 1, 128, gk.p, 128, 1, acc0, st));
        }
      }
      // qkv = xn1 Wqkv^T + b
      {
        Grad gw = find_grad(c, pn + "attn.qkv.weight", 3 * d * d, &rc);
        Grad gb = find_grad(c, pn + "attn.qkv.bias", 3 * d, &rc);
        if (rc) return rc;
        if (gw.p)
          RUN(b2f_gemm_wgrad(img(dqkv, 3 * d), 3 * d, bs3, img(w.xn, d), d, bs1, gw.p, d, B, S_img, (int)(3 * d), (int)d, acc0, st));
        if (gb.p) RUN(bias_grad(img(dqkv, 3 * d), 3 * d, bs3, S_img, (int)(3 * d), gb.p));
      }
      RUN(b2f_gemm_dgrad(img(dqkv, 3 * d), 3 * d, bs3, wt.qkv.w, d, img(w.dxn, d), d, bs1, B, S_img, (int)d, (int)(3 * d),
                         B2F_EPI_BIAS, nullptr, 0, 0, st));
      RUN(b2f_gemm_dgrad(dqkv, 3 * d, bs3, wt.add_qkv.w, d, w.dxn, d, bs1, B, S_txt, (int)d, (int)(3 * d), B2F_EPI_BIAS, nullptr,
                         0, 0, st));
      // xn1 = LN(h) (1 + scale_msa) + shift_msa
      RUN(b2f_ln_modulate_bwd(hin, d, bs1, w.dxn, d, bs1, mt + d, mi + d, mod_ld, w.dh, d, bs1, w.dh, d, bs1, w.partial, B, S,
                              (int)d, eps, S_txt, S_txt, st));
      RUN(b2f_col_reduce(w.partial, nlch, (int)(2 * d), w.red, 2 * d, B, 0, st));
      RUN(cuda_err(cudaMemcpy2DAsync(w.dmod + d, 6 * d * 4, w.red, 2 * d * 4, d * 4, B, cudaMemcpyDeviceToDevice, st),
                   "dscale copy"));
      RUN(cuda_err(cudaMemcpy2DAsync(w.dmod, 6 * d * 4, w.red + d, 2 * d * 4, d * 4, B, cudaMemcpyDeviceToDevice, st),
                   "dshift copy"));
      RUN(adaln_grads(pn + "norm1.linear", 6));
    } else {
      const int si = blk - g.num_double;
      const SingleW& wt = c->sgl[si];
      const std::string pn = "single_transformer_blocks." + std::to_string(si) + ".";
      const bf16_t* ms = modp + (int64_t)g.num_double * 12 * d + (int64_t)si * 3 * d;
      // ------------------------------------------------ recompute
      RUN(b2f_ln_modulate(hin, d, bs1, ms + d, ms, mod_ld, w.xn, d, bs1, B, S, (int)d, eps, 0, nullptr, nullptr, st));
      RUN(b2f_gemm_bf16(w.xn, d, bs1, wt.qkv_mlp.w, d, wt.qkv_mlp.b, w.pre, 7 * d, bs7, B, S, (int)(7 * d), (int)d, B2F_EPI_BIAS,
                        nullptr, 0, 0, nullptr, 0, st));
      RUN(b2f_rmsnorm_rope_out(w.pre, w.pre + d, 7 * d, bs7, w.qkv, w.qkv + d, 3 * d, bs3, nullptr, nullptr, wt.norm_q, wt.norm_k,
                               c->rope_cos, c->rope_sin, B, S, H, 0, eps, st));
      RUN(b2f_attention_fwd_lse(w.qkv, 3 * d, w.qkv + d, 3 * d, w.pre + 2 * d, 7 * d, w.cat, 5 * d, B, H, H, S, S, g.head_dim,
                                scale, 0, w.lse, S_pad, st));
      RUN(b2f_gelu_rows(w.pre + 3 * d, 7 * d, w.cat + d, 5 * d, BS, (int)(4 * d), st));
      RUN(b2f_gemm_bf16(w.cat, 5 * d, bs5, wt.proj_out.w, 5 * d, wt.proj_out.b, w.y1, d, bs1, B, S, (int)d, (int)(5 * d),
                        B2F_EPI_BIAS, nullptr, 0, 0, nullptr, 0, st));
      // ------------------------------------------------ backward
      RUN(b2f_gate_bwd(w.dh, d, bs1, w.y1, d, bs1, ms + 2 * d, nullptr, mod_ld, w.dy, d, bs1, w.partial, B, S, (int)d, 0, 0, st));
      RUN(b2f_col_reduce(w.partial, nch, (int)d, w.dmod + 2 * d, 3 * d, B, 0, st));
      // y = [attn | gelu(u)] Wp^T + b:  dattn = dy . Wp[:, :d];  du = (dy . Wp[:, d:]) * gelu'(u)  -> dpre[.., 3d:7d]
      RUN(b2f_gemm_dgrad(w.dy, d, bs1, wt.proj_out.w, 5 * d, w.dattn, d, bs1, B, S, (int)d, (int)d, B2F_EPI_BIAS, nullptr, 0, 0, st));
      RUN(b2f_gemm_dgrad(w.dy, d, bs1, wt.proj_out.w + d, 5 * d, w.dpre + 3 * d, 7 * d, bs7, B, S, (int)(4 * d), (int)d,
                         B2F_EPI_DGELU, w.pre + 3 * d, 7 * d, bs7, st));
      RUN(b2f_attn_delta(w.cat, 5 * d, w.dattn, d, w.delta, w.lse, B, H, S, (int)S_pad, st));
      RUN(b2f_attention_bwd(w.qkv, 3 * d, w.qkv + d, 3 * d, w.pre + 2 * d, 7 * d, w.dattn, d, w.lse, w.delta, S_pad, w.dpre, 7 * d,
                            w.dpre + d, 7 * d, w.dpre + 2 * d, 7 * d, B, H, S, g.head_dim, scale, st));
      {
        Grad gq = find_grad(c, pn + "attn.norm_q.weight", g.head_dim, &rc);
        Grad gk = find_grad(c, pn + "attn.norm_k.weight", g.head_dim, &rc);
        if (rc) return rc;
        const bool want = gq.p || gk.p;
        RUN(b2f_rmsnorm_rope_bwd(w.dpre, w.dpre + d, 7 * d, bs7, w.pre, w.pre + d, 7 * d, bs7, nullptr, nullptr, wt.norm_q,
                                 wt.norm_k, c->rope_cos, c->rope_sin, want ? w.partial : nullptr, B, S, H, 0, eps, st));
        if (want) {
          RUN(b2f_col_reduce(w.partial, (int)((BS + 7) / 8), 512, w.red, 512, 1, 0, st));
          if (gq.p) RUN(b2f_col_reduce(w.red + 256, 1, 128, gq.p, 128, 1, acc0, st));
          if (gk.p) RUN(b2f_col_reduce(w.red + 384, 1, 128, gk.p, 128, 1, acc0, st));
        }
      }
      {
        Grad gw = find_grad(c, pn + "attn.qkv.weight", 3 * d * d, &rc);
        Grad gb = find_grad(c, pn + "attn.qkv.bias", 3 * d, &rc);
        if (rc) return rc;
        if (gw.p) RUN(b2f_gemm_wgrad(w.dpre, 7 * d, bs7, w.xn, d, bs1, gw.p, d, B, S, (int)(3 * d), (int)d, acc0, st));
        if (gb.p) RUN(bias_grad(w.dpre, 7 * d, bs7, S, (int)(3 * d), gb.p));
      }
      RUN(b2f_gemm_dgrad(w.dpre, 7 * d, bs7, wt.qkv_mlp.w, d, w.dxn, d, bs1, B, S, (int)d, (int)(7 * d), B2F_EPI_BIAS, nullptr, 0,
                         0, st));
      RUN(b2f_ln_modulate_bwd(hin, d, bs1, w.dxn, d, bs1, ms + d, nullptr, mod_ld, w.dh, d, bs1, w.dh, d, bs1, w.partial, B, S,
                              (int)d, eps, 0, 0, st));
      RUN(b2f_col_reduce(w.partial, nlch, (int)(2 * d), w.red, 2 * d, B, 0, st));
      RUN(cuda_err(cudaMemcpy2DAsync(w.dmod + d, 3 * d * 4, w.red, 2 * d * 4, d * 4, B, cudaMemcpyDeviceToDevice, st),
                   "dscale copy"));
      RUN(cuda_err(cudaMemcpy2DAsync(w.dmod, 3 * d * 4, w.red + d, 2 * d * 4, d * 4, B, cudaMemcpyDeviceToDevice, st),
                   "dshift copy"));
      RUN(adaln_grads(pn + "norm.linear", 3));
    }
  }

  // ---------------------------------------------------------------- head: gradient w.r.t. encoder_hidden_states
  if (d_enc && first_block == 0)
    RUN(b2f_gemm_dgrad(w.dh, d, bs1, c->context_embedder.w, g.joint_dim, d_enc, g.joint_dim, (int64_t)S_txt * g.joint_dim, B,
                       S_txt, g.joint_dim, (int)d, B2F_EPI_BIAS, nullptr, 0, 0, st));
#undef RUN
  return B2F_OK;
}

/* debug / test access: copies the running residual-stream gradient dh[B, S, d] (after the last processed block) */
int b2f_flux_train_debug_dh(b2f_flux* h, void* dst, int B, int S_img, int S_txt, void* ws, b2f_stream_t stream_) {
  FluxCtx* c = reinterpret_cast<FluxCtx*>(h);
  if (!c || !dst || !ws) return B2F_ERR_INVALID;
  TrainWs w = carve(c, ws, B, S_img, S_txt, b2f_flux_workspace_bytes(h, B, S_img, S_txt));
  const size_t n = (size_t)B * (S_img + S_txt) * c->d * 2;
  return cuda_err(cudaMemcpyAsync(dst, w.dh, n, cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream_)), "dh copy");
}

}  // extern "C"
