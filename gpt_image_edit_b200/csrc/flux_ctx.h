// Shared state of the FLUX object behind b2f_flux_* (flux_model.cu: inference forward; flux_train.cu: training step).
#pragma once
#include <map>
#include <string>
#include <vector>

#include "host_common.h"

namespace b2f {

typedef uint16_t bf16_t;

// Unfused LoRA of one linear (b2f_flux_bind_lora): Acat [r_pad, in], Bcat [out, r_pad], colscale fp32 [r_pad].
struct LoraBind {
  const bf16_t* A = nullptr;
  const bf16_t* Bc = nullptr;
  const float* cs = nullptr;
  int r_pad = 0;
};
struct Lin {
  const bf16_t* w = nullptr;
  const bf16_t* b = nullptr;
  LoraBind lora;
  // FP8 copy of w (b2f_flux_bind_fp8; block linears only): e4m3 [out, in] and fp32 per-channel scales [out]
  const uint8_t* w8 = nullptr;
  const float* ws = nullptr;
};
// LoRA of one AdaLN linear: rows [row0, row0 + rows) of the fused adaln weight
struct AdalnLora {
  int64_t row0 = 0, rows = 0;
  LoraBind l;
};
struct DoubleW {
  Lin qkv, add_qkv, to_out, to_add_out, ff1, ff2, ffc1, ffc2;
  const bf16_t *norm_q = nullptr, *norm_k = nullptr, *norm_added_q = nullptr, *norm_added_k = nullptr;
};
struct SingleW {
  Lin qkv_mlp, proj_out;
  const bf16_t *norm_q = nullptr, *norm_k = nullptr;
};

struct FluxCtx {
  b2f_flux_cfg cfg;
  int d = 0;
  std::map<std::string, std::pair<const void*, int64_t>> bound;
  Lin x_embedder, context_embedder, proj_out, adaln;
  Lin t1, t2, g1, g2, p1, p2;
  std::vector<DoubleW> dbl;
  std::vector<SingleW> sgl;
  const float* rope_cos = nullptr;
  const float* rope_sin = nullptr;
  int rope_S = 0;
  bool finalized = false;
  int64_t mod_width = 0;
  // unfused LoRA adapters: the AdaLN ones by linear name; every other one sits in its Lin.  lora_scale multiplies every
  // colscale (the per-call `scale` of joint_attention_kwargs).
  std::map<std::string, AdalnLora> adaln_lora;
  float lora_scale = 1.f;
  int lora_count = 0;
  int lora_rmax() const;
  // b2f_flux_set_fp8: the block linears of b2f_flux_forward run in FP8; fp8_lora (mode 2): with unfused adapters
  bool fp8 = false;
  bool fp8_lora = false;
  // b2f_flux_set_fp8_attention: the blocks' attention runs in FP8 (b2f_attn_quant_fp8 + b2f_attention_fp8)
  bool fp8_attn = false;
  // fp32 gradient buffers of the trainable tensors, bound by name (flux_train.cu); an unbound name is frozen
  std::map<std::string, std::pair<float*, int64_t>> grads;
};

// b2f_flux_forward (flux_model.cu) after the handle cast.  x0, when set, receives the image rows of h right after the
// embedders ([B, S_img, d] contiguous): the first-block cache (flux_cache.cu) compares block 0's output with them.
int flux_forward(FluxCtx* c, const void* hidden, const void* enc, const void* mod, int64_t mod_ld, void* out, int B,
                 int S_img, int S_txt, int n_out_rows, void* ws, size_t ws_bytes, int first_block, int last_block,
                 bf16_t* x0, cudaStream_t st);

}  // namespace b2f
