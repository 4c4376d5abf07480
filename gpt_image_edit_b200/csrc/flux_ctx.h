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
  // fp32 gradient buffers of the trainable tensors, bound by name (flux_train.cu); an unbound name is frozen
  std::map<std::string, std::pair<float*, int64_t>> grads;
};

}  // namespace b2f
