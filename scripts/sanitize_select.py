"""Node ids of the toy-shape GPU tests scripts/sanitize.sh runs under compute-sanitizer: every kernel family that
hand-rolls mbarrier / wgmma pipelines, at shapes small enough for a 10-100x slowdown."""
import subprocess
import sys

WANT = [
    ("tests/test_gemm_gpu.py", ["test_gemm_bias[128-128-64]", "test_gemm_bias[256-512-256]", "test_gemm_bias[1000-136-72]",
                                "test_gemm_gate_resid_batched_views", "test_gemm_gelu_silu"]),
    # the persistent GEMM reusing its ring and staging tiles across tiles of one CTA (SMs + 1 tiles)
    ("tests/test_gemm_persistent_gpu.py", ["test_gemm_toy_tile_counts[1]", "test_gemm_toy_tile_counts[3]",
                                           "test_gemm_toy_tile_counts[sms+1]"]),
    # the LoRA K-extended GEMM (extra k-blocks of T / Bcat through the same ring), its down projection and the merge
    ("tests/test_lora_gpu.py", ["test_lora_gemm_ranks_and_shapes[True-0]", "test_lora_gemm_ranks_and_shapes[False-4]",
                                "test_lora_gemm_qkv_norm_rope[True]", "test_lora_fuse_kernel"]),
    # the composed forward's workspace offsets, pitches and split rows, stage by stage (d 256, B 3, one text token)
    ("tests/test_flux_blocks_gpu.py", ["test_stagewise_forward_matches_fp64[toy_text_of_one]"]),
    # the first-block cache's residual / distance / apply / capture kernels (d 256, B 3, one text token)
    ("tests/test_flux_cache_gpu.py", ["test_cached_forward_equals_the_engines_stages[toy]"]),
    ("tests/test_train_kernels_gpu.py", ["test_gemm_dgrad[1-128-128-64]", "test_gemm_dgrad[1-200-136-72]", "test_gemm_dgrad[2-300-256-512]",
                                         "test_gemm_dgrad[2-1024-1024-4096]", "test_gemm_dgrad_pitched_views_and_epilogues",
                                         "test_gemm_wgrad[1-64-128-128]", "test_gemm_wgrad[1-100-136-200]", "test_gemm_wgrad[3-150-256-384]",
                                         "test_gemm_wgrad[2-1000-1024-4608]", "test_gemm_wgrad_row_slices_of_joint_buffer",
                                         "test_attention_lse_and_backward[1-128-1]", "test_attention_lse_and_backward[2-200-2]",
                                         "test_attention_lse_and_backward[1-1000-3]", "test_gate_resid_and_backward",
                                         "test_ln_modulate_backward", "test_rmsnorm_rope_out_of_place_and_backward", "test_gelu_outer_mse",
                                         "test_adamw_matches_torch_and_clip"]),
    ("tests/test_attention_gpu.py", ["test_attention_matches_fp32_reference[1-1-1-128-128-False]",
                                     "test_attention_matches_fp32_reference[2-3-3-300-300-False]",
                                     "test_attention_matches_fp32_reference[2-2-2-640-640-False]",
                                     "test_attention_matches_fp32_reference[1-4-2-768-1000-False]",
                                     "test_attention_matches_fp32_reference[1-4-2-384-384-True]", "test_attention_peaked_softmax_rows"]),
    # FP8 attention: the amax / quantize / scale passes and the e4m3 kernel with its 16 KB tiles and two slots
    ("tests/test_attn_fp8_gpu.py", ["test_attn_quant_fp8_bit_exact[3-129]", "test_attention_fp8_matches_emulation[2-129]",
                                    "test_attention_fp8_matches_emulation[1-255]", "test_attention_fp8_refusals"]),
    ("tests/test_elementwise_gpu.py", ["test_ln_modulate_matches_eager_chain[1-33-256]", "test_ln_modulate_matches_eager_chain[2-300-3072]",
                                       "test_rmsnorm_rope_matches_eager_chain", "test_euler_step_bit_exact"]),
    # the VAE's composed encode / decode stage by stage at toy widths: padded (P = 35) and unpadded (P = 96) attention
    ("tests/test_vae_stages_gpu.py", ["test_stagewise_vae_matches_fp64[toy_40x56-encoder]",
                                      "test_stagewise_vae_matches_fp64[toy_40x56-decoder]",
                                      "test_stagewise_vae_matches_fp64[toy_64x96-encoder]",
                                      "test_stagewise_vae_matches_fp64[toy_64x96-decoder]"]),
    ("tests/test_vae_gpu.py", ["test_conv3x3_matches_torch[1-8-16-64-128-1]", "test_conv3x3_matches_torch[1-33-50-64-256-1]",
                               "test_conv3x3_matches_torch[1-32-48-128-128-2]", "test_groupnorm_silu_matches_torch_chain[1-48-32-1]"]),
]

if __name__ == "__main__":
    print(" ".join(f"{f}::{t}" for f, tests in WANT for t in tests))
