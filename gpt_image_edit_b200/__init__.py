"""H100-native FLUX-Kontext denoising engine (hot path of wyhlovecpp/GPT-Image-Edit).

Python here is host glue over the C ABI in include/b2f.h (libb2f.so, hand-written sm_90a CUDA).
"""
__all__ = ["ops"]
