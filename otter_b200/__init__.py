"""otter_b200 — H100-native (sm_90a) implementation of Otter's vision-fusion hot path.

CLIP ViT patch encoder -> PerceiverResampler -> GatedCrossAttentionBlock, forward + backward, on
hand-written wgmma / TMA CUDA kernels behind a C ABI (include/otter_b200.h), with the reference's
module classes, forward() signatures and state-dict keys (otter_b200.modeling_otter).
"""
__version__ = "0.1.0"


def precision(mode):
    """Context manager: "bf16" (production: bf16 operands, fp32 accumulate) or "fp32" (forward-only parity mode,
    fp32-grade arithmetic — see otter_b200/fp32_path.py)."""
    from .fp32_path import precision as _p
    return _p(mode)
