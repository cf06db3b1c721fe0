"""dreammat_b200 -- H100-native (sm_90a) score-distillation inner loop for DreamMat.

The package holds only what the hot path needs: `csrc/` (CUDA kernels + the C-ABI of
include/dreammat_b200.h), thin torch-facing wrappers, and host-side mirrors of the five
threestudio plugins the path goes through (SURVEY.md section 8b).
"""
__version__ = "0.1.0"
