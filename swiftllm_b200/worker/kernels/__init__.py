"""Drop-in replacements for `swiftllm/worker/kernels/*`: same function names, argument order and in-place
semantics as the reference wrappers, backed by the sm_90a C-ABI library (no Triton, no fallback)."""
