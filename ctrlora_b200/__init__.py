"""ctrlora_b200 — H100-native (sm_90a) implementation of CtrLoRA's denoising hot path.

`ctrlora_b200.csrc`     hand-written CUDA kernels + the C ABI (include/ctrlora_b200.h)
`ctrlora_b200.ops`      tensor-level wrappers over the C ABI
`ctrlora_b200.dropin`   host-side mirror of the reference's `cldm` / `ldm.modules` module contract
"""
__version__ = "0.1.0"
