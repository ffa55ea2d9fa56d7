"""sliders_b200 — H100-native (sm_90a) concept-slider UNet denoise path.

Public surface mirrors rohitgandikota/sliders (trainscripts/textsliders): `LoRANetwork`, `LoRAModule`,
`train_util.predict_noise(_xl)`, `diffusion(_xl)`; the arithmetic runs in hand-written CUDA kernels behind
the C ABI in include/sb200.h.  Importing the package does not load the extension; the first kernel call does,
and fails loudly if libsb200.so is missing.
"""
__version__ = "0.1.0"
