"""imagdressing_b200 — H100-native (sm_90a) kernels + host mirror for the IMAGDressing-v1 denoising hot path.

Only what the path needs lives here: `csrc/` (CUDA kernels + the C ABI of include/imagd_b200.h), `_lib` / `ops`
(ctypes binding), and the host-side mirror of the reference interfaces (UNet / ControlNet hosts, attention
processors, pipelines, DDIM scheduler). See DESIGN.md.
"""
__version__ = "0.1.0"
