"""odise_b200: H100-native (sm_90a) engine for the ODISE open-vocabulary panoptic inference hot path.

Host side is Python (like the reference); all device arithmetic lives in libodise_b200.so (include/odise_b200.h),
hand-written CUDA for sm_90a: wgmma/TMA GEMM + implicit conv, wgmma flash attention, warp-shuffle
deformable / masked attention, fused elementwise passes.  No CPU or eager fallback exists."""
__version__ = "0.1.0"
