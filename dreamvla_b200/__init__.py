"""dreamvla_b200 -- H100-native (sm_90a) implementation of the DreamVLA transformer forward/backward hot path.

Hot ops are hand-written CUDA kernels in libdvla_sm90.so (C ABI: include/dvla.h), driven from
torch.autograd.Function wrappers in dreamvla_b200.ops.  There is no CPU / PyTorch fallback for the kernels.
"""
__version__ = "0.1.0"
