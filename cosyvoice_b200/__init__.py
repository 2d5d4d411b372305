"""H100-native CosyVoice2 hot path: hand-written sm_90a kernels behind the C ABI of include/cvk.h."""
__version__ = "0.1"
