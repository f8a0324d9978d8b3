"""semseg_b200 — H100-native (sm_90a) implementation of the dense-prediction training hot path of
hszhao/semseg: PSPNet / PSANet on a dilated ResNet, hand-written CUDA behind a C-ABI (include/semseg_b200.h)."""
__version__ = "0.1.0"
