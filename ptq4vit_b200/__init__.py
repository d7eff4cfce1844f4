"""ptq4vit_b200: H100-native (sm_90a) scale-factor search for PTQ4ViT's quant layers.

Host side mirrors the reference's operator surface (quant_layers.*, utils.quant_calib,
configs.PTQ4ViT.get_module); the arithmetic runs in hand-written CUDA behind the C ABI
declared in include/ptq4vit_b200.h.
"""
__version__ = "0.1.0"
