"""esvit_b200 - an H100-native (sm_90a) implementation of EsViT's multi-crop self-distillation training step
behind the reference's own module signatures (SwinTransformer.forward(list_of_crops) / MultiCropWrapper /
DINOHead / DINOLoss / DDINOLoss).  See DESIGN.md and INTEGRATION.md."""
__all__ = ["ops", "swin_transformer", "vision_transformer", "losses", "utils", "engine"]
