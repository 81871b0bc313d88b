"""fastervit_b200 — H100-native (sm_90a) FasterViT forward/backward behind the reference's API.

    from fastervit_b200 import create_model
    model = create_model('faster_vit_0_224').cuda().eval()
    logits = model(images)          # runs on libfvit_sm100.so kernels; CPU tensors raise
"""
from .registry import create_model, list_models, is_model, model_entrypoint, load_checkpoint  # noqa: F401
from .model import FasterViT  # noqa: F401
from .optim import FusedAdamW, FusedLamb, FlatEma, param_groups_weight_decay  # noqa: F401

__all__ = ["create_model", "list_models", "is_model", "model_entrypoint", "load_checkpoint", "FasterViT",
           "FusedAdamW", "FusedLamb", "FlatEma", "param_groups_weight_decay"]
