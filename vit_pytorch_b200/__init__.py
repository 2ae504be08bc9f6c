"""vit_pytorch_b200: a Hopper (sm_90a) native ViT encoder forward, drop-in for vit_pytorch.ViT / SimpleViT / NaViT.

    from vit_pytorch_b200 import ViT, SimpleViT      # same constructor keywords and state_dict as the reference

The fused path lives in csrc/ (CUDA, C ABI in include/b200vit.h) and is bound with ctypes (_lib.py).
"""
from .vit import ViT
from .simple_vit import SimpleViT
from .na_vit import NaViT           # padding-free fused path (varlen attention) + the reference's packed PyTorch graph
from .sep_vit import SepViT         # window attention with window tokens, then attention across windows

__all__ = ["ViT", "SimpleViT", "NaViT", "SepViT"]
__version__ = "0.1.0"
