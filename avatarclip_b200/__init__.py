"""avatarclip_b200 -- H100-native (sm_90a) implementation of the AvatarCLIP appearance-optimisation
hot path behind the reference's own Python surface (AvatarGen/AppearanceGen):

    NeuSRenderer / SDFNetwork / RenderingNetwork / SingleVarianceNetwork   (models/renderer.py, fields.py)

All arithmetic runs in libavc_b200.so (hand-written CUDA, C ABI in include/avc_b200.h).  There is no
CPU or PyTorch fallback: importing is cheap, the first call fails loudly if the library is not built.
"""
from ._lib import AvcError, LIB_PATH
from .fields import RenderingNetwork, SDFNetwork, SingleVarianceNetwork
from .renderer import NeuSRenderer

__all__ = ["AvcError", "LIB_PATH", "NeuSRenderer", "SDFNetwork", "RenderingNetwork", "SingleVarianceNetwork"]
