"""council_gan_b200: the Council-GAN training step (dis / dis_council / gen updates) on H100.

Hand-written sm_90a CUDA kernels behind a C ABI (``libcouncil_b200.so``, declared in
``include/council_b200.h``) driven from a ``Council_Trainer`` that keeps the reference's API.
"""
from .trainer_council import Council_Trainer  # noqa: F401
from .utils import get_config  # noqa: F401

__all__ = ['Council_Trainer', 'get_config']
