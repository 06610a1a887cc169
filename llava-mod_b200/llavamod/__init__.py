"""llavamod -- H100-native drop-in for the LLaVA-MoD distillation step (mimic-KL + preference-DPO).

Same public surface as the reference's ``llavamod.model`` / ``llavamod.train`` for this path; device work is
hand-written sm_90a CUDA in ``liblmod_b200.so`` (see include/lmod.h), reached through ``llavamod._C``.
"""
from .constants import IGNORE_INDEX, IMAGE_TOKEN_INDEX  # noqa: F401

__version__ = "0.1.0"
