"""vmap_b200 -- H100-native (sm_90a) implementation of vMAP's vectorised per-object training step.

Only what the hot path needs lives here: the CUDA kernels + C ABI (csrc/, libvmap_b200.so),
the packed ensemble / fused step driver (ensemble.py) and the host-side mirror of the
reference's call surface (cfg, model, embedding, trainer, loss, utils, vmap).
"""
from . import _lib  # noqa: F401
from .layout import ALL_KEYS, FC_KEYS, PE_KEY  # noqa: F401

__all__ = ["ALL_KEYS", "FC_KEYS", "PE_KEY"]
