"""Import the UNMODIFIED reference modules from a checkout of the reference (golden generators only;
set VMAP_REFERENCE_ROOT to its directory, default: ``reference`` beside this repository).

TEST INFRASTRUCTURE ONLY.  The reference's non-numeric imports (open3d, trimesh,
skimage, imgviz, bidict) are absent from this image; they are replaced by
MagicMock / a 10-line bidict stand-in so that ``vmap.sceneObject`` and
``trainer.Trainer`` import (SURVEY.md section 8c).  None of the stubbed modules
takes part in the arithmetic of the hot path.
"""
from __future__ import annotations

import importlib
import os
import sys
import types
from unittest.mock import MagicMock

REF_ROOT = os.environ.get("VMAP_REFERENCE_ROOT") or os.path.join(
    os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))), "reference")


def available() -> bool:
    return os.path.isfile(os.path.join(REF_ROOT, "render_rays.py"))


class _Inv:
    def __init__(self, owner):
        self._o = owner

    def __setitem__(self, value, key):
        for k in [k for k, v in self._o.items() if v == value]:
            dict.__delitem__(self._o, k)
        dict.__setitem__(self._o, key, value)

    def __getitem__(self, value):
        for k, v in self._o.items():
            if v == value:
                return k
        raise KeyError(value)


class _Bidict(dict):
    @property
    def inv(self):
        return _Inv(self)


def load(*names):
    """Return the named reference modules (e.g. ``load('model', 'loss')``)."""
    if not available():
        raise RuntimeError(f"reference tree not found at {REF_ROOT}")
    for stub in ("open3d", "trimesh", "skimage", "skimage.measure", "imgviz"):
        if stub not in sys.modules:
            try:
                importlib.import_module(stub)
            except Exception:
                sys.modules[stub] = MagicMock()
    if "bidict" not in sys.modules:
        try:
            importlib.import_module("bidict")
        except Exception:
            mod = types.ModuleType("bidict")
            mod.bidict = _Bidict
            sys.modules["bidict"] = mod
    # the reference is a flat tree of top-level modules whose names collide with
    # ours (model, loss, vmap ...): import them under their own names from
    # REF_ROOT, then drop REF_ROOT from sys.path again.
    sys.path.insert(0, REF_ROOT)
    try:
        out = []
        for n in names:
            if n in sys.modules and getattr(sys.modules[n], "__file__", "").startswith(REF_ROOT):
                out.append(sys.modules[n])
            else:
                sys.modules.pop(n, None)
                out.append(importlib.import_module(n))
    finally:
        sys.path.remove(REF_ROOT)
    return out[0] if len(out) == 1 else tuple(out)
