"""CPU checks of tools/eval_2d.py: checkpoints written by the reference (which pickle its top-level
``utils.BoundingBox``) load with the box mapped onto ``vmap_b200.utils.BoundingBox``."""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _tool():
    spec = importlib.util.spec_from_file_location("eval_2d", os.path.join(ROOT, "tools", "eval_2d.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_reference_bounding_box_is_remapped(tmp_path):
    from vmap_b200 import utils as vutils
    fake = types.ModuleType("utils")

    class BoundingBox:
        pass
    BoundingBox.__module__ = "utils"
    BoundingBox.__qualname__ = "BoundingBox"
    fake.BoundingBox = BoundingBox
    saved = sys.modules.get("utils")
    sys.modules["utils"] = fake
    try:
        b = BoundingBox()
        b.center, b.R, b.extent = np.zeros(3), np.eye(3), np.ones(3)
        torch.save({"obj_id": 3, "bbox": b, "obj_scale": 2.0}, str(tmp_path / "ck.pth"))
    finally:
        if saved is None:
            del sys.modules["utils"]
        else:
            sys.modules["utils"] = saved
    ck = _tool().load_checkpoint(str(tmp_path / "ck.pth"))
    assert type(ck["bbox"]) is vutils.BoundingBox
    assert np.array_equal(ck["bbox"].extent, np.ones(3)) and ck["obj_id"] == 3
