"""Synthetic Replica-shaped inputs and reference-distribution initial weights for benchmarks and demos.

Product-side utilities (bench.py, tools/): random ensembles with the reference's init distribution
(xavier-normal weights, torch.nn.Linear default biases, icosahedron PE directions; model.py:4-6,
trainer.py:32, embedding.py:51-76) and training batches whose sample depths follow the reference's
depth-guided strategy (vmap.py:366-459) in closed form.  No oracle code is imported here.

``sphere_room_sequence`` renders a posed RGB-D + instance + class sequence of spheres in a room in closed form (fp64,
on the host) for SLAM tests and timing; ``write_replica`` stores it in the directory layout ``dataset.Replica``
reads and ``write_scannet`` in the one ``dataset.ScanNet`` reads.
"""
from __future__ import annotations

import math
import os
from typing import Dict

import numpy as np
import torch

from .embedding import ICOSAHEDRON_DIRS
from .layout import PE_KEY, tensor_shapes


def icosahedron_dirs(dtype=torch.float32) -> torch.Tensor:
    return torch.tensor(ICOSAHEDRON_DIRS, dtype=dtype)


def param_shapes(hidden: int, max_deg: int = 5):
    return tensor_shapes(hidden, max_deg)


def init_params(n_obj: int, hidden: int, max_deg: int = 5, seed: int = 0,
                dtype=torch.float32) -> Dict[str, torch.Tensor]:
    """Random ensemble with the reference's init distribution: xavier-normal
    weights (model.py:4-6, trainer.py:32), torch.nn.Linear default bias
    U(-1/sqrt(fan_in), 1/sqrt(fan_in)), PE = icosahedron (embedding.py:76)."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k, shp in param_shapes(hidden, max_deg).items():
        if k == PE_KEY:
            out[k] = icosahedron_dirs(dtype).expand(n_obj, -1, -1).clone()
        elif k.endswith("weight"):
            fan_out, fan_in = shp
            std = math.sqrt(2.0 / (fan_in + fan_out))
            out[k] = (torch.randn((n_obj,) + shp, generator=g) * std).to(dtype)
        else:
            wshape = param_shapes(hidden, max_deg)[k[:-4] + "weight"]
            bound = 1.0 / math.sqrt(wshape[1])
            out[k] = ((torch.rand((n_obj,) + shp, generator=g) * 2 - 1) * bound).to(dtype)
    return out



def synthetic_batch(n_obj: int, n_rays: int, n_samples: int, seed: int = 0,
                    n_cam2surf: int = 1, dtype=torch.float32, empty_prob=(0.1, 0.3, 0.6, 0.1)):
    """Replica-shaped synthetic training batch (BASELINE.md section 3 / SURVEY.md 8d):
    depth U(0.5,4.5) with 10% invalid, labels p=(0.3,0.6,0.1), z drawn with the
    reference's depth-guided strategy (vmap.py:366-459) in closed form, pcs = o + d*z."""
    g = torch.Generator().manual_seed(seed)
    B, R, S = n_obj, n_rays, n_samples
    n1 = n_cam2surf
    n2 = S - n1
    depth = torch.rand(B, R, generator=g) * 4.0 + 0.5
    invalid = torch.rand(B, R, generator=g) < empty_prob[0]
    depth = torch.where(invalid, torch.zeros_like(depth), depth)
    u = torch.rand(B, R, generator=g)
    sem = torch.where(u < empty_prob[1], 0, torch.where(u < empty_prob[1] + empty_prob[2], 1, 2)).to(torch.uint8)
    rgb = torch.randint(0, 256, (B, R, 3), generator=g).to(torch.float32) / 255.0
    eps, other_eps = 0.1, 0.05
    maxb = depth.max(dim=1, keepdim=True).values
    ur = torch.rand(B, R, S, generator=g)
    lin1 = torch.arange(n1).view(1, 1, -1)
    lin2 = torch.arange(n2).view(1, 1, -1)
    linS = torch.arange(S).view(1, 1, -1)
    z = torch.empty(B, R, S)
    hi = (depth - eps)[..., None]
    z[..., :n1] = (lin1 + ur[..., :n1]) * hi / n1
    nrm = (torch.randn(B, R, n2, generator=g) * (eps / 3)).sort(-1).values.clamp(-eps, eps)
    z_this = depth[..., None] + nrm
    z_other = (depth - eps)[..., None] + (lin2 + ur[..., n1:]) * (eps + other_eps) / n2
    z[..., n1:] = torch.where((sem == 1)[..., None], z_this, z_other)
    z_inv = (linS + ur) * maxb[..., None] / S
    z = torch.where(invalid[..., None], z_inv, z)
    origin = (torch.rand(B, R, 3, generator=g) - 0.5)
    px = torch.rand(B, R, 2, generator=g)
    dirs = torch.stack([(px[..., 0] * 1200 - 599.5) / 600.0, (px[..., 1] * 680 - 339.5) / 600.0,
                        torch.ones(B, R)], -1)
    pcs = origin[..., None, :] + dirs[..., None, :] * z[..., None]
    return {
        "pcs": pcs.to(dtype).contiguous(), "z": z.to(dtype).contiguous(),
        "gt_depth": depth.to(dtype).contiguous(), "gt_colour": rgb.to(dtype).contiguous(),
        "sem": sem.contiguous(), "mask_depth": (~invalid).contiguous(),
    }


# ---- a synthetic RGB-D sequence: spheres in a room ---------------------------------------------------------------------

SPHERE_CLASS = 3                                    # not one of Replica's background classes (dataset.py:69)
ROOM_CLASSES = (93, 93, 31, 40, 93, 93)             # wall, wall, ceiling, floor, wall, wall: background classes
ROOM_IDS = tuple(range(20, 26))
# the room: x in [-3, 3], y in [-1.5, 1.5] (y points down: the floor is y = 1.5), z in [-2, 5]; planes n . p = h
ROOM_PLANES = ((1, 0, 0, -3.0), (1, 0, 0, 3.0), (0, 1, 0, -1.5), (0, 1, 0, 1.5), (0, 0, 1, -2.0), (0, 0, 1, 5.0))


def _rot(axis: int, a: float) -> np.ndarray:
    c, s = math.cos(a), math.sin(a)
    i, j = [(1, 2), (2, 0), (0, 1)][axis]
    R = np.eye(3)
    R[i, i], R[i, j], R[j, i], R[j, j] = c, -s, s, c
    return R


def sphere_room_scene(half_fov_x: float, n_extra: int = 0) -> list:
    """Spheres ``(instance id, centre [3], radius)``: ids 1-3 in front of the first camera, id 4 just outside its
    horizontal field of view (half angle ``half_fov_x`` radians) on the side the camera path turns to, and
    ``n_extra`` small spheres (ids 5, 6, ...) on a grid in front of the far wall."""
    r, D = 0.35, 3.0
    a = half_fov_x + math.asin(r / D) + math.radians(8.0)
    out = [(1, np.array([-0.6, 0.3, 2.5]), 0.35), (2, np.array([0.5, 0.4, 3.0]), 0.4),
           (3, np.array([0.0, -0.35, 2.2]), 0.25), (4, np.array([D * math.sin(a), 0.1, D * math.cos(a)]), r)]
    for j in range(n_extra):
        out.append((5 + j, np.array([-1.5 + 0.6 * (j % 6), -0.9 + 0.6 * (j // 6 % 4), 4.3 - 0.1 * (j // 24)]), 0.2))
    return out


def sphere_room_path(n_frames: int, yaw_deg: float = 25.0) -> np.ndarray:
    """Camera-to-world poses [N, 4, 4] fp64 along a smooth path: a yaw of ``yaw_deg`` towards +x with a small pitch
    wave, while the camera moves 0.4 m along x, 0.1 m along z and waves 5 cm in y.  Frame 0 is the identity."""
    T = np.tile(np.eye(4), (n_frames, 1, 1))
    for k in range(n_frames):
        s = k / max(n_frames - 1, 1)
        yaw = math.radians(yaw_deg) * (s + 0.05 * math.sin(2 * math.pi * s))
        pitch = math.radians(2.0) * math.sin(math.pi * s)
        T[k, :3, :3] = _rot(1, yaw) @ _rot(0, pitch)
        T[k, :3, 3] = [0.4 * s, 0.05 * math.sin(math.pi * s), 0.1 * s]
    return T


def sphere_room_colour(p: np.ndarray, inst: np.ndarray) -> np.ndarray:
    """Colour in [0, 1] as a smooth, non-constant function of the world position ``p`` [..., 3], with a per-instance
    phase so neighbouring surfaces differ."""
    ph = 0.7 * inst[..., None].astype(np.float64)
    f = np.array([[2.1, 0.7, 1.3], [0.9, 2.3, 0.5], [1.1, 1.7, 2.6]])
    return 0.5 + 0.4 * np.sin(p @ f.T + ph + np.array([0.0, 2.0, 4.0]))


def render_sphere_room(T_wc: np.ndarray, W: int, H: int, fx: float, fy: float, cx: float, cy: float, spheres):
    """Exact images of the scene from camera-to-world pose ``T_wc``, all [W, H] as everywhere in the package: z-depth
    fp64 (the ray parameter along ((u - cx) / fx, (v - cy) / fy, 1)), colour fp64 in [0, 1], instance and class int32.
    Each pixel takes the nearest positive hit of every sphere (|o + z d - c| = r) and room plane (n . (o + z d) = h)."""
    T = np.asarray(T_wc, np.float64)
    u = (np.arange(W, dtype=np.float64) - cx) / fx
    v = (np.arange(H, dtype=np.float64) - cy) / fy
    dc = np.stack(np.broadcast_arrays(u[:, None], v[None, :], np.ones((1, 1))), -1)     # [W, H, 3]
    d = dc @ T[:3, :3].T
    o = T[:3, 3]
    depth = np.full((W, H), np.inf)
    inst = np.zeros((W, H), np.int32)
    cls = np.zeros((W, H), np.int32)
    for (n0, n1, n2, h), i, c in zip(ROOM_PLANES, ROOM_IDS, ROOM_CLASSES):
        n = np.array([n0, n1, n2], np.float64)
        den = d @ n
        with np.errstate(divide="ignore", invalid="ignore"):
            z = (h - n @ o) / den
        hit = (den != 0) & (z > 0) & (z < depth)
        depth[hit], inst[hit], cls[hit] = z[hit], i, c
    for i, ctr, r in spheres:
        oc = o - ctr
        a = np.einsum("whk,whk->wh", d, d)
        b = d @ oc
        disc = b * b - a * (oc @ oc - r * r)
        with np.errstate(invalid="ignore"):
            z = (-b - np.sqrt(disc)) / a
        hit = (disc >= 0) & (z > 0) & (z < depth)
        depth[hit], inst[hit], cls[hit] = z[hit], i, SPHERE_CLASS
    p = o + depth[..., None] * d
    return depth, sphere_room_colour(p, inst), inst, cls


def sphere_room_sequence(n_frames: int, W: int, H: int, fx: float, fy: float, cx: float, cy: float,
                         yaw_deg: float = 25.0, n_extra: int = 0) -> dict:
    """The synthetic sequence: ``poses`` [N, 4, 4] fp64 (GT camera-to-world), ``depth`` [N, W, H] fp64, ``rgb``
    [N, W, H, 3] uint8 (the colour rounded), ``inst`` / ``cls`` [N, W, H] int32, ``spheres`` and the room's
    ``background_cls``.  Spheres are instances 1-4 of class ``SPHERE_CLASS``; the room's planes are instances 20-25 of
    background classes, which the ingest relabels to the background (0).  Sphere 4 comes into view partway;
    ``n_extra`` adds small spheres (``sphere_room_scene``).  ``intrinsics`` is (fx, fy, cx, cy)."""
    spheres = sphere_room_scene(math.atan((W / 2) / fx), n_extra)
    poses = sphere_room_path(n_frames, yaw_deg)
    out = {k: [] for k in ("depth", "rgb", "inst", "cls")}
    for T in poses:
        depth, col, inst, cls = render_sphere_room(T, W, H, fx, fy, cx, cy, spheres)
        out["depth"].append(depth)
        out["rgb"].append(np.clip(np.round(col * 255.0), 0, 255).astype(np.uint8))
        out["inst"].append(inst)
        out["cls"].append(cls)
    seq = {k: np.stack(v) for k, v in out.items()}
    seq.update(poses=poses, spheres=spheres, background_cls=sorted(set(ROOM_CLASSES)), intrinsics=(fx, fy, cx, cy))
    return seq


def write_replica(root: str, seq: dict, depth_scale: float = 1.0 / 1000.0) -> None:
    """Write ``seq`` in the layout ``dataset.Replica`` reads (dataset.py:63-89,135): ``rgb/rgb_{i}.png`` (BGR, as cv2
    writes), ``depth/depth_{i}.png`` uint16 in units of ``depth_scale`` metres, ``semantic_instance/`` and
    ``semantic_class/`` uint16, images stored [H, W] (the loader transposes them back), and ``traj_w_c.txt`` with
    one row-major 4 x 4 pose per line."""
    import cv2
    for d in ("rgb", "depth", "semantic_instance", "semantic_class"):
        os.makedirs(os.path.join(root, d), exist_ok=True)
    for i in range(len(seq["poses"])):
        cv2.imwrite(os.path.join(root, "rgb", f"rgb_{i}.png"), cv2.cvtColor(seq["rgb"][i].transpose(1, 0, 2),
                                                                          cv2.COLOR_RGB2BGR))
        dq = np.clip(np.round(seq["depth"][i] / depth_scale), 0, 65535).astype(np.uint16)
        cv2.imwrite(os.path.join(root, "depth", f"depth_{i}.png"), dq.T)
        cv2.imwrite(os.path.join(root, "semantic_instance", f"semantic_instance_{i}.png"),
                    seq["inst"][i].astype(np.uint16).T)
        cv2.imwrite(os.path.join(root, "semantic_class", f"semantic_class_{i}.png"), seq["cls"][i].astype(np.uint16).T)
    np.savetxt(os.path.join(root, "traj_w_c.txt"), np.asarray(seq["poses"]).reshape(-1, 16), delimiter=" ")


# ScanNet classes of the scene (dataset.py:187's background list holds 1, 3 and 41; 5 is not in it)
SCANNET_ROOM_CLASSES = (1, 1, 41, 3, 1, 1)          # wall, wall, ceiling, floor, wall, wall
SCANNET_SPHERE_CLASS = 5


def scannet_classes(inst: np.ndarray) -> np.ndarray:
    """The ScanNet class image ``write_scannet`` writes for the instance image ``inst`` of the sphere room."""
    cls = np.full(inst.shape, SCANNET_SPHERE_CLASS, np.int32)
    for i, c in zip(ROOM_IDS, SCANNET_ROOM_CLASSES):
        cls[inst == i] = c
    return cls


def write_scannet(root: str, seq: dict, mw: int = 10, inf_frames=(), depth_scale: float = 1.0 / 1000.0,
                  color_size=(1296, 968)) -> None:
    """Write the sphere-room sequence ``seq`` (``sphere_room_sequence``) in the layout ``dataset.ScanNet`` reads
    (dataset.py:150-262): every frame is rendered again at (W + 2 mw) x (H + 2 mw) with the principal point moved by
    ``mw``, so the loader's edge crop of ``mw`` pixels gives back ``seq``'s camera and images.  Files: ``color/{i}.jpg``
    at ``color_size`` (the loader resizes it to the depth size), ``depth/{i}.png`` uint16 in units of ``depth_scale``
    metres, ``instance-filt/{i}.png`` the instance id - 1 (the loader adds 1, so its ids are ``seq``'s),
    ``label-filt/{i}.png`` the ScanNet class (``scannet_classes``: the room's planes get background classes, the
    spheres a class that is not one), ``pose/{i}.txt`` the camera-to-world pose (every entry inf for the frames in
    ``inf_frames``, as ScanNet marks frames without a pose) and ``intrinsic/intrinsic_depth.txt`` (4 x 4)."""
    import cv2
    fx, fy, cx, cy = seq["intrinsics"]
    W, H = seq["depth"].shape[1:3]
    Wf, Hf = W + 2 * mw, H + 2 * mw
    for d in ("color", "depth", "instance-filt", "label-filt", "pose", "intrinsic"):
        os.makedirs(os.path.join(root, d), exist_ok=True)
    K = np.eye(4)
    K[0, 0], K[1, 1], K[0, 2], K[1, 2] = fx, fy, cx + mw, cy + mw
    np.savetxt(os.path.join(root, "intrinsic", "intrinsic_depth.txt"), K)
    inf_frames = set(int(i) for i in inf_frames)
    for i, T in enumerate(seq["poses"]):
        depth, col, inst, _ = render_sphere_room(T, Wf, Hf, fx, fy, cx + mw, cy + mw, seq["spheres"])
        rgb = np.clip(np.round(col * 255.0), 0, 255).astype(np.uint8)
        bgr = cv2.cvtColor(rgb.transpose(1, 0, 2), cv2.COLOR_RGB2BGR)
        cv2.imwrite(os.path.join(root, "color", f"{i}.jpg"), cv2.resize(bgr, color_size, interpolation=cv2.INTER_LINEAR))
        dq = np.clip(np.round(depth / depth_scale), 0, 65535).astype(np.uint16)
        cv2.imwrite(os.path.join(root, "depth", f"{i}.png"), dq.T)
        cv2.imwrite(os.path.join(root, "instance-filt", f"{i}.png"), np.maximum(inst - 1, 0).astype(np.uint16).T)
        cv2.imwrite(os.path.join(root, "label-filt", f"{i}.png"), scannet_classes(inst).astype(np.uint16).T)
        P = np.full((4, 4), np.inf) if i in inf_frames else np.asarray(T, np.float64)
        with open(os.path.join(root, "pose", f"{i}.txt"), "w") as f:
            f.write("\n".join(" ".join(repr(float(x)) for x in row) for row in P) + "\n")
