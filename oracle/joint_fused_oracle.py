"""fp16-faithful restatement (torch, fp64) of the joint map-and-pose step at hidden 32 (``vmb_joint_step_fused``).

TEST INFRASTRUCTURE ONLY -- see ``oracle/__init__.py``.

The step is three kernels in a row; each is restated by code that already lives here, none copied:

- ``k_joint_world`` (``vmap_b200/csrc/k_track_lw.cuh``): each camera-frame point q moves to the world by the pose of its
  ray's draw, ``pose_point(T_f, q, 1.0f)`` in fp32 and in its fma order -- ``track_fused_oracle.posed_points`` at
  scale 1 (with ``proj32`` off the fp64 ``R q + t``).  A ray whose frame is outside the table keeps ``p = q``.  The
  caller can pass the kernel's own points (``world=``, from ``pcs_world_out``).
- ``k_step_fused<S, true>`` (``vmap_b200/csrc/k_step_fused.cuh``): the mapping step on those points,
  ``fused_oracle.fused_step`` with its ``Rounding`` switches and the mapping loss's whole-batch empty-mask rule (a term
  is off for every object when one object's count of it is 0).  Its ``pe_backward`` also forms each point's
  ``dL/dt = INV_LS (dE1_xyz + dproj @ dirs)`` from the fp32 ``dproj``, not from the fp16 block the dB wgrad reads, and
  from the PE directions before this launch's AdamW (``fused_step``'s ``aux["dt"]``).
- ``k_joint_rows`` / ``pose_terms`` (``vmap_b200/csrc/k_track.cuh``): ``g = dt / scale[b]``; the row of a ray is the sum
  over its samples of ``((R q) x g, g)``, R from the fp64 pose and q the fp32 camera point widened to fp64; a ray
  without a frame gets a zero row.  ``pose_rows`` is this stage alone, so a caller can form rows from any ``dt``.

Inputs the kernel decides per ray are taken as given, as ``fused_step`` takes them: ``emb`` (the kernel's embedding,
``tests/test_fused_faithful_gpu.probe_embedding``), ``signs``, ``var`` and ``counts``.  With ``ROUND_OFF`` and no empty
mask the per-frame sums of the rows are ``ba_oracle.evaluate``'s gradient (``tests/test_joint_fused_oracle.py``): the
loss of a ray depends on its own pose only, and both losses normalise by the counts of the whole slice.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch

from . import fused_oracle as fo
from . import track_fused_oracle as tfo

Rounding = fo.Rounding
ROUND_ALL = fo.ROUND_ALL
ROUND_OFF = fo.ROUND_OFF


def _frames(frames, B: int, R: int, dev) -> torch.Tensor:
    return torch.as_tensor(frames, dtype=torch.int64).reshape(B, R).to(dev)


def world_points(poses, frames, q: torch.Tensor, fp32: bool = True) -> torch.Tensor:
    """[B,R,S,3] fp64 world points of the camera-frame points q [B,R,S,3] (``k_joint_world``): ``pose_point`` at scale 1
    in fp32 (or fp64 with ``fp32`` off); a ray whose frame is -1 keeps q."""
    B, R = q.shape[:2]
    qc = q.detach().to("cpu", torch.float64)
    t, _ = tfo.posed_points(poses, _frames(frames, B, R, "cpu"), qc, 1.0, fp32)
    ok = (_frames(frames, B, R, "cpu") >= 0)[..., None, None]
    return torch.where(ok, t, qc).to(q.device)


def pose_rows(dt: torch.Tensor, scale, q: torch.Tensor, poses, frames) -> torch.Tensor:
    """[B,R,6] fp64 rows (``k_joint_rows``): the sum over each ray's samples of ``((R_f q) x g, g)``, g = dt / scale[b],
    from dt [B,R*S,3] or [B,R,S,3] and the camera-frame points q [B,R,S,3]; zero where the ray's frame is -1."""
    B, R, S, _ = q.shape
    dev = q.device
    f64 = dict(dtype=torch.float64, device=dev)
    T = tfo._pose_table(poses).to(dev)
    fr = _frames(frames, B, R, dev)
    ok = fr >= 0
    rq = torch.einsum("brij,brsj->brsi", T[fr.clamp(min=0)][..., :3, :3], q.to(**f64))
    sc = torch.as_tensor(scale, **f64).expand(B).reshape(B, 1, 1, 1)
    g = dt.to(**f64).reshape(B, R, S, 3) / sc
    pt = torch.cat([torch.cross(rq, g, dim=-1), g], -1) * ok[..., None, None]
    return pt.sum(2)


def frame_grads(rows: torch.Tensor, frames, n_frames: int) -> torch.Tensor:
    """[F,6] the rows summed per frame (rays without a frame add nothing)."""
    B, R = rows.shape[:2]
    fr = _frames(frames, B, R, rows.device).reshape(-1)
    ok = fr >= 0
    g = torch.zeros(n_frames, 6, dtype=torch.float64, device=rows.device)
    g.index_add_(0, fr[ok], rows.reshape(-1, 6)[ok])
    return g


def evaluate(params: Dict[str, torch.Tensor], scale, batch: Dict[str, torch.Tensor], poses, frames,
             world: Optional[torch.Tensor] = None, emb: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
             signs: Optional[torch.Tensor] = None, var: Optional[torch.Tensor] = None,
             counts: Optional[torch.Tensor] = None, rounding: Rounding = ROUND_ALL) -> dict:
    """One joint step of a stack of B hidden-32 objects.

    params: stacked ``[B, *shape]`` weights (those the launch reads, before its AdamW); scale: scalar or [B];
    batch: the step inputs with ``pcs`` [B,R,S,3] camera-frame points; poses: [F,4,4] fp64; frames: [B,R] each ray's
    row of ``poses`` (-1: none); world: [B,R,S,3] the world points to use (default: ``world_points``, fp32 under
    ``proj32``); emb, signs, var, counts, rounding: as ``fused_oracle.fused_step``.

    Returns dict(rows [B,R,6], grad [F,6], render (D, V, C, O), terms [B,4], grads {key: [B, *shape]}, world
    [B,R,S,3], dt [B,R*S,3], dproj [B,R*S,21] (before its fp16 pack)), all fp64."""
    q = batch["pcs"]
    if world is None:
        world = world_points(poses, frames, q, rounding.proj32)
    aux = {}
    render, terms, grads = fo.fused_step(params, scale, dict(batch, pcs=world.to(q.device)), counts=counts,
                                         signs=signs, emb=emb, var=var, rounding=rounding, aux=aux)
    rows = pose_rows(aux["dt"], scale, q, poses, frames)
    return {"rows": rows, "grad": frame_grads(rows, frames, tfo._pose_table(poses).shape[0]), "render": render,
            "terms": terms, "grads": grads, "world": world, "dt": aux["dt"], "dproj": aux["dproj"]}
