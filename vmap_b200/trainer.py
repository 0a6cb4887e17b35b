"""Trainer with the reference's attributes (trainer.py:9-33): ``fc_occ_map``, ``pe``,
``obj_scale``, ``hidden_feature_size``, ``emb_size1``, ``emb_size2``, ``bound_extent``;
``eval_points`` runs the batched forward-only kernel (trainer.py:77-95) and ``meshing`` the
marching-cubes kernels (trainer.py:35-75)."""
from __future__ import annotations

import numpy as np
import torch

from . import embedding, model
from .lazy import ensemble_for_modules


class Trainer:
    def __init__(self, cfg):
        self.obj_id = cfg.obj_id
        self.device = cfg.training_device
        self.hidden_feature_size = cfg.hidden_feature_size
        self.obj_scale = cfg.obj_scale
        self.n_unidir_funcs = cfg.n_unidir_funcs
        self.emb_size1 = 21 * (3 + 1) + 3
        self.emb_size2 = 21 * (self.n_unidir_funcs + 1) + 3 - self.emb_size1
        self.load_network()
        self.bound_extent = 0.995 if self.obj_id == 0 else 0.9

    def load_network(self):
        self.fc_occ_map = model.OccupancyMap(self.emb_size1, self.emb_size2, hidden_size=self.hidden_feature_size)
        self.fc_occ_map.apply(model.init_weights).to(self.device)
        self.pe = embedding.UniDirsEmbed(max_deg=self.n_unidir_funcs, scale=self.obj_scale).to(self.device)

    def eval_points(self, points, chunk_size=100000):
        """(occupancy [N], colour [N,3]) or None when everything is empty (trainer.py:77-95).
        ``chunk_size`` bounds the points per launch (at least 131072: the kernel tiles internally)."""
        ens = ensemble_for_modules(self.fc_occ_map, self.pe)
        row = self.fc_occ_map._vmb_binding[1]
        pts = points.to(ens.device, torch.float32).reshape(-1, 3).contiguous()
        # one-row call: only THIS object's network runs, however many objects share the packed stack
        alpha, colour = ens.eval_points(pts, row=row, chunk=max(int(chunk_size), 1 << 17))
        occ = torch.sigmoid(alpha)
        if float(occ.max()) == 0:
            print("no occ")
            return None
        return occ, colour

    def meshing(self, bound, obj_center, grid_dim=256):
        """Mesh of the object inside ``bound`` (trainer.py:35-75): occupancy of the network on a grid_dim^3 grid
        spanning the box, marching cubes at level 0.5 on the GPU (K5) with the grid -> world map folded into the
        kernel, and vertex colours from a second ``eval_points`` on the vertices.  Returns a mesh.Mesh, or None
        where the reference does ("no occ", no crossing).  ``bound``: anything with ``center``, ``R``, ``extent``."""
        from . import mesh as mesh_mod
        D = int(grid_dim)
        R = np.asarray(bound.R, dtype=np.float64)
        center = np.asarray(bound.center, dtype=np.float64)
        scene_scale_np = np.asarray(bound.extent, dtype=np.float64) / (2.0 * self.bound_extent)
        scene_scale = torch.from_numpy(scene_scale_np).float().to(self.device)
        transform_np = np.eye(4, dtype=np.float32)
        transform_np[:3, 3] = center
        transform_np[:3, :3] = R
        transform = torch.from_numpy(transform_np).to(self.device)
        grid_pc = make_3D_grid(occ_range=(-1., 1.), dim=D, device=self.device, scale=scene_scale,
                               transform=transform).view(-1, 3)
        grid_pc -= torch.as_tensor(obj_center).to(grid_pc.device)
        ret = self.eval_points(grid_pc)
        if ret is None:
            return None
        occ, _ = ret
        # grid index i -> R (scene_scale * (2 i / (D - 1) - 1)) + center (the [-1, 1] shift and scalings of
        # trainer.py:60-65, applied by the kernel as it writes each vertex)
        affine = np.concatenate([R @ np.diag(scene_scale_np) * (2.0 / (D - 1)), (center - R @ scene_scale_np)[:, None]], 1)
        out = mesh_mod.marching_cubes(occ.view(D, D, D), 0.5, affine)
        if out is None:
            print("marching cube failed")
            return None
        verts, faces, normals = out
        ret = self.eval_points(verts)
        if ret is None:
            return None
        _, colour = ret
        rgb = (colour * 255).to(torch.uint8)                 # truncation, like astype(np.uint8)
        rgba = torch.cat([rgb, torch.full_like(rgb[:, :1], 255)], 1)
        return mesh_mod.Mesh(verts.cpu().numpy(), faces.cpu().numpy(), normals.cpu().numpy(), rgba.cpu().numpy())


def make_3D_grid(occ_range=(-1., 1.), dim=256, device="cuda:0", transform=None, scale=None):
    """render_rays.make_3D_grid (render_rays.py:98-122): dim^3 query points."""
    t = torch.linspace(occ_range[0], occ_range[1], steps=dim, device=device)
    g = torch.stack(torch.meshgrid(t, t, t, indexing="ij"), dim=-1)
    if scale is not None:
        g = g * scale
    if transform is not None:
        g = g @ transform[:3, :3].T + transform[:3, 3]
    return g
