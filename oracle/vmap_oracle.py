"""CPU restatement (torch, fp32 or fp64) of vMAP's vectorised training step.

TEST INFRASTRUCTURE ONLY -- see ``oracle/__init__.py``.  Parity is pinned by
``tests/golden/*.npz`` (generated from the reference's own modules by
``oracle/make_golden.py``) and replayed by ``tests/test_oracle_golden.py``.

Every function cites the reference lines it follows (paths relative to the
reference tree).  The ensemble is held as a dict of *stacked* tensors
``[n_obj, *shape]`` keyed by the reference's ``state_dict`` names, which is
what ``functorch.combine_state_for_ensemble`` produces (utils.py:30-34).
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import torch

# named_parameters() order of OccupancyMap (model.py:17-52) -- also the order of
# ``fc_param`` in train.py:181,335-336.
FC_KEYS = (
    "in_layer.0.weight", "in_layer.0.bias",
    "mid1.0.0.weight", "mid1.0.0.bias",
    "cat_layer.0.weight", "cat_layer.0.bias",
    "mid2.0.0.weight", "mid2.0.0.bias",
    "out_alpha.weight", "out_alpha.bias",
    "color_linear.0.weight", "color_linear.0.bias",
    "out_color.weight", "out_color.bias",
)
PE_KEY = "B_layer.weight"            # embedding.py:75-76 (trainable)
ALL_KEYS = FC_KEYS + (PE_KEY,)

N_DIRS = 21
_G = 0.8506508
_S = 0.5257311
_A = 0.809017
_B = 0.309017


def icosahedron_dirs(dtype=torch.float32) -> torch.Tensor:
    """The 21 unit directions used as the initial PE projection (embedding.py:51-73)."""
    rows = [
        (_G, 0, _S), (_A, .5, _B), (_S, _G, 0), (1, 0, 0), (_A, .5, -_B), (_G, 0, -_S),
        (_B, _A, -.5), (0, _S, -_G), (.5, _B, -_A), (0, 1, 0), (-_S, _G, 0), (-_B, _A, -.5),
        (0, _S, _G), (-_B, _A, .5), (_B, _A, .5), (.5, _B, _A), (.5, -_B, _A), (0, 0, 1),
        (-.5, _B, _A), (-_A, .5, _B), (-_A, .5, -_B),
    ]
    return torch.tensor(rows, dtype=dtype)


def emb_sizes(max_deg: int = 5) -> Tuple[int, int]:
    """(emb_size1, emb_size2) as in trainer.py:16-17 (87, 42 for max_deg=5)."""
    e1 = N_DIRS * (3 + 1) + 3
    return e1, N_DIRS * (max_deg + 1) + 3 - e1


def param_shapes(hidden: int, max_deg: int = 5) -> Dict[str, Tuple[int, ...]]:
    e1, e2 = emb_sizes(max_deg)
    h = hidden
    return {
        "in_layer.0.weight": (h, e1), "in_layer.0.bias": (h,),
        "mid1.0.0.weight": (h, h), "mid1.0.0.bias": (h,),
        "cat_layer.0.weight": (h, h + e1), "cat_layer.0.bias": (h,),
        "mid2.0.0.weight": (h, h), "mid2.0.0.bias": (h,),
        "out_alpha.weight": (1, h), "out_alpha.bias": (1,),
        "color_linear.0.weight": (h, h + e2), "color_linear.0.bias": (h,),
        "out_color.weight": (3, h), "out_color.bias": (3,),
        PE_KEY: (N_DIRS, 3),
    }


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


def _blinear(x: torch.Tensor, w: torch.Tensor, b: Optional[torch.Tensor]) -> torch.Tensor:
    """Per-object ``F.linear``: x [B,N,K], w [B,O,K], b [B,O] (what vmap lowers
    ``torch.nn.Linear`` to: one batched GEMM, SURVEY.md 2a)."""
    if b is None:
        return torch.bmm(x, w.transpose(1, 2))
    return torch.baddbmm(b.unsqueeze(1), x, w.transpose(1, 2))


def unidir_embed(pcs: torch.Tensor, dirs: torch.Tensor, scale: torch.Tensor,
                 max_deg: int = 5) -> torch.Tensor:
    """UniDirsEmbed.forward for a stack of objects (embedding.py:82-91).

    pcs [B,R,S,3], dirs [B,21,3], scale [B] -> [B,R,S,3+21*(max_deg+1)];
    feature order: xyz/scale, then frequency-major sin(pi*2^k*proj_d)."""
    B, R, S, _ = pcs.shape
    t = (pcs / scale.view(B, 1, 1, 1)).reshape(B, R * S, 3)                 # :83
    proj = _blinear(t, dirs, None)                                            # :84
    freqs = 2.0 ** torch.linspace(0, max_deg, max_deg + 1, dtype=pcs.dtype, device=pcs.device)   # :78
    bands = proj.unsqueeze(-2) * freqs.view(1, 1, -1, 1)                      # :85
    feat = torch.sin(bands.reshape(B, R * S, -1) * math.pi)                   # :86-88
    return torch.cat([t, feat], dim=-1).reshape(B, R, S, -1)                  # :89


def occupancy_mlp(emb: torch.Tensor, p: Dict[str, torch.Tensor], max_deg: int = 5
                  ) -> Tuple[torch.Tensor, torch.Tensor]:
    """OccupancyMap.forward for a stack of objects (model.py:54-85).
    emb [B,R,S,E] -> alpha [B,R,S,1] (already x10, :77), colour [B,R,S,3]."""
    B, R, S, E = emb.shape
    e1, _ = emb_sizes(max_deg)
    x = emb.reshape(B, R * S, E)
    x1, x2 = x[..., :e1], x[..., e1:]
    fc1 = torch.relu(_blinear(x1, p["in_layer.0.weight"], p["in_layer.0.bias"]))           # :59
    fc2 = torch.relu(_blinear(fc1, p["mid1.0.0.weight"], p["mid1.0.0.bias"]))              # :60
    fc3 = torch.relu(_blinear(torch.cat((fc2, x1), -1),
                              p["cat_layer.0.weight"], p["cat_layer.0.bias"]))             # :63-64
    fc4 = torch.relu(_blinear(fc3, p["mid2.0.0.weight"], p["mid2.0.0.bias"]))              # :67
    alpha = _blinear(fc4, p["out_alpha.weight"], p["out_alpha.bias"]) * 10.0               # :71,77
    hc = torch.relu(_blinear(torch.cat((fc4, x2), -1),
                             p["color_linear.0.weight"], p["color_linear.0.bias"]))        # :81
    colour = torch.sigmoid(_blinear(hc, p["out_color.weight"], p["out_color.bias"]))       # :82-83
    return alpha.reshape(B, R, S, 1), colour.reshape(B, R, S, 3)


def termination(alpha: torch.Tensor) -> torch.Tensor:
    """occupancy_activation + occupancy_to_termination(is_batch=True)
    (render_rays.py:4-8, 26-34): w_s = occ_s * prod_{j<s}(1 - occ_j + 1e-10)."""
    occ = torch.sigmoid(alpha)
    free = (1.0 - occ + 1e-10)[..., :-1]
    free = torch.cat([torch.ones_like(occ[..., :1]), free], dim=-1)
    return occ * torch.cumprod(free, dim=-1)


def render_outputs(alpha: torch.Tensor, colour: torch.Tensor, z: torch.Tensor):
    """Rendered depth, variance, colour, opacity (loss.py:23-32, render_rays.py:47-51).
    alpha [B,R,S,1] or [B,R,S]; colour [B,R,S,3]; z [B,R,S]."""
    if alpha.dim() == 4:
        alpha = alpha.squeeze(-1)
    w = termination(alpha)
    depth = (w * z).sum(-1)
    var = (w * (z - depth[..., None]) ** 2).sum(-1)
    col = (w[..., None] * colour).sum(-2)
    opa = w.sum(-1)
    return depth, var, col, opa


class LossExplode(RuntimeError):
    """The reference prints 'loss explode' and exit(-1)s (render_rays.py:88-90)."""


def _masked_mean(loss_mat, mask, info=None):
    """reduce_batch_loss(avg=True, mask=...) (render_rays.py:67-96) incl. the
    whole-batch early-out when ANY object has an empty mask (:68-73)."""
    cnt = mask.sum(-1)
    if bool((cnt == 0).any()):
        return torch.zeros_like(loss_mat).mean(-1)
    if info is not None:
        loss_mat = loss_mat * info
    out = loss_mat.sum(-1) / (cnt + 1e-10)
    if bool((out > 100000).any()):
        raise LossExplode("loss explode")
    return out


def batch_loss_terms(alpha, colour, gt_depth, gt_colour, sem, mask_depth, z):
    """Per-object (L_depth, L_colour, L_opacity), each [B] (loss.py:5-56)."""
    m_obj = sem != 0                                                    # loss.py:16
    m_sem = sem != 2                                                    # loss.py:18
    depth, var, col, opa = render_outputs(alpha, colour, z)
    var = var.detach()                                                  # loss.py:29
    m_d = mask_depth.bool() & m_obj                                     # loss.py:38
    l_d = _masked_mean((depth - gt_depth).abs() * m_d, m_d,
                       info=1.0 / (torch.sqrt(var) + 1e-4))              # render_rays.py:74-80
    l_c = _masked_mean((col - gt_colour).abs().sum(-1) * m_obj, m_obj)  # loss.py:43-46
    l_o = _masked_mean((opa - m_obj.to(opa.dtype)).abs() * m_sem, m_sem)  # loss.py:53-56
    return l_d, l_c, l_o


def step_batch_loss(alpha, colour, gt_depth, gt_colour, sem, mask_depth, z,
                    colour_scaling: float = 5.0, opacity_scaling: float = 10.0):
    """loss.step_batch_loss (loss.py:5-62); argument order as called at
    train.py:303-306 (labels before the depth mask)."""
    l_d, l_c, l_o = batch_loss_terms(alpha, colour, gt_depth, gt_colour, sem, mask_depth, z)
    return (l_d + l_c * colour_scaling + l_o * opacity_scaling).sum()


def forward(params: Dict[str, torch.Tensor], scale: torch.Tensor, pcs: torch.Tensor,
            max_deg: int = 5):
    """vmap(pe_model) then vmap(fc_model) (train.py:293-294)."""
    emb = unidir_embed(pcs, params[PE_KEY], scale, max_deg)
    return occupancy_mlp(emb, params, max_deg)


class OracleEnsemble:
    """Stacked ensemble + torch.optim.AdamW exactly as the reference drives it:
    one optimiser over the stacked leaves (train.py:67, utils.py:33), lr /
    weight-decay from the config (room0_vMAP.json:10-11), step + zero_grad
    (train.py:324-326)."""

    def __init__(self, params: Dict[str, torch.Tensor], scale, max_deg: int = 5,
                 lr: float = 1e-3, weight_decay: float = 0.013):
        self.params = {k: v.detach().clone().requires_grad_(True) for k, v in params.items()}
        b = next(iter(self.params.values())).shape[0]
        dt = next(iter(self.params.values())).dtype
        self.scale = torch.as_tensor(scale, dtype=dt).expand(b).clone() if not torch.is_tensor(scale) \
            or scale.dim() == 0 else scale.to(dt)
        self.max_deg = max_deg
        self.opt = torch.optim.AdamW([self.params[k] for k in ALL_KEYS if k in self.params],
                                     lr=lr, weight_decay=weight_decay)

    def forward(self, pcs):
        return forward(self.params, self.scale, pcs, self.max_deg)

    def loss(self, batch) -> torch.Tensor:
        alpha, colour = self.forward(batch["pcs"])
        return step_batch_loss(alpha, colour, batch["gt_depth"], batch["gt_colour"],
                               batch["sem"], batch["mask_depth"], batch["z"])

    def loss_terms(self, batch) -> torch.Tensor:
        """Per-object [B,4]: L_depth, L_colour, L_opacity and the weighted total (loss.py:57-60), what the kernels
        write into ``loss_terms``."""
        with torch.no_grad():
            alpha, colour = self.forward(batch["pcs"])
            l_d, l_c, l_o = batch_loss_terms(alpha, colour, batch["gt_depth"], batch["gt_colour"], batch["sem"],
                                             batch["mask_depth"], batch["z"])
            return torch.stack([l_d, l_c, l_o, l_d + 5.0 * l_c + 10.0 * l_o], dim=1)

    def grads(self, batch):
        self.opt.zero_grad(set_to_none=True)
        loss = self.loss(batch)
        loss.backward()
        return loss.detach(), {k: v.grad.detach().clone() for k, v in self.params.items()}

    def step(self, batch) -> torch.Tensor:
        loss = self.loss(batch)
        loss.backward()
        self.opt.step()
        self.opt.zero_grad(set_to_none=True)
        return loss.detach()

    def render(self, batch):
        with torch.no_grad():
            alpha, colour = self.forward(batch["pcs"])
            return render_outputs(alpha, colour, batch["z"])


def adamw_math(p, g, m, v, t: int, lr=1e-3, wd=0.013, b1=0.9, b2=0.999, eps=1e-8):
    """Closed form of one torch.optim.AdamW step (what train.py:325 executes),
    used to check the fused Adam kernel in fp64. Returns (p, m, v)."""
    p = p * (1 - lr * wd)
    m = m + (g - m) * (1 - b1)
    v = v * b2 + (1 - b2) * g * g
    bc1 = 1 - b1 ** t
    bc2 = 1 - b2 ** t
    denom = v.sqrt() / math.sqrt(bc2) + eps
    return p - (lr / bc1) * (m / denom), m, v


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
