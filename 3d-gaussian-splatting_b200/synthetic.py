"""Seeded synthetic scenes and cameras shared by tests, golden scripts and bench.py.

Host-side helper only (CPU tensors; callers move them).  Definition: SURVEY.md §8(d)
"Synthetic scene generator": one `torch.Generator('cpu')` seeded `seed`; draw order
pos[N,3], scale[N,3], quat[N,4], opa[N], colour DC[N,3], SH higher-order[N,3,K-1];
`grad_output` from a second generator seeded `seed+1`.
Parameter conventions are the reference's (splatter.py:399-406): opa / rgb are logits,
quat is wxyz un-normalised, scale is the raw value fed to the `abs`(+1e-4) activation.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch

SH_C0 = 0.28209479177387814


@dataclass
class View:
    width: int
    height: int
    fx: float
    fy: float
    rot: torch.Tensor      # [3,3] world->camera
    tran: torch.Tensor     # [3]
    near: float = 0.3

    @property
    def padded_width(self):
        return int(math.ceil(self.width / 16)) * 16

    @property
    def padded_height(self):
        return int(math.ceil(self.height / 16)) * 16


def make_view(width: int, height: int, k: int = 0) -> View:
    """Camera k: 60 deg horizontal fov, orbiting the origin at distance 4 (R_y(k*45deg))."""
    fx = width / (2.0 * math.tan(math.radians(30.0)))
    ang = math.radians(45.0 * k)
    c, s = math.cos(ang), math.sin(ang)
    rot = torch.tensor([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]], dtype=torch.float32)
    tran = torch.tensor([0.0, 0.0, 4.0], dtype=torch.float32)
    return View(width, height, fx, fx, rot, tran)


def _logit(u):
    return torch.log(u) - torch.log1p(-u)


def make_gaussians(n: int, width: int, height: int, seed: int = 0, sh_dim: int = 3,
                   opa_range=(0.05, 0.9), sigma_px=(0.6, 5.0)):
    """Returns dict(pos, rgb, opa, quat, scale) of fp32 CPU tensors.

    sh_dim: 3 -> RGB logits [N,3]; 27 / 48 -> channel-major SH coefficients [N, sh_dim]
    (layout [c*K+k], gaussian.cu:942) with DC = logit/C0 (utils.py:345-348).
    """
    g = torch.Generator("cpu").manual_seed(seed)
    fx = width / (2.0 * math.tan(math.radians(30.0)))
    pos = (torch.rand(n, 3, generator=g) * 2 - 1) * torch.tensor([1.6, 1.6 * height / width, 1.0])
    lo, hi = math.log(sigma_px[0]), math.log(sigma_px[1])
    scale = torch.exp(torch.rand(n, 3, generator=g) * (hi - lo) + lo) * (4.0 / fx)
    quat = torch.randn(n, 4, generator=g)
    opa = _logit(torch.rand(n, generator=g) * (opa_range[1] - opa_range[0]) + opa_range[0])
    dc = _logit(torch.rand(n, 3, generator=g) * 0.96 + 0.02)
    if sh_dim == 3:
        rgb = dc
    else:
        k = sh_dim // 3
        hi_order = torch.randn(n, 3, k - 1, generator=g) * 0.1
        rgb = torch.cat([(dc / SH_C0).unsqueeze(-1), hi_order], dim=-1).reshape(n, sh_dim)
    return dict(pos=pos.float().contiguous(), rgb=rgb.float().contiguous(), opa=opa.float().contiguous(),
                quat=quat.float().contiguous(), scale=scale.float().contiguous())


def make_grad_output(height: int, width: int, seed: int = 0):
    """Upstream gradient of the (cropped) image: U(-1,1)/P, generator seeded seed+1."""
    g = torch.Generator("cpu").manual_seed(seed + 1)
    return ((torch.rand(height, width, 3, generator=g) * 2 - 1) / float(height * width)).float()


def appearance_jitter(images, strength: float, seed: int = 0):
    """Per-view photometric differences of strength S, as a camera that sets exposure and white balance per shot
    would make them: image k becomes clamp(e_k * wb_k * x, 0, 1) ** gamma_k with log e_k ~ N(0, (0.5 S)^2),
    log wb_k ~ N(0, (0.2 S)^2) per channel and log gamma_k ~ N(0, (0.3 S)^2), drawn from one CPU generator seeded
    `seed` in view order.  images: list of [H, W, 3] tensors; returns a new list."""
    g = torch.Generator("cpu").manual_seed(seed)
    out = []
    for x in images:
        e = math.exp(0.5 * strength * float(torch.randn(1, generator=g)))
        wb = torch.exp(0.2 * strength * torch.randn(3, generator=g))
        gamma = math.exp(0.3 * strength * float(torch.randn(1, generator=g)))
        out.append((x * (e * wb).to(x.device, x.dtype)).clamp(0.0, 1.0) ** gamma)
    return out
