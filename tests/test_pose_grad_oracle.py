"""CPU checks of the camera gradients of the fp64 oracle, and of the argument validation of gs_render_backward_cam.

The oracle (oracle/gs_oracle.py, composed with tests/aux_oracle.py and tests/sh_gaussian_oracle.py) already
differentiates through rot / tran when they are leaf tensors of O.Camera, with the semantics the fused path keeps for
pos: the projection Jacobian is detached, rot stays live in JW = J rot.  Nothing else computes camera gradients here, so
these tests hold the oracle to two exact invariances of the frame:

  translation: moving every mean by d equals t -> t + R d (the SH view direction moves with them), so
               dL/dt = R sum_i dL/dpos_i
  rotation:    rotating the world by Q with R -> R Q^T leaves an RGB frame of isotropic Gaussians unchanged, so for
               w = e_x, e_y, e_z:  sum_i dL/dpos_i . (w x pos_i) = <dL/dR, R [w]x>_F
"""
import ctypes
import math
import os

import pytest
import torch

import aux_oracle as A
import gs_oracle as O
import sh_gaussian_oracle as G
from helpers import scene

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "3d-gaussian-splatting_b200")
BG = (0.2, 0.5, 0.9)


def _skew(w):
    x, y, z = w
    return torch.tensor([[0.0, -z, y], [z, 0.0, -x], [-y, x, 0.0]], dtype=torch.float64)


def _pose(v):
    """Camera 1 of synthetic.make_view (R_y(45 deg), t = (0, 0, 4)) with a small extra tilt, built in fp64 so that the
    rotation is orthonormal to fp64 precision (the invariances need R^T R = I), as leaf tensors."""
    rot = torch.linalg.matrix_exp(_skew((0.05, -0.08, 0.03))) @ torch.linalg.matrix_exp(_skew((0.0, math.pi / 4, 0.0)))
    return rot.clone().requires_grad_(True), v.tran.double().clone().requires_grad_(True)


def _loss(sh, which, p, cam, seed=3):
    """Scalar loss of one output of the frame under a seeded random upstream gradient."""
    if which == "image" and not sh:
        out = O.render(p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], cam)
    elif which == "image":
        out = G.render(p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], cam)
    else:
        f = G.render_maps if sh else A.render_maps
        out = f(p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], cam, background=BG)[which]
    w = torch.rand(out.shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64) * 2 - 1
    return (out * w).sum()


def _grads(g, v, sh, which):
    rot, tran = _pose(v)
    cam = O.Camera(v.width, v.height, v.fx, v.fy, rot, tran, v.near)
    p = {k: t.double().clone().requires_grad_(True) for k, t in g.items()}
    _loss(sh, which, p, cam).backward()
    return p, rot, tran


@pytest.mark.parametrize("sh_dim,which", [(3, "image"), (3, "depth"), (3, "alpha"), (27, "image"), (48, "image"),
                                          (48, "depth"), (27, "alpha")])
def test_translation_identity(sh_dim, which):
    g, v, _ = scene(400, 64, 48, k=1, sh_dim=sh_dim, opa_range=(0.05, 0.9))
    p, rot, tran = _grads(g, v, sh_dim != 3, which)
    gsum = p["pos"].grad.sum(0)
    want = rot.detach() @ gsum
    assert float(tran.grad.abs().max()) > 1e-3 * float(p["pos"].grad.abs().max())
    scale = float(p["pos"].grad.abs().sum())
    assert float((tran.grad - want).abs().max()) < 1e-10 * scale, (tran.grad, want)
    assert rot.grad is not None and bool(torch.isfinite(rot.grad).all())


@pytest.mark.parametrize("which", ["image", "depth", "alpha"])
def test_rotation_identity(which):
    g, v, _ = scene(400, 64, 48, k=1, sh_dim=3, opa_range=(0.05, 0.9))
    g["scale"] = g["scale"][:, :1].repeat(1, 3).contiguous()     # isotropic: the Gaussians have no orientation
    p, rot, tran = _grads(g, v, False, which)
    pos, gpos, R = p["pos"].detach(), p["pos"].grad, rot.detach()
    seen = 0.0
    for w in torch.eye(3, dtype=torch.float64):
        lhs = float((gpos * torch.cross(w.expand_as(pos), pos, dim=-1)).sum())
        rhs = float((rot.grad * (R @ _skew(w.tolist()))).sum())
        seen = max(seen, abs(rhs))
        assert abs(lhs - rhs) < 1e-10 * float((gpos.abs() * pos.norm(dim=-1, keepdim=True)).sum()), (w, lhs, rhs)
    assert seen > 0


def test_backward_cam_rejects_bad_arguments_without_gpu():
    lib = ctypes.CDLL(os.path.join(PKG, "libgs_b200.so"))
    lib.gs_last_error.restype = ctypes.c_char_p
    P, I = ctypes.c_void_p, ctypes.c_int
    lib.gs_render_backward_cam.argtypes = [P, P, P, P, P, P, P, P, I, P, P, P, P, P, P, P, P, P]
    fake = 0x1000                                   # never dereferenced: every check below precedes any use
    grads = [fake] * 5

    def call(ctx, grads, grad_cam):
        return lib.gs_render_backward_cam(ctx, None, None, None, None, None, fake, fake, 0, None, None, *grads,
                                          grad_cam, None)

    assert call(None, grads, fake) == -1
    assert "null ctx" in lib.gs_last_error().decode()
    assert call(None, [None] * 5, fake) == -1
    assert "null ctx" in lib.gs_last_error().decode()
    assert call(fake, grads, None) == -1
    assert "null grad_cam" in lib.gs_last_error().decode()
    for k in range(5):
        partial = list(grads)
        partial[k] = None
        assert call(fake, partial, fake) == -1
        assert "all NULL or all non-NULL" in lib.gs_last_error().decode()
