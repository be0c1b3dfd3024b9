"""CPU checks of the 2-D screen-space filter oracle (tests/filter_oracle.py) and of gs_ctx_set_filter2d's argument
validation.  The reference has no such filter, so the oracle is held to the unfiltered oracle, to the closed-form
screen-space integral of a Gaussian and to central finite differences."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

import aux_oracle as A
import filter_oracle as F
import gs_oracle as O
from helpers import scene

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "3d-gaussian-splatting_b200")
NAMES = ("pos", "rgb", "opa", "quat", "scale")


def _p(g, grad=False):
    return {k: t.double().clone().requires_grad_(grad) for k, t in g.items()}


def test_none_is_the_unfiltered_oracle_bit_for_bit():
    g, v, cam = scene(600, 96, 64, k=1, opa_range=(0.05, 0.9))
    p = _p(g)
    assert torch.equal(F.render(*(p[q] for q in NAMES), cam, "none"), O.render(*(p[q] for q in NAMES), cam))
    a = F.render_maps(*(p[q] for q in NAMES), cam, "none", background=(0.2, 0.5, 0.9))
    b = A.render_maps(*(p[q] for q in NAMES), cam, background=(0.2, 0.5, 0.9))
    for k in ("padded_image", "padded_depth", "padded_alpha"):
        assert torch.equal(a[k], b[k]), k


@pytest.mark.parametrize("mode", ["dilate", "antialias"])
def test_converges_to_unfiltered_as_variance_vanishes(mode):
    g, v, cam = scene(600, 96, 64, k=1, opa_range=(0.05, 0.9), sigma_px=(0.8, 5.0))
    p = _p(g)
    ref = F.render_maps(*(p[q] for q in NAMES), cam, "none")["padded_image"]
    errs = [float((F.render_maps(*(p[q] for q in NAMES), cam, mode, s)["padded_image"] - ref).abs().max())
            for s in (0.3, 3e-3, 3e-5)]
    assert errs[0] > 1e-3                                       # the filter does change the frame
    assert errs[1] < errs[0] / 20 and errs[2] < errs[1] / 20 and errs[2] < 1e-5, errs


def _single(sigma_px=3.0, opacity=0.01, w=32, h=32):
    """One isotropic Gaussian of sigma_px pixels at the image centre, camera at the origin looking down +z."""
    fx = fy = 40.0
    z = 5.0
    cam = O.Camera(w, h, fx, fy, torch.eye(3), torch.zeros(3))
    s = sigma_px * z / fx - 1e-4                                # abs activation adds 1e-4
    g = dict(pos=torch.tensor([[0.0, 0.0, z]]), rgb=torch.zeros(1, 3),
             opa=torch.tensor([math.log(opacity / (1 - opacity))]), quat=torch.tensor([[1.0, 0.0, 0.0, 0.0]]),
             scale=torch.full((1, 3), s))
    return g, cam


def test_single_gaussian_integral():
    """Sum of alpha over the image (a unit-pixel Riemann sum, exact to far below the tolerance for sigma = 3 px) against
    the closed form opa * 2 pi sqrt(det) fx fy px^2: antialias keeps it, dilate scales it by sqrt(det'/det)."""
    g, cam = _single(w=64, h=64)
    p = _p(g)
    nq, ns, _, _ = O.preactivate(p["quat"], p["scale"], p["opa"], p["rgb"])
    _, rc, _ = O.global_culling(p["pos"], nq, ns, cam.rot.double(), cam.tran.double(), cam.near, cam.half_w, cam.half_h)
    det = float(torch.linalg.det(rc[0]))
    ex, ey = F.filter_eps(cam, 0.3)
    c = rc[0].detach().numpy()
    detf = (c[0, 0] + ex) * (c[1, 1] + ey) - c[0, 1] * c[1, 0]
    opa = torch.sigmoid(p["opa"]).item()
    closed = opa * 2 * math.pi * math.sqrt(det) * cam.fx * cam.fy
    sums = {m: float(F.render_maps(*(p[q] for q in NAMES), cam, m)["padded_alpha"].sum()) for m in F.MODES}
    assert abs(sums["none"] / closed - 1) < 1e-6, sums
    assert abs(sums["antialias"] / closed - 1) < 1e-6, sums
    assert abs(sums["dilate"] / (closed * math.sqrt(detf / det)) - 1) < 1e-6, sums
    assert abs(math.sqrt(detf / det) - 9.3 / 9) < 1e-6                # sigma = 3 px: (9 + 0.3) / 9


def test_compensation_formula_of_the_kernels():
    """The device adds g_l2o * k to dL/dcov with k = ((d, -c, -b, a) / det - (d', -c, -b, a') / det') / (2 ln 2), the
    gradient of 0.5 log2(det / det') (gs_filter2d in csrc/project.cuh): central differences in fp64."""
    rng = np.random.default_rng(0)
    ex, ey = 0.01, 0.02
    for _ in range(20):
        m = rng.normal(size=(2, 2)) * 0.1
        cov = m @ m.T + np.eye(2) * 1e-3
        a, b, c, d = cov[0, 0], cov[0, 1], cov[1, 0], cov[1, 1]

        def l2o(a, b, c, d):
            return 0.5 * math.log2((a * d - b * c) / ((a + ex) * (d + ey) - b * c))

        det, detf = a * d - b * c, (a + ex) * (d + ey) - b * c
        k = np.array([d / det - (d + ey) / detf, -c / det + c / detf, -b / det + b / detf,
                      a / det - (a + ex) / detf]) / (2 * math.log(2))
        x, h = np.array([a, b, c, d]), 1e-7
        num = np.array([(l2o(*(x + h * e)) - l2o(*(x - h * e))) / (2 * h) for e in np.eye(4)])
        assert np.allclose(k, num, rtol=1e-5, atol=1e-5 * np.abs(num).max())


def _frozen_culling(base_pos, base_rot, base_tran):
    """global_culling with the projection Jacobian evaluated at a fixed (pos, rot, tran): the oracle detaches that
    Jacobian (rot stays live in JW = J rot), so this is the function whose differences match its autograd gradient."""
    culling = O.global_culling

    def f(pos, quat_n, scale_a, rot, tran, near, hw, hh):
        rp, _, mask = culling(pos, quat_n, scale_a, rot, tran, near, hw, hh)
        x, y, z = (base_pos @ base_rot.T + base_tran).unbind(-1)
        zero = torch.zeros_like(x)
        J = torch.stack([1 / z, zero, -x / (z * z), zero, 1 / z, -y / (z * z)], dim=-1).reshape(-1, 2, 3)
        RS = O.quat_to_rot(quat_n) * scale_a.unsqueeze(-2)
        JW = J @ rot
        cov2 = JW @ (RS @ RS.transpose(-1, -2)) @ JW.transpose(-1, -2)
        return rp, cov2 * mask.to(pos.dtype).reshape(-1, 1, 1), mask

    return f


@pytest.mark.parametrize("which", ["image", "alpha"])
def test_antialias_gradient_matches_finite_differences(which, monkeypatch):
    """Image and alpha-map losses of a small antialiased scene of sub-pixel to few-pixel Gaussians (compensation
    0.64 - 0.86): fp64 autograd against central differences in the five parameters and in rot / tran."""
    g, v, _ = scene(5, 32, 32, seed=7, opa_range=(0.2, 0.6), sigma_px=(0.4, 2.0))
    p = _p(g, True)
    rot = v.rot.double().clone().requires_grad_(True)
    tran = v.tran.double().clone().requires_grad_(True)
    w = torch.rand(32, 32, 3, generator=torch.Generator().manual_seed(11), dtype=torch.float64)

    def loss(q, r, t):
        cam = O.Camera(32, 32, v.fx, v.fy, r, t, v.near)
        out = F.render_maps(*(q[k] for k in NAMES), cam, "antialias", background=(0.2, 0.5, 0.9))
        return (out["image"] * w).sum() if which == "image" else (out["alpha"] * w[..., 0]).sum()

    cam0 = O.Camera(32, 32, v.fx, v.fy, rot, tran, v.near)
    nq, ns, opa_a, _ = O.preactivate(p["quat"], p["scale"], p["opa"], p["rgb"])
    _, rc, mask = O.global_culling(p["pos"], nq, ns, rot, tran, cam0.near, cam0.half_w, cam0.half_h)
    assert int(mask.sum()) == 5
    _, o_f, _ = F.filtered(rc, opa_a, cam0, "antialias")
    comp = (o_f / opa_a).detach()
    assert float(comp.min()) < 0.7 and float(comp.max()) < 0.9, comp  # the compensation really acts

    loss(p, rot, tran).backward()
    monkeypatch.setattr(O, "global_culling", _frozen_culling(p["pos"].detach().clone(), rot.detach().clone(),
                                                             tran.detach().clone()))
    eps = 1e-6
    leaves = dict(p, rot=rot, tran=tran)
    for name, leaf in leaves.items():
        ana = leaf.grad if leaf.grad is not None else torch.zeros_like(leaf)
        num = torch.zeros_like(ana)
        for i in range(leaf.numel()):
            vals = {k: t.detach().clone() for k, t in leaves.items()}
            vals[name].view(-1)[i] += eps
            lp = float(loss({k: vals[k] for k in NAMES}, vals["rot"], vals["tran"]))
            vals[name].view(-1)[i] -= 2 * eps
            lm = float(loss({k: vals[k] for k in NAMES}, vals["rot"], vals["tran"]))
            num.view(-1)[i] = (lp - lm) / (2 * eps)
        assert (float(ana.abs().max()) > 0) == (name != "rgb" or which == "image"), name
        err = float((ana - num).abs().max() / (num.abs().max() + 1e-12))
        assert err < 1e-5, (which, name, err)


def test_set_filter2d_rejects_bad_arguments_without_gpu():
    lib = ctypes.CDLL(os.path.join(PKG, "libgs_b200.so"))
    lib.gs_last_error.restype = ctypes.c_char_p
    lib.gs_ctx_set_filter2d.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_float]
    fake = 0x1000                                   # never dereferenced: every check precedes any use
    assert lib.gs_ctx_set_filter2d(None, 1, 0.3) == -1
    assert "null ctx" in lib.gs_last_error().decode()
    for mode in (-1, 3):
        assert lib.gs_ctx_set_filter2d(fake, mode, 0.3) == -1
        assert "mode must be" in lib.gs_last_error().decode()
    for mode in (0, 1, 2):
        for var in (0.0, -0.3, float("nan"), float("inf")):
            assert lib.gs_ctx_set_filter2d(fake, mode, var) == -1, (mode, var)
            assert "variance" in lib.gs_last_error().decode()
