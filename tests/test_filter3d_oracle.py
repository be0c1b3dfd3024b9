"""CPU checks of the 3-D smoothing filter oracle (tests/filter3d_oracle.py): a zero filter is the unfiltered
computation bit for bit, the filter keeps each Gaussian's 3-D integral, the oracle's gradients agree with central
finite differences and with the device's closed-form scale chain, and the sampling rate behaves as Mip-Splatting's on
hand-built cases."""
import itertools
import math

import numpy as np
import pytest
import torch

import filter3d_oracle as F3
import filter_oracle as F
import gs_oracle as O
from helpers import scene

NAMES = ("pos", "rgb", "opa", "quat", "scale")


def _p(g, grad=False):
    return {k: t.double().clone().requires_grad_(grad) for k, t in g.items()}


def _cam(z_axis_tran=0.0, fx=100.0, fy=100.0, w=200, h=100, near=0.3, rot=None):
    return dict(width=w, height=h, focal_x=fx, focal_y=fy, rot=np.eye(3) if rot is None else rot,
                tran=np.array([0.0, 0.0, z_axis_tran]), near=near)


@pytest.mark.parametrize("mode", F.MODES)
def test_zero_filter_is_the_unfiltered_oracle_bit_for_bit(mode):
    g, v, cam = scene(500, 96, 64, k=1)
    p = _p(g)
    ref = F.render(*(p[q] for q in NAMES), cam, mode)
    with F3.applied(torch.zeros(500, dtype=torch.float64)):
        got = F.render(*(p[q] for q in NAMES), cam, mode)
    assert torch.equal(got, ref)


@pytest.mark.parametrize("act", ["abs", "exp"])
def test_the_3d_integral_is_kept(act):
    gen = torch.Generator().manual_seed(3)
    raw = torch.randn(200, 3, generator=gen, dtype=torch.float64) * (0.5 if act == "exp" else 0.05) - (3 if act == "exp" else 0)
    s = raw.abs() + O.EPS if act == "abs" else torch.exp(raw)
    opa = torch.rand(200, generator=gen, dtype=torch.float64)
    f = torch.rand(200, generator=gen, dtype=torch.float64) * 0.05
    f[::7] = 0
    sf, of = F3.filtered(s, opa, f)
    assert torch.allclose(of * sf.prod(1), opa * s.prod(1), rtol=1e-12, atol=0)
    assert torch.equal(sf[::7], s[::7]) and torch.equal(of[::7], opa[::7])
    assert bool((sf >= s).all()) and bool((sf >= f.unsqueeze(1)).all())


@pytest.mark.parametrize("act", ["abs", "exp"])
def test_gradients_match_central_differences(act):
    g, v, cam = scene(40, 48, 32, k=1, opa_range=(0.3, 0.8), sigma_px=(1.0, 3.0))
    if act == "exp":
        g["scale"] = g["scale"].abs().clamp_min(1e-3).log()
    p = _p(g, grad=True)
    f3 = torch.full((40,), 0.004, dtype=torch.float64)
    f3[::3] = 0
    w = torch.rand(cam.height, cam.width, 3, generator=torch.Generator().manual_seed(1), dtype=torch.float64)

    def loss(q):
        with F3.applied(f3):
            return (F.render_maps(*(q[k] for k in NAMES), cam, "antialias", scale_activation=act)["image"] * w).sum()

    loss(p).backward()
    # scale and opacity: what the filter changes (pos's gradient detaches the projection Jacobian, as the reference's)
    for name, idx in (("scale", (5, 1)), ("scale", (7, 2)), ("scale", (9, 0)), ("opa", (4,)), ("opa", (6,))):
        eps = 1e-6
        qp = {k: t.detach().clone() for k, t in p.items()}
        qm = {k: t.detach().clone() for k, t in p.items()}
        qp[name][idx] += eps
        qm[name][idx] -= eps
        fd = float((loss(qp) - loss(qm)) / (2 * eps))
        if name == "scale" and act == "exp":                 # the reference's clamped derivative of exp
            x = float(p["scale"][idx])
            fd *= math.exp(min(max(x, -1.0), 1.0)) / math.exp(x)
        ad = float(p[name].grad[idx])
        assert abs(fd - ad) <= 1e-5 * max(1.0, abs(fd)), (name, idx, fd, ad)


def test_closed_form_scale_chain_is_autograd_of_the_filtered_activation():
    gen = torch.Generator().manual_seed(5)
    s = (torch.rand(64, 3, generator=gen, dtype=torch.float64) * 0.1 + 1e-3).requires_grad_(True)
    f = torch.rand(64, generator=gen, dtype=torch.float64) * 0.03
    f[::5] = 0
    opa = torch.rand(64, generator=gen, dtype=torch.float64) * 0.9 + 0.05
    sf, of = F3.filtered(s, opa, f)
    g_sf = torch.randn(64, 3, generator=gen, dtype=torch.float64)
    g_l2o = torch.randn(64, generator=gen, dtype=torch.float64)
    (g_sf * sf).sum().backward(retain_graph=True)
    (g_l2o * torch.log2(of)).sum().backward()
    got = F3.scale_grad(g_sf.numpy(), g_l2o.numpy(), s.detach().numpy(), f.numpy())
    assert np.allclose(got, s.grad.numpy(), rtol=1e-12, atol=1e-12)


def test_one_view_at_depth_z():
    pos = np.array([[0.0, 0.0, 4.0], [0.1, -0.2, 9.0]])
    f, seen = F3.sampling_filter(pos, [_cam(fx=250.0)], variance=0.2)
    assert seen.all()
    assert np.allclose(f, math.sqrt(0.2) * pos[:, 2] / 250.0, rtol=1e-15)


def test_margin_boundary_is_inclusive():
    # u = fx x / z + W / 2 = -m W exactly at x = -(m + 0.5) W z / fx (values exact in binary)
    w, fx, z, m = 200, 100.0, 2.0, 0.25
    x_edge = -(m + 0.5) * w * z / fx
    pos = np.array([[x_edge, 0.0, z], [x_edge - 1e-3, 0.0, z], [-x_edge, 0.0, z], [-x_edge + 2 * w * z / fx * 0.0, 0.0, z]])
    pos[2, 0] = (1 + m - 0.5) * w * z / fx                   # u = (1 + m) W exactly
    pos[3, 0] = pos[2, 0] + 1e-3
    f, seen = F3.sampling_filter(pos, [_cam(fx=fx, w=w)], margin=m)
    assert seen.tolist() == [True, False, True, False]


def test_near_plane():
    pos = np.array([[0.0, 0.0, 0.3], [0.0, 0.0, 0.31], [0.0, 0.0, -1.0]])
    f, seen = F3.sampling_filter(pos, [_cam(near=0.3)])
    assert seen.tolist() == [False, True, False]


def test_unseen_gaussians_get_the_largest_filter():
    pos = np.array([[0.0, 0.0, 2.0], [0.0, 0.0, 5.0], [100.0, 0.0, 3.0]])
    f, seen = F3.sampling_filter(pos, [_cam()], variance=0.1)
    assert seen.tolist() == [True, True, False]
    assert f[2] == f[1] == max(f)


def test_no_seen_gaussian_gives_zeros():
    pos = np.array([[0.0, 0.0, -2.0], [50.0, 0.0, 1.0]])
    f, seen = F3.sampling_filter(pos, [_cam()])
    assert not seen.any() and (f == 0).all()


def test_the_finest_view_wins_and_the_order_of_views_does_not_matter():
    gen = np.random.default_rng(0)
    pos = gen.normal(size=(300, 3)) * [1.5, 1.0, 1.0] + [0, 0, 6]
    cams = []
    for k in range(6):
        a = 0.15 * (k - 2.5)
        rot = np.array([[math.cos(a), 0, math.sin(a)], [0, 1, 0], [-math.sin(a), 0, math.cos(a)]])
        cams.append(_cam(z_axis_tran=0.5 * k, fx=80.0 + 15 * k, fy=80.0 + 15 * k, rot=rot))
    f, seen = F3.sampling_filter(pos, cams)
    for perm in itertools.islice(itertools.permutations(range(6)), 0, 720, 97):
        g, s2 = F3.sampling_filter(pos, [cams[i] for i in perm])
        assert np.array_equal(f, g) and np.array_equal(seen, s2)


def test_projected_covariance_is_at_least_the_variance_in_the_finest_view():
    # in the view attaining nu_i every filtered Gaussian's 2-D covariance has lambda_min >= v px^2 (J J^T >= I / z^2)
    g, v, cam = scene(400, 96, 64, k=0, sigma_px=(0.05, 0.5))
    pos = g["pos"].double()
    view = dict(width=cam.width, height=cam.height, focal_x=cam.fx, focal_y=cam.fx, rot=cam.rot.numpy(),
                tran=cam.tran.numpy(), near=cam.near)
    var = 0.2
    f, seen = F3.sampling_filter(pos.numpy(), [view], margin=0.0, variance=var)
    nq, ns, _, _ = O.preactivate(g["quat"].double(), g["scale"].double(), g["opa"].double(), g["rgb"].double())
    sf, _ = F3.filtered(ns, torch.ones(400, dtype=torch.float64), torch.from_numpy(f))
    c = O.Camera(cam.width, cam.height, cam.fx, cam.fx, cam.rot, cam.tran, cam.near)
    rp, rc, mask = O.global_culling(pos, nq, sf, c.rot.double(), c.tran.double(), c.near, 1e9, 1e9)
    ok = torch.from_numpy(seen) & mask.bool()
    assert int(ok.sum()) > 100
    lam = torch.linalg.eigvalsh(rc[ok]).min(dim=1).values * cam.fx ** 2
    assert float(lam.min()) >= var * (1 - 1e-9)
