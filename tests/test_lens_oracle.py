"""The lens oracle (tests/lens_oracle.py) against independent restatements: COLMAP's OPENCV and OPENCV_FISHEYE
world-to-image in numpy, central finite differences of the map for J_D, the fisheye map's behaviour on and near the
optical axis, and rho_max against a dense scan of the radial derivative."""
import math

import numpy as np
import pytest
import torch

import lens_oracle as L

CASES = [("OPENCV", [-0.12, 0.03, 0.002, -0.001]), ("OPENCV", [0.2, -0.05, -0.01, 0.004]),
         ("FISHEYE", [0.05, -0.02, 0.004, -0.0005]), ("FISHEYE", [-0.3, 0.1, -0.02, 0.001]),
         ("PINHOLE", [0.0] * 4)]


def _colmap(u, v, model, k):
    """COLMAP's distortion, restated from its documented formulas (numpy fp64)."""
    if model == "OPENCV":
        k1, k2, p1, p2 = k
        r2 = u * u + v * v
        rad = k1 * r2 + k2 * r2 * r2
        return u + u * rad + 2 * p1 * u * v + p2 * (r2 + 2 * u * u), v + v * rad + 2 * p2 * u * v + p1 * (r2 + 2 * v * v)
    if model == "FISHEYE":
        r = np.hypot(u, v)
        th = np.arctan(r)
        th2 = th * th
        thd = th * (1 + k[0] * th2 + k[1] * th2 ** 2 + k[2] * th2 ** 3 + k[3] * th2 ** 4)
        s = np.where(r > 0, thd / np.where(r > 0, r, 1), 1.0)
        return u * s, v * s
    return u, v


def _points(n=400, lim=0.9, seed=0):
    rng = np.random.default_rng(seed)
    return rng.uniform(-lim, lim, n), rng.uniform(-lim, lim, n)


@pytest.mark.parametrize("model,k", CASES)
def test_map_matches_colmap(model, k):
    u, v = _points()
    ad, bd = L.lens_map(torch.from_numpy(u), torch.from_numpy(v), model, k)
    eu, ev = _colmap(u, v, model, k)
    assert np.abs(ad.numpy() - eu).max() < 1e-12 and np.abs(bd.numpy() - ev).max() < 1e-12
    # with intrinsics: pixel = f * distorted + c, and the stored mean is distorted + (c - W/2) / f
    fx, cx, W = 300.0, 70.25, 128
    ox = (cx - W / 2) / fx
    assert np.abs((ad.numpy() + ox) * fx + W / 2 - (fx * eu + cx)).max() < 1e-9


@pytest.mark.parametrize("model,k", CASES)
def test_jacobian_matches_finite_differences(model, k):
    u, v = _points(200, 0.8, 1)
    a, b = torch.from_numpy(u), torch.from_numpy(v)
    J = L.lens_jacobian(a, b, model, k)
    h = 1e-6
    for j, (da, db) in enumerate(((h, 0.0), (0.0, h))):
        p = L.lens_map(a + da, b + db, model, k)
        m = L.lens_map(a - da, b - db, model, k)
        for i in range(2):
            fd = (p[i] - m[i]) / (2 * h)
            assert (fd - J[:, i, j]).abs().max() < 1e-7, (i, j)


def test_fisheye_on_and_near_the_axis():
    k = [0.05, -0.02, 0.004, -0.0005]
    zero = torch.zeros(1, dtype=torch.float64)
    ad, bd = L.lens_map(zero, zero, "FISHEYE", k)
    J = L.lens_jacobian(zero, zero, "FISHEYE", k)
    assert float(ad) == 0.0 and float(bd) == 0.0
    assert torch.allclose(J[0], torch.eye(2, dtype=torch.float64))
    # continuous across the series threshold rho^2 = SERIES_R2: map and J_D on both sides agree to the series' error
    r = math.sqrt(L.SERIES_R2)
    for s in (1 - 1e-9, 1 + 1e-9):
        a = torch.tensor([r * s * 0.6], dtype=torch.float64)
        b = torch.tensor([r * s * 0.8], dtype=torch.float64)
        ad, bd = L.lens_map(a, b, "FISHEYE", k)
        eu, ev = _colmap(a.numpy(), b.numpy(), "FISHEYE", k)
        assert abs(float(ad) - eu[0]) < 1e-15 and abs(float(bd) - ev[0]) < 1e-15
    lo = L.lens_jacobian(torch.tensor([r * 0.6 * (1 - 1e-9)]), torch.tensor([r * 0.8 * (1 - 1e-9)]), "FISHEYE", k)
    hi = L.lens_jacobian(torch.tensor([r * 0.6 * (1 + 1e-9)]), torch.tensor([r * 0.8 * (1 + 1e-9)]), "FISHEYE", k)
    assert (lo - hi).abs().max() < 1e-10
    # the gradient through the map is finite on the axis
    a = torch.zeros(1, dtype=torch.float64, requires_grad=True)
    b = torch.zeros(1, dtype=torch.float64, requires_grad=True)
    ad, bd = L.lens_map(a, b, "FISHEYE", k)
    (ad + 2 * bd).sum().backward()
    assert float(a.grad) == pytest.approx(1.0) and float(b.grad) == pytest.approx(2.0)


@pytest.mark.parametrize("model,k", CASES + [("OPENCV", [-0.5, 0.0, 0.0, 0.0]), ("OPENCV", [0.0, -0.2, 0, 0]),
                                             ("FISHEYE", [0.0] * 4), ("FISHEYE", [-0.2, 0.0, 0.0, 0.0])])
def test_rho_max_against_a_dense_scan(model, k):
    rm = L.rho_max(model, k)
    if model == "PINHOLE":
        assert rm == math.inf
        return
    if model == "OPENCV":
        u = np.linspace(1e-6, 50.0, 2_000_001)            # rho^2
        d = 1 + 3 * k[0] * u + 5 * k[1] * u * u
        bad = np.nonzero(d <= 0)[0]
        want = math.sqrt(u[bad[0]]) if len(bad) else math.inf
    else:
        th = np.linspace(1e-6, math.pi / 2 - 1e-9, 2_000_001)
        t = th * th
        d = 1 + 3 * k[0] * t + 5 * k[1] * t ** 2 + 7 * k[2] * t ** 3 + 9 * k[3] * t ** 4
        bad = np.nonzero(d <= 0)[0]
        want = math.tan(th[bad[0]]) if len(bad) else math.inf
    if want == math.inf:
        assert rm == math.inf or rm > 6.0
    else:
        assert rm == pytest.approx(want, rel=1e-4)
