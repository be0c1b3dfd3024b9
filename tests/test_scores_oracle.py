"""The fp64 blend-weight score oracle (tests/scores_oracle.py) against independent statements of what it scores: a
lone Gaussian's alpha, a front Gaussian's transmittance, the early stop of a saturated tile, the crop, and the alpha
map's sum.  CPU only."""
import math

import torch

import aux_oracle as A
import filter_oracle as F
import scores_oracle as SO
from helpers import scene

FX = FY = 40.0


def _one_tile_per_instance(pos, opa, cov, Hp, Wp):
    """Every Gaussian in every tile, in index order: (sorted pos, opa, cov, accum, gauss_idx)."""
    n = pos.shape[0]
    T = (Hp // 16) * (Wp // 16)
    gidx = torch.arange(n).repeat(T)
    accum = torch.arange(T + 1, dtype=torch.int64) * n
    return pos[gidx], opa[gidx], cov[gidx], accum, gidx


def _alpha(pos, opa, cov, Hp, Wp):
    """[Hp, Wp] alpha of one Gaussian: opa exp(-x^T cov^-1 x / 2), written without `draw`'s expression."""
    x = (torch.arange(Wp, dtype=torch.float64) + 0.5 - Wp // 2) / FX - pos[0]
    y = (torch.arange(Hp, dtype=torch.float64) + 0.5 - Hp // 2) / FY - pos[1]
    X, Y = x.reshape(1, -1), y.reshape(-1, 1)
    ci = torch.inverse(cov)
    q = ci[0, 0] * X * X + (ci[0, 1] + ci[1, 0]) * X * Y + ci[1, 1] * Y * Y
    return opa * torch.exp(-0.5 * q)


def _cov(sx, sy, rho=0.0):
    return torch.tensor([[sx * sx, rho * sx * sy], [rho * sx * sy, sy * sy]], dtype=torch.float64)


def test_single_gaussian_sum_and_peak():
    Hp = Wp = 48
    pos = torch.tensor([[0.05, -0.03, 2.0]], dtype=torch.float64)
    cov = _cov(0.12, 0.08, 0.3).unsqueeze(0)
    opa = torch.tensor([0.7], dtype=torch.float64)
    ws, wm, npix = SO.weights(*_one_tile_per_instance(pos, opa, cov, Hp, Wp), 1, Hp, Wp, FX, FY)
    a = _alpha(pos[0], 0.7, cov[0], Hp, Wp)
    assert math.isclose(float(ws[0]), float(a.sum()), rel_tol=1e-8)
    assert math.isclose(float(wm[0]), float(a.max()), rel_tol=1e-8)
    assert float(npix[0]) == Hp * Wp


def test_rear_gaussian_sees_the_front_transmittance():
    Hp = Wp = 32
    pos = torch.tensor([[0.0, 0.0, 1.0], [0.04, 0.02, 2.0]], dtype=torch.float64)
    cov = torch.stack([_cov(0.1, 0.1), _cov(0.15, 0.1, -0.2)])
    opa = torch.tensor([0.6, 0.8], dtype=torch.float64)
    ws, wm, _ = SO.weights(*_one_tile_per_instance(pos, opa, cov, Hp, Wp), 2, Hp, Wp, FX, FY)
    a0 = _alpha(pos[0], 0.6, cov[0], Hp, Wp)
    a1 = _alpha(pos[1], 0.8, cov[1], Hp, Wp)
    rear = a1 * (1 - a0)
    assert math.isclose(float(ws[0]), float(a0.sum()), rel_tol=1e-8)
    assert math.isclose(float(ws[1]), float(rear.sum()), rel_tol=1e-8)
    assert math.isclose(float(wm[1]), float(rear.max()), rel_tol=1e-8)


def test_saturated_tile_stops_weighting():
    """Ten broad Gaussians of alpha ~0.92 over one tile: T drops below 1e-4 after the fourth; later ones weigh 0."""
    Hp = Wp = 16
    k = 10
    pos = torch.zeros(k, 3, dtype=torch.float64)
    pos[:, 2] = torch.arange(k) + 1.0
    cov = _cov(100.0, 100.0).expand(k, 2, 2).clone()                 # alpha ~ opa over the whole tile
    opa = torch.full((k,), 0.92, dtype=torch.float64)
    ws, wm, _ = SO.weights(*_one_tile_per_instance(pos, opa, cov, Hp, Wp), k, Hp, Wp, FX, FY)
    T = 1.0
    for i in range(k):
        expect = 0.92 * T * 256 if T >= 1e-4 else 0.0
        assert math.isclose(float(ws[i]), expect, rel_tol=1e-4, abs_tol=1e-12), i
        if T >= 1e-4:
            T *= 0.08
    assert float(ws[4:].abs().sum()) == 0.0 and float(wm[4:].abs().sum()) == 0.0
    assert float(ws.sum()) <= 256.0


def test_padding_pixels_are_excluded():
    """A 40 x 24 image in a 48 x 32 padded frame: a Gaussian in the padding weighs 0, one across the border only by
    its pixels inside the image."""
    Hp, Wp, width, height = 32, 48, 40, 24
    crop = ((Wp - width) // 2, (Hp - height) // 2, width, height)
    x_pad = (0.5 - Wp // 2) / FX                                       # the centre of padded column 0
    pos = torch.tensor([[x_pad, 0.0, 1.0], [(4 - Wp // 2) / FX, 0.0, 2.0]], dtype=torch.float64)
    cov = torch.stack([_cov(0.004, 0.004), _cov(0.1, 0.1)])
    opa = torch.tensor([0.9, 0.5], dtype=torch.float64)
    ws, wm, npix = SO.weights(*_one_tile_per_instance(pos, opa, cov, Hp, Wp), 2, Hp, Wp, FX, FY, crop)
    assert float(ws[0]) < 1e-30 and float(wm[0]) < 1e-30
    a0 = _alpha(pos[0], 0.9, cov[0], Hp, Wp)
    a1 = _alpha(pos[1], 0.5, cov[1], Hp, Wp) * (1 - a0)
    inside = torch.zeros(Hp, Wp, dtype=torch.bool)
    inside[crop[1]:crop[1] + height, crop[0]:crop[0] + width] = True
    assert math.isclose(float(ws[1]), float(a1[inside].sum()), rel_tol=1e-8)
    assert float(ws[1]) < float(a1.sum())
    assert float(npix[1]) == width * height


def test_weight_sums_equal_the_alpha_map():
    """sum_i weight_sum = sum_p alpha over the cropped image (alpha = sum_i w = 1 - T_f), on a random scene."""
    g, v, cam = scene(1500, 88, 72, k=1)
    p = {q: t.double() for q, t in g.items()}
    ws, wm, _ = SO.scores(g, cam)
    pos, rgb, opa, cov, accum, rays, _, _ = F._front(p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], cam, "none",
                                                      0.3, 0.05, "abs", False, None)
    _, _, alp = A.draw_maps(pos, rgb, opa, cov, accum, cam.Hp, cam.Wp, cam.fx, cam.fy)
    alpha = cam.crop(alp.unsqueeze(-1)).squeeze(-1)
    assert math.isclose(float(ws.sum()), float(alpha.sum()), rel_tol=1e-10)
    assert float(wm.max()) <= 1.0 and float(ws.min()) >= 0.0
