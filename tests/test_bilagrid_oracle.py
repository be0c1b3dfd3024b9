"""The bilateral-grid oracle (tests/bilagrid_oracle.py) against its definition, torch's grid_sample (border,
align_corners) followed by the affine, in value and autograd gradient; its analytic backward; gradcheck; the TV term;
and bilagrid.color_correct.  CPU only."""
import numpy as np
import pytest
import torch

import bilagrid_oracle as BO


def _image(b, h, w, seed, lo=0.0, hi=1.0):
    g = torch.Generator().manual_seed(seed)
    return (lo + (hi - lo) * torch.rand(b, h, w, 3, generator=g, dtype=torch.float64)).float().double()


def _check(image, grids, ids, tol=1e-10):
    """oracle forward / analytic backward == grid_sample forward / autograd backward"""
    go = torch.randn(image.shape, generator=torch.Generator().manual_seed(7), dtype=torch.float64)
    outs, grads = [], []
    for fn in (BO.slice_forward, BO.slice_grid_sample):
        im = image.clone().requires_grad_(True)
        gr = grids.clone().requires_grad_(True)
        out = fn(im, gr, ids)
        out.backward(go)
        outs.append(out.detach())
        grads.append((im.grad, gr.grad))
    assert float((outs[0] - outs[1]).abs().max()) < tol
    gi, gg = BO.slice_backward(image, grids, ids, go)
    for (a_i, a_g) in [grads[1], grads[0], (gi, gg)]:
        assert float((a_i - grads[1][0]).abs().max()) <= tol * (1 + float(grads[1][0].abs().max()))
        assert float((a_g - grads[1][1]).abs().max()) <= tol * (1 + float(grads[1][1].abs().max()))


@pytest.mark.parametrize("shape", [(16, 16, 8), (8, 4, 4), (2, 2, 2), (3, 5, 9)])
@pytest.mark.parametrize("hw", [(24, 40), (5, 8)])
def test_random_inputs_match_grid_sample(shape, hw):
    grids = BO.random_grids(3, *shape, seed=1)
    _check(_image(2, *hw, seed=2), grids, [2, 0])


@pytest.mark.parametrize("gl", [2, 3, 5, 9])
def test_pixels_on_luminance_knots(gl):
    px = torch.from_numpy(BO.knot_pixels(gl, 48, seed=gl)).double().reshape(1, 6, 8, 3)
    z = BO.guide_f32(px)
    assert np.all((z * (gl - 1)) == np.round(z * (gl - 1)))             # every guide sits on a knot
    assert len(set(np.round(z * (gl - 1)).ravel().tolist())) > 1
    _check(px, BO.random_grids(2, 4, 5, gl, seed=3), [1])


def test_black_white_and_out_of_range_pixels():
    img = _image(1, 12, 10, seed=4, lo=-0.5, hi=1.5)
    img[0, :3] = 0.0                  # black: z = 0
    img[0, 3:6] = 1.0                 # white: z = 1 exactly in fp32
    z = BO.guide_f32(img)
    assert np.all(z[0, :3] == 0) and np.all(z[0, 3:6] == 1.0)
    assert (0.299 * 1.0 + 0.587 * 1.0 + 0.114 * 1.0) != 1.0              # but not in fp64
    assert (z < 0).any() and (z > 1).any()
    _check(img, BO.random_grids(2, 6, 5, 8, seed=5), [0])
    # no z-gradient where the guide is clamped: only the affine's own term remains
    go = torch.ones_like(img)
    gi, _ = BO.slice_backward(img, BO.random_grids(1, 6, 5, 8, seed=9), [0], go)
    assert torch.isfinite(gi).all()


def test_single_image_shape():
    grids = BO.random_grids(2, 4, 4, 4, seed=6)
    img = _image(1, 7, 9, seed=8)
    a = BO.slice_forward(img[0], grids, [1])
    b = BO.slice_forward(img, grids, [1])[0]
    assert a.shape == (7, 9, 3) and torch.equal(a, b)


def test_repeated_views_add():
    grids = BO.random_grids(3, 4, 4, 4, seed=10)
    img = _image(3, 9, 11, seed=11)
    go = torch.randn(img.shape, generator=torch.Generator().manual_seed(12), dtype=torch.float64)
    _, g_all = BO.slice_backward(img, grids, [1, 2, 1], go)
    parts = [BO.slice_backward(img[i:i + 1], grids, [v], go[i:i + 1])[1] for i, v in enumerate([1, 2, 1])]
    assert torch.allclose(g_all, parts[0] + parts[1] + parts[2], rtol=0, atol=1e-12)
    assert torch.equal(g_all[0], torch.zeros_like(g_all[0]))


def test_gradcheck_away_from_knots():
    grids = BO.random_grids(2, 3, 4, 5, seed=13).requires_grad_(True)
    img = (0.1 + 0.8 * torch.rand(1, 4, 6, 3, generator=torch.Generator().manual_seed(14), dtype=torch.float64))
    z = BO.LUM[0] * img[..., 0] + BO.LUM[1] * img[..., 1] + BO.LUM[2] * img[..., 2]
    frac = (z * 4) - (z * 4).floor()
    assert float(torch.minimum(frac, 1 - frac).min()) > 1e-3                # away from the knots
    img.requires_grad_(True)
    assert torch.autograd.gradcheck(lambda i, g: BO.slice_forward(i, g, [1], z_fp32=False), (img, grids),
                                    eps=1e-6, atol=1e-6)


def test_tv_matches_torch_expression():
    import bilagrid
    grids = BO.random_grids(3, 5, 4, 6, seed=15)
    ref = sum(float(((torch.diff(grids, dim=d)) ** 2).mean()) for d in (1, 2, 3))
    assert abs(BO.tv(grids) - ref) < 1e-12
    assert abs(float(bilagrid.tv_loss(grids)) - ref) < 1e-12
    assert float(bilagrid.tv_loss(BO.identity(2, 4, 4, 4))) == 0.0


def test_color_correct_recovers_known_affine():
    import bilagrid
    img = torch.rand(40, 30, 3, generator=torch.Generator().manual_seed(16), dtype=torch.float64)
    M = torch.tensor([[0.8, 0.1, -0.05, 0.02], [0.05, 1.2, 0.0, -0.03], [-0.1, 0.02, 0.9, 0.1]], dtype=torch.float64)
    target = img @ M[:, :3].T + M[:, 3]
    out = bilagrid.color_correct(img, target)
    assert float((out - target).abs().max()) < 1e-12
    noisy = target + 0.01 * torch.randn(target.shape, generator=torch.Generator().manual_seed(17), dtype=torch.float64)
    assert float(((bilagrid.color_correct(img, noisy) - noisy) ** 2).mean()) <= float(((target - noisy) ** 2).mean())


def test_fmaf32_is_correctly_rounded():
    rng = np.random.default_rng(18)
    a, b, c = (rng.standard_normal(20000).astype(np.float32) for _ in range(3))
    got = BO.fmaf32(a, b, c)
    from fractions import Fraction
    for i in range(0, 20000, 997):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        lo = np.float32(float(exact))
        cands = [np.nextafter(lo, np.float32(-np.inf)), lo, np.nextafter(lo, np.float32(np.inf))]
        best = min(cands, key=lambda v: (abs(Fraction(float(v)) - exact), int(np.float32(v).view(np.int32)) & 1))
        assert got[i] == best
    assert BO.guide_f32(np.ones(3, dtype=np.float32)) == np.float32(1.0)
