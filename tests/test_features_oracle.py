"""The feature-map oracle (tests/feat_oracle.py) against closed forms and finite differences (CPU, fp64)."""
import pytest
import torch

import feat_oracle as FT
from helpers import scene

NAMES = ("pos", "rgb", "opa", "quat", "scale")


def _params(g):
    return {q: t.double().clone().requires_grad_(True) for q, t in g.items()}


@pytest.mark.parametrize("F", [8, 16, 32])
def test_constant_features_are_c_times_alpha(F):
    g, _, cam = scene(300, 64, 48, opa_range=(0.05, 0.9))
    p = _params(g)
    c = torch.linspace(-2.0, 3.0, F, dtype=torch.float64)
    o = FT.render_feat(*(p[q] for q in NAMES), c.expand(300, F).contiguous(), cam, background=(0.2, 0.5, 0.9))
    want = o["padded_alpha"].unsqueeze(-1) * c
    assert torch.allclose(o["padded_features"], want, rtol=0, atol=1e-12)
    assert torch.allclose(o["features"], o["alpha"].unsqueeze(-1) * c, rtol=0, atol=1e-12)


def test_one_hot_features_are_per_gaussian_weights():
    """feat = I: channel k is Gaussian k's weight per pixel; the weights sum to alpha, and weighted by the depth
    |p_c| they give the depth map."""
    F = 16
    g, _, cam = scene(F, 48, 32, opa_range=(0.3, 0.9), sigma_px=(2.0, 8.0))
    p = _params(g)
    o = FT.render_feat(*(p[q] for q in NAMES), torch.eye(F, dtype=torch.float64), cam)
    fm = o["padded_features"]
    assert float(o["padded_alpha"].detach().max()) > 0.1
    assert float(fm.min()) >= 0.0
    assert torch.allclose(fm.sum(-1), o["padded_alpha"], rtol=0, atol=1e-12)
    # |p_c| of each Gaussian, from a depth render of that Gaussian alone (its depth map / its alpha)
    t = torch.zeros(F, dtype=torch.float64)
    for k in range(F):
        sel = {q: p[q].detach()[k:k + 1] for q in NAMES}
        ok = FT.render_feat(*(sel[q] for q in NAMES), torch.ones(1, 1, dtype=torch.float64).expand(1, 8).contiguous(),
                            cam)
        a = ok["padded_alpha"]
        if float(a.max()) > 0:
            i = int(a.argmax())
            t[k] = ok["padded_depth"].flatten()[i] / a.flatten()[i]
    used = fm.sum(dim=(0, 1)) > 0
    assert int(used.sum()) > F // 2
    assert torch.allclose((fm * t).sum(-1), o["padded_depth"], rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("mode", ["none", "antialias"])
def test_finite_differences(mode):
    F = 8
    g, _, cam = scene(60, 48, 32, opa_range=(0.1, 0.8), sigma_px=(1.5, 5.0))
    p = _params(g)
    gen = torch.Generator().manual_seed(1)
    feat = (torch.rand(60, F, generator=gen, dtype=torch.float64) * 2 - 1).requires_grad_(True)
    gF = torch.rand(cam.Hp, cam.Wp, F, generator=gen, dtype=torch.float64) * 2 - 1
    gI = torch.rand(cam.Hp, cam.Wp, 3, generator=gen, dtype=torch.float64) * 2 - 1

    def loss(pp, ff):
        o = FT.render_feat(*(pp[q] for q in NAMES), ff, cam, mode=mode)
        return (o["padded_features"] * gF).sum() + (o["padded_image"] * gI).sum()

    L = loss(p, feat)
    grads = torch.autograd.grad(L, [p[q] for q in NAMES] + [feat])
    h = 1e-6
    # (pos is left out: the projection treats its Jacobian as a constant, see tests/test_render_aux_oracle.py)
    checks = [("feat", feat, grads[5])] + [(q, p[q], grads[i]) for i, q in enumerate(NAMES) if q in ("opa", "scale")]
    for name, t, gr in checks:
        for idx in [(3, 0), (17, 1), (41, 2)] if t.dim() == 2 else [(3,), (17,), (41,)]:
            with torch.no_grad():
                old = float(t[idx])
                t[idx] = old + h
                lp = float(loss(p, feat))
                t[idx] = old - h
                lm = float(loss(p, feat))
                t[idx] = old
            fd = (lp - lm) / (2 * h)
            assert abs(fd - float(gr[idx])) <= 1e-5 * max(1.0, abs(fd)), (name, idx, fd, float(gr[idx]))
