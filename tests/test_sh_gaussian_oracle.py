"""CPU checks of the per-Gaussian SH oracle (tests/sh_gaussian_oracle.py) and of the argument validation of
gs_ctx_set_sh_eval.  No other renderer evaluates SH this way here, so the oracle is checked against the per-pixel
oracle where the two models must agree (DC-only colour) and against central finite differences."""
import ctypes
import os

import pytest
import torch

import gs_oracle as O
import sh_gaussian_oracle as G
from helpers import scene

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "3d-gaussian-splatting_b200")
NAMES = ("pos", "rgb", "opa", "quat", "scale")


def _grads(fn, g, go):
    p = {k: t.double().clone().requires_grad_(True) for k, t in g.items()}
    img = fn(p)
    img.backward(go)
    return img.detach(), {k: p[k].grad for k in NAMES}


@pytest.mark.parametrize("sh_dim", [27, 48])
def test_dc_only_matches_per_pixel_oracle(sh_dim):
    """With only the DC coefficients non-zero the basis is constant: both colour models give the same image and the
    same gradients (pos: the direction term vanishes), except for the higher-order coefficients, whose gradients are
    the basis at different directions."""
    g, v, cam = scene(300, 64, 48, k=1, sh_dim=sh_dim, opa_range=(0.05, 0.9))
    K = sh_dim // 3
    rgb = g["rgb"].reshape(-1, 3, K).clone()
    rgb[:, :, 1:] = 0
    g["rgb"] = rgb.reshape(-1, sh_dim)
    go = torch.rand(cam.height, cam.width, 3, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    gi, gg = _grads(lambda p: G.render(p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], cam), g, go)
    pi, pg = _grads(lambda p: O.render(p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], cam, use_sh_coeff=True),
                    g, go)
    assert float(gi.max()) > 0.1
    assert torch.allclose(gi, pi, atol=1e-12, rtol=0)
    for k in ("pos", "opa", "quat", "scale"):
        assert float(pg[k].abs().max()) > 0, k
        assert torch.allclose(gg[k], pg[k], atol=1e-10 * float(pg[k].abs().max()), rtol=0), k
    dc_g = gg["rgb"].reshape(-1, 3, K)[:, :, 0]
    dc_p = pg["rgb"].reshape(-1, 3, K)[:, :, 0]
    assert torch.allclose(dc_g, dc_p, atol=1e-10 * float(dc_p.abs().max()), rtol=0)
    hi_g = gg["rgb"].reshape(-1, 3, K)[:, :, 1:]
    hi_p = pg["rgb"].reshape(-1, 3, K)[:, :, 1:]
    assert float(hi_g.abs().max()) > 0 and not torch.allclose(hi_g, hi_p)


@pytest.mark.parametrize("sh_dim", [27, 48])
def test_gradients_match_finite_differences(sh_dim, monkeypatch):
    """pos (with the direction term) and coefficient gradients of the oracle against central differences in fp64."""
    g, v, cam = scene(5, 32, 32, seed=7, sh_dim=sh_dim, opa_range=(0.2, 0.6), sigma_px=(2.0, 6.0))
    K = sh_dim // 3
    rgb = g["rgb"].reshape(-1, 3, K).clone()
    rgb[:, :, 1:] *= 5                                   # a direction term well above the difference noise
    g["rgb"] = rgb.reshape(-1, sh_dim)
    p = {k: t.double().clone().requires_grad_(True) for k, t in g.items()}
    w = torch.rand(cam.Hp, cam.Wp, 3, generator=torch.Generator().manual_seed(11), dtype=torch.float64)
    # The projection treats its Jacobian as a constant (the reference's semantics: no d cov2d / d pos), so the function
    # whose differences match the autograd gradient evaluates that Jacobian at the unperturbed positions.  The view
    # direction is NOT frozen: its dependence on pos is part of the model.
    base_pos = p["pos"].detach().clone()
    culling = O.global_culling

    def _shifted(pos, quat_n, scale_a, rot, tran, near, hw, hh):
        rp, _, mask = culling(pos, quat_n, scale_a, rot, tran, near, hw, hh)
        _, rc, _ = culling(base_pos, quat_n, scale_a, rot, tran, near, hw, hh)
        return rp, rc, mask

    def loss(q, detach_dir=False):
        logits = G.gaussian_logits(q["pos"], q["rgb"], cam, detach_dir)
        _, aux = O.render(q["pos"], logits, q["opa"], q["quat"], q["scale"], cam, return_aux=True)
        return (aux["padded"] * w).sum()                 # un-clamped: no kinks

    loss(p).backward()
    ana = {k: p[k].grad.clone() for k in ("pos", "rgb")}
    q = {k: t.detach().clone().requires_grad_(True) for k, t in p.items()}
    loss(q, detach_dir=True).backward()
    dir_term = ana["pos"] - q["pos"].grad
    assert float(dir_term.abs().max()) > 1e-3 * float(ana["pos"].abs().max())
    monkeypatch.setattr(O, "global_culling", _shifted)
    eps = 1e-6
    for name in ("pos", "rgb"):
        num = torch.zeros_like(ana[name])
        flat = p[name].detach().view(-1)
        for i in range(flat.numel()):
            q = {k: t.detach().clone() for k, t in p.items()}
            q[name].view(-1)[i] += eps
            lp = float(loss(q))
            q[name].view(-1)[i] -= 2 * eps
            lm = float(loss(q))
            num.view(-1)[i] = (lp - lm) / (2 * eps)
        assert float(num.abs().max()) > 0, name
        err = float((ana[name] - num).abs().max() / num.abs().max())
        assert err < 1e-5, (name, err)


def test_set_sh_eval_rejects_bad_arguments_without_gpu():
    lib = ctypes.CDLL(os.path.join(PKG, "libgs_b200.so"))
    lib.gs_last_error.restype = ctypes.c_char_p
    lib.gs_ctx_set_sh_eval.argtypes = [ctypes.c_void_p, ctypes.c_int]
    for mode in (0, 1):
        assert lib.gs_ctx_set_sh_eval(None, mode) == -1
        assert "null ctx" in lib.gs_last_error().decode()
    for mode in (-1, 2, 27):
        assert lib.gs_ctx_set_sh_eval(None, mode) == -1
        assert "mode must be" in lib.gs_last_error().decode()
