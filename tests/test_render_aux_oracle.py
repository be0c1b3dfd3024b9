"""CPU checks of the depth / alpha / background oracle (tests/aux_oracle.py) and of the argument validation of
gs_render_forward_aux / gs_render_backward_aux.  The reference renders none of these outputs, so this parity is
unpinned externally: the oracle is checked against closed-form identities and central finite differences."""
import ctypes
import os

import torch

import aux_oracle as A
import gs_oracle as O
from helpers import scene

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "3d-gaussian-splatting_b200")


def _sorted(g, cam, dtype=torch.float64):
    p = {k: v.to(dtype) for k, v in g.items()}
    nq, ns, opa_a, rgb_a = O.preactivate(p["quat"], p["scale"], p["opa"], p["rgb"])
    rp, rc, mask = O.global_culling(p["pos"], nq, ns, cam.rot.to(dtype), cam.tran.to(dtype), cam.near,
                                    cam.half_w, cam.half_h)
    idx = torch.nonzero(mask.bool()).squeeze(-1)
    p_c, c_c = rp[idx], rc[idx]
    rects = O.tile_rects(p_c[:, :2], c_c, 0.05, cam.tile_lx, cam.tile_ly, cam.ntx, cam.nty, cam.leftmost, cam.topmost)
    gi, accum = O.bin_and_sort(p_c, c_c, rects, cam.ntx, cam.nty)
    return p_c[gi], rgb_a[idx][gi], opa_a[idx][gi], c_c[gi], accum


def _sequential_alpha(pos, opa, cov, accum, Hp, Wp, fx, fy):
    """1 - T_f by the blend loop itself: one pixel at a time, stop before an instance once T < 1e-4."""
    out = torch.zeros(Hp, Wp, dtype=torch.float64)
    ntx = Wp // 16
    cov4 = cov.reshape(-1, 4)
    for t in range(len(accum) - 1):
        s, e = int(accum[t]), int(accum[t + 1])
        ty, tx = divmod(t, ntx)
        for yy in range(16):
            for xx in range(16):
                X = (tx * 16 + xx + 0.5 - Wp // 2) / fx
                Y = (ty * 16 + yy + 0.5 - Hp // 2) / fy
                T = 1.0
                for i in range(s, e):
                    if T < 1e-4:
                        break
                    a, b, c, d = (float(v) for v in cov4[i])
                    dx, dy = X - float(pos[i, 0]), Y - float(pos[i, 1])
                    power = -(d * dx * dx - (b + c) * dx * dy + a * dy * dy) / (2 * (a * d - b * c) + 1e-14)
                    T *= 1 - float(opa[i]) * torch.exp(torch.tensor(power, dtype=torch.float64)).item()
                out[ty * 16 + yy, tx * 16 + xx] = 1 - T
    return out


def test_alpha_is_one_minus_transmittance_with_early_stop():
    g, v, cam = scene(400, 48, 32, opa_range=(0.6, 0.98))         # opaque: the early stop is reached
    pos, rgb, opa, cov, accum = _sorted(g, cam)
    _, _, alpha = A.draw_maps(pos, rgb, opa, cov, accum, cam.Hp, cam.Wp, cam.fx, cam.fy)
    ref = _sequential_alpha(pos, opa, cov, accum, cam.Hp, cam.Wp, cam.fx, cam.fy)
    assert float(ref.max()) > 1 - 1e-4                               # some pixels saturate
    assert torch.allclose(alpha, ref, atol=1e-12, rtol=0)


def test_background_adds_bg_times_transmittance():
    g, v, cam = scene(300, 64, 48)
    pos, rgb, opa, cov, accum = _sorted(g, cam)
    bg = torch.tensor([0.25, 1.0, -0.5], dtype=torch.float64)
    black, _, alpha = A.draw_maps(pos, rgb, opa, cov, accum, cam.Hp, cam.Wp, cam.fx, cam.fy)
    img, _, _ = A.draw_maps(pos, rgb, opa, cov, accum, cam.Hp, cam.Wp, cam.fx, cam.fy, background=bg)
    assert torch.allclose(img - black, bg * (1 - alpha).unsqueeze(-1), atol=1e-12, rtol=0)
    # without a background the image is gs_oracle.draw's
    assert torch.allclose(black, O.draw(pos, rgb, opa, cov, accum, cam.Hp, cam.Wp, cam.fx, cam.fy), atol=1e-12, rtol=0)


def test_isolated_gaussian_depth_is_distance_times_alpha():
    g, v, cam = scene(1, 48, 48, seed=3)
    g["pos"] = torch.tensor([[0.1, -0.05, 0.3]])
    p = {k: t.double() for k, t in g.items()}
    out = A.render_maps(p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], cam)
    pc = p["pos"][0] @ cam.rot.double().T + cam.tran.double()
    assert float(out["padded_alpha"].max()) > 0.01
    assert torch.allclose(out["padded_depth"], pc.norm() * out["padded_alpha"], atol=1e-12, rtol=0)


def _fd_check(which, monkeypatch):
    g, v, cam = scene(5, 32, 32, seed=7, opa_range=(0.2, 0.6), sigma_px=(2.0, 6.0))
    p = {k: t.double().clone().requires_grad_(True) for k, t in g.items()}
    gen = torch.Generator().manual_seed(11)
    w = torch.rand(cam.height, cam.width, generator=gen, dtype=torch.float64)
    # The projection treats its Jacobian as a constant (the reference's semantics: no d cov2d / d pos), so the
    # function whose differences match the autograd gradient evaluates that Jacobian at the unperturbed positions.
    base_pos = p["pos"].detach().clone()
    culling = O.global_culling

    def _shifted(pos, quat_n, scale_a, rot, tran, near, hw, hh):
        # value at pos, Jacobian at base_pos: res_cov from base_pos, res_pos / mask from pos
        rp, _, mask = culling(pos, quat_n, scale_a, rot, tran, near, hw, hh)
        _, rc, _ = culling(base_pos, quat_n, scale_a, rot, tran, near, hw, hh)
        return rp, rc, mask

    def loss(q):
        return (A.render_maps(q["pos"], q["rgb"], q["opa"], q["quat"], q["scale"], cam)[which] * w).sum()

    loss(p).backward()
    monkeypatch.setattr(O, "global_culling", _shifted)
    eps = 1e-6
    for name in p:
        ana = p[name].grad if p[name].grad is not None else torch.zeros_like(p[name])   # depth / alpha: no rgb
        num = torch.zeros_like(ana)
        flat = p[name].detach().view(-1)
        for i in range(flat.numel()):
            q = {k: t.detach().clone() for k, t in p.items()}
            q[name].view(-1)[i] += eps
            lp = float(loss(q))
            q[name].view(-1)[i] -= 2 * eps
            lm = float(loss(q))
            num.view(-1)[i] = (lp - lm) / (2 * eps)
        assert (float(ana.abs().max()) > 0) == (name != "rgb"), name
        err = float((ana - num).abs().max() / (num.abs().max() + 1e-12))
        assert err < 1e-5, (which, name, err)


def test_depth_gradient_matches_finite_differences(monkeypatch):
    _fd_check("depth", monkeypatch)


def test_alpha_gradient_matches_finite_differences(monkeypatch):
    _fd_check("alpha", monkeypatch)


def test_aux_entry_points_reject_bad_arguments_without_gpu():
    lib = ctypes.CDLL(os.path.join(PKG, "libgs_b200.so"))
    lib.gs_last_error.restype = ctypes.c_char_p
    P, I = ctypes.c_void_p, ctypes.c_int
    lib.gs_render_forward_aux.argtypes = [P, P, P, P, P, P, I, I, I, P, P, P, P, P, P]
    assert lib.gs_render_forward_aux(None, None, None, None, None, None, 0, 3, 0, None, 0x1000, None, None, None,
                                     None) == -1
    assert "bad arguments" in lib.gs_last_error().decode()
    lib.gs_render_backward_aux.argtypes = [P, P, P, P, P, P, P, P, I, P, P, P, P, P, P, P, P]
    assert lib.gs_render_backward_aux(None, None, None, None, None, None, None, None, 0, None, 0x1000, None, None,
                                      None, None, None, None) == -1
    assert "null ctx" in lib.gs_last_error().decode()
