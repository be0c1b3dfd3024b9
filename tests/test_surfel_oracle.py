"""The surfel oracle (tests/surfel_oracle.py) against independent answers: a direct 3-D ray / plane solve, densely
sampled 3-sigma circles, the closed-form Gaussian of a fronto-parallel surfel, the O(n^2) distortion sum, the median
rule on hand-built lists and central finite differences."""
import math

import numpy as np
import torch

import gs_oracle as O
import helpers as H
import surfel_oracle as SO


def _cam(w=64, h=48, f=60.0):
    return O.Camera(w, h, f, f, torch.eye(3, dtype=torch.float64), torch.zeros(3, dtype=torch.float64), near=0.2)


def _surfel(pos, quat, s, opa=2.0, rgb=(0.5, -0.3, 1.0)):
    """one surfel's raw parameters (abs scale activation: raw s - 1e-4 activates to s)"""
    d = torch.float64
    return dict(pos=torch.tensor([pos], dtype=d), quat=torch.tensor([quat], dtype=d),
                scale=torch.tensor([[s[0] - 1e-4, s[1] - 1e-4, 0.0]], dtype=d), opa=torch.tensor([opa], dtype=d),
                rgb=torch.tensor([rgb], dtype=d))


def _stack(*gs):
    return {k: torch.cat([g[k] for g in gs]) for k in gs[0]}


def test_intersection_matches_a_ray_plane_solve():
    g, _, cam = H.scene(40, 64, 48, seed=3)
    p = {k: v.double() for k, v in g.items()}
    M, _, pc = SO.surfel_matrix(p["pos"], p["quat"], p["scale"], cam)
    rng = np.random.default_rng(0)
    for i in range(40):
        qx, qy = rng.uniform(-0.5, 0.5, 2)
        h = SO.ray_hit(M[i], torch.tensor(qx, dtype=torch.float64), torch.tensor(qy, dtype=torch.float64))
        a, b = float(h[0] / h[2]), float(h[1] / h[2])
        z = float(M[i, 2, 0] * a + M[i, 2, 1] * b + M[i, 2, 2])
        # t (qx, qy, 1) = p_c + a u + b v
        A = np.stack([[qx, qy, 1.0], -M[i, :, 0].numpy(), -M[i, :, 1].numpy()], axis=1)
        t, a2, b2 = np.linalg.solve(A, pc[i].numpy())
        assert abs(a - a2) < 1e-9 * max(1, abs(a2)) and abs(b - b2) < 1e-9 * max(1, abs(b2))
        assert abs(z - t) < 1e-9 * max(1, abs(t))


def test_disk_box_contains_the_projected_circle_and_is_tight():
    g, _, cam = H.scene(60, 64, 48, seed=4)
    p = {k: v.double() for k, v in g.items()}
    M, _, _ = SO.surfel_matrix(p["pos"], p["quat"], p["scale"], cam)
    ex, ey, hx, hy, c22 = SO.disk_box(M)
    th = torch.linspace(0, 2 * math.pi, 200001, dtype=torch.float64)
    n_checked = 0
    for i in range(M.shape[0]):
        if not c22[i] < 0:
            continue
        P = M[i, :, 2][None] + 3 * torch.cos(th)[:, None] * M[i, :, 0][None] + 3 * torch.sin(th)[:, None] * M[i, :, 1][None]
        x, y = P[:, 0] / P[:, 2], P[:, 1] / P[:, 2]
        scale = float(max(hx[i], hy[i], 1e-3))
        assert float(x.min()) >= float(ex[i] - hx[i]) - 1e-9 * scale and float(x.max()) <= float(ex[i] + hx[i]) + 1e-9 * scale
        assert float(y.min()) >= float(ey[i] - hy[i]) - 1e-9 * scale and float(y.max()) <= float(ey[i] + hy[i]) + 1e-9 * scale
        assert abs(float(x.min()) - float(ex[i] - hx[i])) < 1e-6 * scale
        assert abs(float(y.max()) - float(ey[i] + hy[i])) < 1e-6 * scale
        n_checked += 1
    assert n_checked > 30


def test_fronto_parallel_surfel_is_the_closed_form_gaussian():
    cam = _cam()
    z, s = 3.0, 0.15                      # std s fx / z = 3 px: the intersection wins past the centre pixel
    g = _surfel((0.0, 0.0, z), (1.0, 0.0, 0.0, 0.0), (s, s))
    img, mp, _ = SO.render(g["pos"], g["rgb"], g["opa"], g["quat"], g["scale"], cam)
    sig = s * cam.fx / z
    ys, xs = torch.meshgrid(torch.arange(cam.Hp, dtype=torch.float64), torch.arange(cam.Wp, dtype=torch.float64),
                            indexing="ij")
    r2 = ((xs + 0.5 - cam.Wp // 2) ** 2 + (ys + 0.5 - cam.Hp // 2) ** 2)
    alpha = torch.sigmoid(torch.tensor(2.0, dtype=torch.float64)) * torch.exp(-r2 / (2 * sig * sig))
    alpha = torch.where(alpha < 1 / 255, torch.zeros_like(alpha), alpha)
    inside = r2 < (2.5 * sig) ** 2
    assert float((mp["alpha"] - alpha)[inside].abs().max()) < 1e-12
    assert float((mp["depth"] - alpha * z)[inside].abs().max()) < 1e-12
    col = torch.sigmoid(g["rgb"][0])
    assert float((img - alpha[..., None] * col)[inside].abs().max()) < 1e-12
    # the normal faces the camera: (0, 0, -1)
    assert float((mp["normal"][..., 2] + alpha)[inside].abs().max()) < 1e-12


def test_distortion_running_sums_equal_the_double_sum():
    rng = np.random.default_rng(1)
    w = torch.tensor(rng.uniform(0, 0.3, 12))
    m = torch.tensor(rng.uniform(0, 1, 12))
    A = torch.cumsum(w, 0) - w
    D = torch.cumsum(w * m, 0) - w * m
    D2 = torch.cumsum(w * m * m, 0) - w * m * m
    run = float((w * (m * m * A - 2 * m * D + D2)).sum())
    dbl = sum(float(w[i] * w[j] * (m[i] - m[j]) ** 2) for i in range(12) for j in range(i))
    assert abs(run - dbl) < 1e-14


def test_median_is_the_last_instance_blended_above_half_transmittance():
    cam = _cam()
    op = math.log(0.3 / 0.7)               # sigmoid = 0.3: T before = 1, 0.7, 0.49
    big = (2.0, 2.0)
    g = _stack(*[_surfel((0.0, 0.0, z), (1.0, 0.0, 0.0, 0.0), big, opa=op) for z in (2.0, 3.0, 4.0)])
    _, mp, _ = SO.render(g["pos"], g["rgb"], g["opa"], g["quat"], g["scale"], cam)
    c = (cam.Hp // 2, cam.Wp // 2)
    assert abs(float(mp["median"][c]) - 3.0) < 1e-6
    g1 = _stack(*[_surfel((0.0, 0.0, z), (1.0, 0.0, 0.0, 0.0), big, opa=math.log(0.6 / 0.4)) for z in (2.0, 3.0)])
    _, mp1, _ = SO.render(g1["pos"], g1["rgb"], g1["opa"], g1["quat"], g1["scale"], cam)
    assert abs(float(mp1["median"][c]) - 2.0) < 1e-6          # T = 1, then 0.4
    g0 = _surfel((5.0, 0.0, 2.0), (1.0, 0.0, 0.0, 0.0), (0.01, 0.01))
    _, mp0, _ = SO.render(g0["pos"], g0["rgb"], g0["opa"], g0["quat"], g0["scale"], cam)
    assert float(mp0["median"][c]) == 0.0                     # nothing blended: 0


def test_gradients_match_central_differences():
    g, _, cam = H.scene(6, 32, 32, seed=7)
    base = {k: v.double() for k, v in g.items()}
    rng = np.random.default_rng(2)
    W = {k: torch.tensor(rng.normal(size=s)) for k, s in
         (("img", (cam.Hp, cam.Wp, 3)), ("alpha", (cam.Hp, cam.Wp)), ("depth", (cam.Hp, cam.Wp)),
          ("median", (cam.Hp, cam.Wp)), ("distortion", (cam.Hp, cam.Wp)), ("normal", (cam.Hp, cam.Wp, 3)))}

    def loss(p):
        img, mp, _ = SO.render(p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], cam, background=[0.2, 0.1, 0.4])
        return (img * W["img"]).sum() + sum((mp[k] * W[k]).sum() for k in mp) * 0.3

    p = {k: v.clone().requires_grad_(True) for k, v in base.items()}
    loss(p).backward()
    eps = 1e-6
    for k in ("pos", "rgb", "opa", "quat", "scale"):
        flat = base[k].reshape(-1)
        for j in range(0, flat.numel(), max(1, flat.numel() // 7)):
            qp = {kk: v.clone() for kk, v in base.items()}
            qm = {kk: v.clone() for kk, v in base.items()}
            qp[k].view(-1)[j] += eps
            qm[k].view(-1)[j] -= eps
            fd = float(loss(qp) - loss(qm)) / (2 * eps)
            an = float(p[k].grad.reshape(-1)[j])
            assert abs(fd - an) <= 1e-4 * max(1.0, abs(fd)), (k, j, fd, an)
    assert float(p["scale"].grad[:, 2].abs().max()) == 0.0
