"""CPU tests of the oracle itself: internal consistency (analytic properties of the
reference's algorithm) and agreement with the golden fixtures produced by the reference's
own CUDA build on a GPU (tests/golden/make_golden.py)."""
import math

import pytest
import torch

import gs_oracle as O
import synthetic as S
from helpers import abs_err, load_golden, rel_err, scene, sorted_instances_cpu


def test_generator_is_deterministic_and_matches_survey_workload():
    g1 = S.make_gaussians(10000, 256, 256, 0)
    g2 = S.make_gaussians(10000, 256, 256, 0)
    for k in g1:
        assert torch.equal(g1[k], g2[k])
    _, v, cam = scene(10, 256, 256)
    inst = sorted_instances_cpu(g1, cam)
    counts = inst["accum"][1:] - inst["accum"][:-1]
    # SURVEY.md §8d probe of the reference's binning rule: C1 -> M = 29.7k, max 273 / tile
    assert int(inst["accum"][-1]) == 29725 and int(counts.max()) == 273


def test_projection_matches_closed_form_for_axis_aligned_gaussian():
    # identity rotation, isotropic scale s, point on the optical axis at depth z:
    # cov2d = (s/z)^2 * I, pos_i = (0, 0, z)
    cam = O.Camera(64, 64, 50.0, 50.0, torch.eye(3), torch.zeros(3))
    pos = torch.tensor([[0.0, 0.0, 2.0]])
    q = torch.tensor([[1.0, 0, 0, 0]])
    s = torch.tensor([[0.1, 0.1, 0.1]])
    rp, rc, m = O.global_culling(pos, q, s, cam.rot, cam.tran, 0.3, cam.half_w, cam.half_h)
    assert int(m[0]) == 1
    assert torch.allclose(rp[0], torch.tensor([0.0, 0.0, 2.0]))
    assert torch.allclose(rc[0], torch.eye(2) * (0.1 / 2.0) ** 2, atol=1e-9)


def test_projection_jacobian_is_detached():
    # reference gaussian.cu:1397-1421: d cov2d / d pos is NOT propagated
    g, v, cam = scene(50, 64, 64)
    nq, ns, _, _ = O.preactivate(g["quat"], g["scale"], g["opa"], g["rgb"])
    pos = g["pos"].double().requires_grad_(True)
    rp, rc, m = O.global_culling(pos, nq.double(), ns.double(), cam.rot.double(), cam.tran.double(), 0.3,
                                 cam.half_w, cam.half_h)
    assert not rc.requires_grad          # cov2d carries no graph back to pos at all
    (rp.sum() * 0 + rc.sum()).backward()
    assert float(pos.grad.abs().max()) == 0.0


def test_culling_rules():
    cam = O.Camera(64, 64, 50.0, 50.0, torch.eye(3), torch.zeros(3), near=0.3)
    pos = torch.tensor([[0, 0, 0.3], [0, 0, 0.31], [10.0, 0, 1.0], [0, 0, -1.0]])
    q = torch.tensor([[1.0, 0, 0, 0]]).repeat(4, 1)
    s = torch.full((4, 3), 0.01)
    _, _, m = O.global_culling(pos, q, s, cam.rot, cam.tran, cam.near, cam.half_w, cam.half_h)
    assert m.tolist() == [0, 1, 0, 0]       # z <= near culled; outside 1.2x frustum culled


def test_tile_rect_rule():
    cam = O.Camera(64, 64, 64.0, 64.0, torch.eye(3), torch.zeros(3))
    # sigma = 1 px in normalised units, centred on the image centre -> bbox +-2.45 px -> 2x2 tiles
    sig = 1.0 / 64.0
    cov = torch.tensor([[sig ** 2, 0, 0, sig ** 2]])
    r = O.tile_rects(torch.tensor([[0.0, 0.0]]), cov, 0.05, cam.tile_lx, cam.tile_ly, cam.ntx, cam.nty, cam.leftmost,
                     cam.topmost)
    assert [int(x) for x in r] == [1, 3, 1, 3]
    # centre of a tile, same sigma -> stays inside one tile
    c = (8.0 - 32.0) / 64.0
    r = O.tile_rects(torch.tensor([[c, c]]), cov, 0.05, cam.tile_lx, cam.tile_ly, cam.ntx, cam.nty, cam.leftmost,
                     cam.topmost)
    assert [int(x) for x in r] == [0, 1, 0, 1]
    # det <= 0 -> never binned (gaussian.cu:227)
    r = O.tile_rects(torch.tensor([[0.0, 0.0]]), torch.tensor([[1.0, 1.0, 1.0, 1.0]]), 0.05, cam.tile_lx, cam.tile_ly,
                     cam.ntx, cam.nty, cam.leftmost, cam.topmost)
    assert int(r[1] - r[0]) * int(r[3] - r[2]) == 0


def test_blend_matches_sequential_loop():
    """The vectorised blend equals a literal per-pixel loop with the reference's early stop."""
    g, v, cam = scene(300, 32, 32, opa_range=(0.3, 0.95))
    inst = sorted_instances_cpu(g, cam, dtype=torch.float64)
    img = O.draw(inst["pos"], inst["rgb"], inst["opa"], inst["cov"], inst["accum"], cam.Hp, cam.Wp, cam.fx, cam.fy)
    acc = inst["accum"]
    for (iy, ix) in [(0, 0), (5, 17), (16, 16), (31, 31), (20, 3)]:
        t = (iy // 16) * cam.ntx + ix // 16
        px = (ix + 0.5 - cam.Wp // 2) / cam.fx
        py = (iy + 0.5 - cam.Hp // 2) / cam.fy
        T, col = 1.0, torch.zeros(3, dtype=torch.float64)
        for i in range(int(acc[t]), int(acc[t + 1])):
            if T < 0.0001:
                break
            a, b, c, d = inst["cov"][i].reshape(-1).tolist()
            x, y = px - float(inst["pos"][i, 0]), py - float(inst["pos"][i, 1])
            det = a * d - b * c
            alpha = math.exp(-(d * x * x - (b + c) * x * y + a * y * y) / (2 * det + 1e-14)) * float(inst["opa"][i])
            col += inst["rgb"][i] * alpha * T
            T *= 1 - alpha
        assert torch.allclose(img[iy, ix], col, atol=1e-12)


def test_render_gradients_finite_difference():
    g, v, cam = scene(60, 32, 32, opa_range=(0.2, 0.6), sigma_px=(1.5, 4.0))
    p = {k: t.double().clone().requires_grad_(True) for k, t in g.items()}
    go = S.make_grad_output(32, 32, 0).double()

    def loss(pp):
        return (O.render(pp["pos"], pp["rgb"], pp["opa"], pp["quat"], pp["scale"], cam) * go).sum()

    loss(p).backward()
    eps = 1e-6
    # opa / rgb / quat / scale are fully differentiated; pos only through the 2-D mean (J detached)
    for name, idx in (("opa", (7,)), ("rgb", (3, 1)), ("scale", (11, 2)), ("quat", (5, 3))):
        q = {k: t.detach().clone() for k, t in p.items()}
        q[name][idx] += eps
        up = loss(q)
        q[name][idx] -= 2 * eps
        dn = loss(q)
        fd = float((up - dn) / (2 * eps))
        an = float(p[name].grad[idx])
        assert abs(fd - an) <= 1e-4 * max(abs(fd), abs(an)) + 1e-12, (name, fd, an)


@pytest.mark.parametrize("name", ["project.npz", "tiles.npz", "draw_rgb.npz", "draw_sh.npz", "frame_c1.npz"])
def test_oracle_matches_reference_golden(name):
    gold = load_golden(name)
    if gold is None:
        pytest.skip(f"tests/golden/{name} not generated yet (needs the reference build on a GPU)")
    import golden_cases as GC
    GC.check_oracle_against(name, gold)
