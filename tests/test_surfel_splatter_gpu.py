"""Splatter(primitive="surfel") end to end on the GPU: a synthetic scene of surfels trained from a perturbed start with
the fused flat Adam (loss falls, grad_scale[:, 2] stays exactly 0, scale[:, 2] stays at the activation's floor), the
maps of render_surfel_maps, and a checkpoint that round-trips with the reference's five keys."""
import math
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "examples"))

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("act", ["abs", "exp"])
def test_surfel_splatter_trains_and_round_trips_a_checkpoint(tmp_path, act):
    import loss as L
    import optim
    import splatter
    import synthetic as S
    dev = torch.device("cuda", 0)
    n, w, h = 3000, 96, 64
    teacher = S.make_gaussians(n, w, h, 0)
    if act == "exp":
        teacher["scale"] = torch.log(teacher["scale"].abs() + 1e-4)
    views = [S.make_view(w, h, k) for k in range(4)]
    vd = [dict(width=v.width, height=v.height, focal_x=v.fx, focal_y=v.fy, rot=v.rot, tran=v.tran) for v in views]
    sp_t = splatter.Splatter.from_tensors(teacher, vd, device=dev, primitive="surfel", scale_activation=act)
    floor = 0.0 if act == "abs" else math.log(1e-4)
    assert torch.all(sp_t.gaussian_3ds.scale[:, 2] == floor)
    with torch.no_grad():
        gts = [sp_t(k).clone() for k in range(len(vd))]
    g = torch.Generator().manual_seed(1)
    student = {k: v.clone() for k, v in teacher.items()}
    student["pos"] += torch.randn(n, 3, generator=g) * 0.01
    student["rgb"] = torch.zeros_like(teacher["rgb"])
    student["opa"] = torch.full_like(teacher["opa"], -2.0)
    sp = splatter.Splatter.from_tensors(student, vd, device=dev, primitive="surfel", scale_activation=act)
    gs = sp.gaussian_3ds
    opt = optim.FlatAdam([{"params": gs.opa, "lr": 0.03}, {"params": gs.rgb, "lr": 0.03}, {"params": gs.pos, "lr": 0.003},
                          {"params": gs.scale, "lr": 0.003}, {"params": gs.quat, "lr": 0.003}], betas=(0.9, 0.99))
    losses = []
    for it in range(300):
        opt.zero_grad(set_to_none=True)
        v = it % len(vd)
        out = sp.render_surfel_maps(v)
        loss = ((out["image"] - gts[v]).abs().mean()
                + 0.01 * L.surfel_normal_consistency(out["normal"], out["depth"], out["alpha"], vd[v]["focal_x"],
                                                     vd[v]["focal_y"])
                + 10.0 * out["distortion"].mean())
        loss.backward()
        assert torch.all(gs.scale.grad[:, 2] == 0)
        opt.step()
        losses.append(float(loss.detach()))
    first, last = sum(losses[:20]) / 20, sum(losses[-20:]) / 20
    assert math.isfinite(last) and last < 0.6 * first, (first, last)
    assert torch.all(gs.scale[:, 2] == floor)                  # Adam never moved the flat axis
    assert sp.n_tile_gaussians > 0

    path = str(tmp_path / "surfel.pt")
    sp.save_checkpoint(path)
    ck = torch.load(path, map_location="cpu", weights_only=False)
    assert {"pos", "rgb", "opa", "quat", "scale"} <= set(ck)
    sp2 = splatter.Splatter.from_tensors(student, vd, device=dev, primitive="surfel", scale_activation=act,
                                         load_ckpt=path)
    for k in ("pos", "rgb", "opa", "quat", "scale"):
        assert torch.equal(getattr(sp2.gaussian_3ds, k).detach(), getattr(gs, k).detach()), k
    with torch.no_grad():
        assert torch.equal(sp2(1), sp(1))


def test_surfel_splatter_refuses_3dgs_only_renders():
    import splatter
    import synthetic as S
    dev = torch.device("cuda", 0)
    v = S.make_view(64, 48, 0)
    sp = splatter.Splatter.from_tensors(S.make_gaussians(100, 64, 48, 0),
                                        [dict(width=64, height=48, focal_x=v.fx, focal_y=v.fy, rot=v.rot, tran=v.tran)],
                                        device=dev, primitive="surfel")
    for call in (lambda: sp.render_maps(0), lambda: sp.render_batch([0]), lambda: sp.render_features(0)):
        with pytest.raises(ValueError, match="primitive='surfel'"):
            call()
    assert sp.render_padded().shape == (48, 64, 3)
