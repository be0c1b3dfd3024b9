"""Mip-Splatting's 3-D smoothing filter on the fused frame path (gs_filter3d_compute, gs_ctx_set_filter3d,
`Splatter(..., filter3d=True)`) against the fp64 oracle of tests/filter3d_oracle.py: the sampling-rate kernel up to
2.4 M Gaussians x 300 views, frames of every colour model with every 2-D filter mode, aux maps, a batch with camera
gradients, feature maps, the zero filter's bit identity, extreme scales, the densification statistics, the
data-parallel push, the refusals and a Mip-Splatting-configured training run through Splatter."""
import math

import numpy as np
import pytest
import torch

import filter3d_oracle as F3
import filter_oracle as F
import gs_oracle as O
import sh_gaussian_oracle as G
import synthetic as S
from helpers import abs_err, device_depth_keys, rel_err, scene

pytestmark = pytest.mark.gpu

IMG_ATOL = 1e-4
GRAD_RTOL = 1e-3
BG = (0.2, 0.5, 0.9)
NAMES = ("pos", "rgb", "opa", "quat", "scale")
VAR = 2.0   # a filter of ~1.4 px in the scene's views: large enough that every frame below differs from the unfiltered


def _cams_of(views, near=0.3):
    return dict(size=torch.tensor([[v.width, v.height] for v in views], dtype=torch.int64),
                focal=torch.tensor([[v.fx, v.fy] for v in views], dtype=torch.float32),
                rot=torch.stack([torch.as_tensor(v.rot, dtype=torch.float32) for v in views]),
                tran=torch.stack([torch.as_tensor(v.tran, dtype=torch.float32) for v in views]), near=near)


def _oracle_cams(views, near=0.3):
    return [dict(width=v.width, height=v.height, focal_x=v.fx, focal_y=v.fy, rot=np.asarray(v.rot),
                 tran=np.asarray(v.tran), near=near) for v in views]


def _compute(gs, rctx, pos, views, margin=0.15, variance=0.2, near=0.3):
    c = _cams_of(views, near)
    return gs[0].filter3d_compute(rctx, pos, c["size"], c["focal"], c["rot"], c["tran"], near, margin, variance)


def _ulp_err(got, ref64):
    ref = torch.from_numpy(ref64).float()
    spacing = torch.from_numpy(np.spacing(np.abs(ref.numpy()))).double()
    d = (got.double() - torch.from_numpy(ref64)).abs()
    return float((d / spacing.clamp_min(1e-45)).max())


def _orbit_views(w, h, k_views, seed=0):
    """k_views views around the synthetic scene at several distances and focal lengths (no two alike)."""
    gen = np.random.default_rng(seed)
    out = []
    for k in range(k_views):
        v = S.make_view(w, h, k % 8)
        scale = 0.6 + 0.8 * gen.random()
        ang = gen.uniform(-0.3, 0.3)
        c, s = math.cos(ang), math.sin(ang)
        rx = np.array([[1, 0, 0], [0, c, -s], [0, s, c]])
        rot = (rx @ np.asarray(v.rot, dtype=np.float64)).astype(np.float32)
        tran = (np.asarray(v.tran, dtype=np.float64) * scale).astype(np.float32)
        out.append(S.View(v.width, v.height, float(np.float32(v.fx * (0.7 + 0.6 * gen.random()))),
                          float(np.float32(v.fy)), torch.from_numpy(rot), torch.from_numpy(tran), v.near))
    return out


@pytest.mark.parametrize("n,k_views", [(20_000, 7), (2_400_000, 50), (2_400_000, 300)])
def test_sampling_rate_kernel_vs_oracle(gs, cuda, n, k_views):
    """f within 2 ulp of the fp64 oracle, the same seen set (the scene drops the Gaussians at a view-boundary tie, where
    the device's float32 margin test and the oracle's fp64 one may disagree), the same bits on a second call and for a
    permutation of the views; the C3 size with 50 and 300 views."""
    g = S.make_gaussians(n, 640, 360, seed=1)
    pos = g["pos"] * 1.3
    pos[: n // 50] += torch.tensor([0.0, 1000.0, 0.0])         # some Gaussians no view sees (far above every view)
    views = _orbit_views(640, 360, k_views)
    tie = F3.boundary_ties(pos.numpy(), _oracle_cams(views))
    assert int(tie.sum()) < n // 200
    pos = pos[torch.from_numpy(~tie)].contiguous()             # a scene away from view-boundary ties
    rctx = gs[0].RenderContext()
    pd = pos.to(cuda)
    before = gs[0].kernel_launches()
    f = _compute(gs, rctx, pd, views)
    assert gs[0].kernel_launches() - before == 2
    ref, seen = F3.sampling_filter(pos.numpy(), _oracle_cams(views))
    assert seen.any() and not seen.all()
    got = f.cpu()
    assert bool(torch.isfinite(got).all()) and bool((got > 0).all())
    assert _ulp_err(got, ref) <= 2.0
    # an unseen row carries the largest filter (a seen row the device took for unseen would fail the ulp check)
    assert bool((got[torch.from_numpy(~seen)] == got.max()).all())
    assert torch.equal(_compute(gs, rctx, pd, views), f)
    perm = np.random.default_rng(3).permutation(k_views)
    assert torch.equal(_compute(gs, rctx, pd, [views[i] for i in perm]), f)


def test_sampling_rate_kernel_edge_cases(gs, cuda):
    rctx = gs[0].RenderContext()
    v = S.View(64, 48, 50.0, 50.0, torch.eye(3), torch.zeros(3), 0.3)
    none_seen = torch.tensor([[0.0, 0.0, -3.0], [0.0, 0.0, 0.1]], device=cuda)
    assert torch.equal(_compute(gs, rctx, none_seen, [v]), torch.zeros(2, device=cuda))
    one = torch.tensor([[0.0, 0.0, 4.0], [0.0, 0.0, 8.0], [900.0, 0.0, 4.0]], device=cuda)
    f = _compute(gs, rctx, one, [v], variance=0.2).cpu()
    assert f[0] == np.float32(math.sqrt(0.2) * 4.0 / 50.0) and f[2] == f[1] == np.float32(math.sqrt(0.2) * 8.0 / 50.0)
    before = gs[0].kernel_launches()
    assert _compute(gs, rctx, torch.zeros(0, 3, device=cuda), [v]).numel() == 0
    assert gs[0].kernel_launches() == before


# ---- frames against the oracle -------------------------------------------------------------------------------------
COLOURS = {"rgb": (3, "pixel"), "sh27-pixel": (27, "pixel"), "sh48-gauss": (48, "gaussian")}


def _splatter(g, v, dev, f3d, **kw):
    import splatter
    vs = [dict(width=v.width, height=v.height, focal_x=v.fx, focal_y=v.fy, rot=v.rot, tran=v.tran)]
    sp = splatter.Splatter.from_tensors(g, vs, device=dev, use_sh_coeff=g["rgb"].shape[1] != 3, filter3d=True,
                                        filter3d_variance=VAR, **kw)
    sp._set_filter3d(f3d.to(dev))
    return sp


def _scene_filter(gs, cuda, g, v):
    return _compute(gs, gs[0].RenderContext(), g["pos"].to(cuda), [v], variance=VAR).cpu()


@pytest.mark.parametrize("mode", F.MODES)
@pytest.mark.parametrize("colour", list(COLOURS))
def test_frame_vs_oracle(gs, cuda, colour, mode):
    """Splatter frames with the 3-D filter (and each 2-D filter mode) against the oracle: image 1e-4 abs, the five
    gradients 1e-3 relative; abs scale for RGB, exp for SH; final and padded images alternate."""
    sh_dim, sh_eval = COLOURS[colour]
    act = "abs" if sh_dim == 3 else "exp"
    final = mode != "dilate"
    n, w, h = (4000, 128, 96) if sh_dim == 3 else (2500, 112, 80)
    g, v, cam = scene(n, w, h, k=1, sh_dim=sh_dim, opa_range=(0.05, 0.9), sigma_px=(0.3, 3.0))
    if act == "exp":
        g["scale"] = g["scale"].abs().log()
    f3 = _scene_filter(gs, cuda, g, v)
    p = {q: t.double().clone().requires_grad_(True) for q, t in g.items()}
    rgb = G.gaussian_logits(p["pos"], p["rgb"], cam) if sh_eval == "gaussian" else p["rgb"]
    use_sh = sh_dim != 3 and sh_eval == "pixel"
    with F3.applied(f3.double()):
        img, aux = F.render(p["pos"], rgb, p["opa"], p["quat"], p["scale"], cam, mode, scale_activation=act,
                            use_sh_coeff=use_sh, return_aux=True, depth_key=device_depth_keys(g, cam, cuda, act))
    unfiltered = F.render(*(t.detach() for t in (p["pos"], rgb, p["opa"], p["quat"], p["scale"])), cam, mode,
                          scale_activation=act, use_sh_coeff=use_sh)
    out = img if final else aux["padded"]
    assert abs_err(img, unfiltered) > 20 * IMG_ATOL                # the filter changes this frame
    gen = torch.Generator().manual_seed(0)
    go = torch.rand(out.shape, generator=gen, dtype=torch.float64) * 2 - 1
    out.backward(go)
    sp = _splatter(g, v, cuda, f3, sh_eval=sh_eval, filter2d=mode, scale_activation=act)
    if final:
        got = sp(0)
    else:
        sp.set_camera(0)
        got = sp.render_padded()
    got.backward(go.float().to(cuda))
    torch.cuda.synchronize()
    assert abs_err(got, out) < IMG_ATOL
    for q in NAMES:
        gq = getattr(sp.gaussian_3ds, q).grad
        assert bool(torch.isfinite(gq).all()), q
        assert rel_err(gq, p[q].grad) < GRAD_RTOL, (q, rel_err(gq, p[q].grad))


def test_aux_maps_and_background_vs_oracle(gs, cuda):
    g, v, cam = scene(4000, 128, 96, k=1, opa_range=(0.05, 0.9), sigma_px=(0.3, 3.0))
    f3 = _scene_filter(gs, cuda, g, v)
    p = {q: t.double().clone().requires_grad_(True) for q, t in g.items()}
    with F3.applied(f3.double()):
        o = F.render_maps(*(p[q] for q in NAMES), cam, "antialias", background=BG,
                          depth_key=device_depth_keys(g, cam, cuda))
    gen = torch.Generator().manual_seed(2)
    ga = torch.rand(o["alpha"].shape, generator=gen, dtype=torch.float64) * 2 - 1
    gi = torch.rand(o["image"].shape, generator=gen, dtype=torch.float64) * 2 - 1
    ((o["alpha"] * ga).sum() + (o["image"] * gi).sum()).backward()
    sp = _splatter(g, v, cuda, f3, filter2d="antialias")
    m = sp.render_maps(0, background=BG)
    ((m["alpha"] * ga.float().to(cuda)).sum() + (m["image"] * gi.float().to(cuda)).sum()).backward()
    assert abs_err(m["image"], o["image"]) < IMG_ATOL and abs_err(m["alpha"], o["alpha"]) < IMG_ATOL
    assert abs_err(m["depth"], o["depth"]) < 1e-4 * float(o["depth"].detach().abs().max())
    for q in NAMES:
        assert rel_err(getattr(sp.gaussian_3ds, q).grad, p[q].grad) < GRAD_RTOL, q


def test_camera_gradient_single_and_batched_vs_oracle(gs, cuda):
    """render_at_pose (one view) and render_batch_at_poses (B = 4): the image, the parameter gradients (the sum over
    the views) and each view's pose gradient against the oracle."""
    w, h = 112, 80
    g = S.make_gaussians(3000, w, h, seed=2, opa_range=(0.05, 0.9), sigma_px=(0.3, 3.0))
    views = [S.make_view(w, h, k) for k in range(4)]
    f3 = _compute(gs, gs[0].RenderContext(), g["pos"].to(cuda), views, variance=VAR).cpu()
    import splatter
    vd = [dict(width=v.width, height=v.height, focal_x=v.fx, focal_y=v.fy, rot=v.rot, tran=v.tran) for v in views]
    p = {q: t.double().clone().requires_grad_(True) for q, t in g.items()}
    rots = [torch.as_tensor(v.rot, dtype=torch.float64).clone().requires_grad_(True) for v in views]
    trans = [torch.as_tensor(v.tran, dtype=torch.float64).clone().requires_grad_(True) for v in views]
    gen = torch.Generator().manual_seed(4)
    gos = [torch.rand(h, w, 3, generator=gen, dtype=torch.float64) * 2 - 1 for _ in views]
    imgs = []
    with F3.applied(f3.double()):
        for k, v in enumerate(views):
            cam = O.Camera(w, h, v.fx, v.fy, rots[k], trans[k], v.near)
            dk = device_depth_keys(g, O.Camera(w, h, v.fx, v.fy, v.rot, v.tran, v.near), cuda)
            imgs.append(F.render_maps(*(p[q] for q in NAMES), cam, "antialias", depth_key=dk)["image"])
    sum((im * go).sum() for im, go in zip(imgs, gos)).backward()
    for batched in (False, True):
        sp = splatter.Splatter.from_tensors(g, vd, device=cuda, filter2d="antialias", filter3d=True,
                                            filter3d_variance=VAR)
        sp._set_filter3d(f3.to(cuda))
        R = torch.stack([torch.as_tensor(v.rot) for v in views]).to(cuda).requires_grad_(True)
        T = torch.stack([torch.as_tensor(v.tran) for v in views]).to(cuda).requires_grad_(True)
        if batched:
            out = sp.render_batch_at_poses(R, T, list(range(4)))["image"]
            (out * torch.stack(gos).float().to(cuda)).sum().backward()
            for k in range(4):
                assert abs_err(out[k], imgs[k]) < IMG_ATOL, k
            for q in NAMES:
                assert rel_err(getattr(sp.gaussian_3ds, q).grad, p[q].grad) < GRAD_RTOL, q
        else:
            out = sp.render_at_pose(R[0], T[0], camera_id=0)["image"]
            (out * gos[0].float().to(cuda)).sum().backward()
            assert abs_err(out, imgs[0]) < IMG_ATOL
        for k in range(4 if batched else 1):
            assert rel_err(R.grad[k], rots[k].grad) < 5 * GRAD_RTOL, (batched, k, rel_err(R.grad[k], rots[k].grad))
            assert rel_err(T.grad[k], trans[k].grad) < 5 * GRAD_RTOL, (batched, k)


def test_feature_maps_follow_the_filter(gs, cuda):
    """F = 8 features: the image of render_features equals render_maps' under the same filter, and the features'
    weights are the filtered ones (a constant feature gives the alpha map)."""
    g, v, cam = scene(3000, 128, 96, k=1, sigma_px=(0.3, 3.0))
    f3 = _scene_filter(gs, cuda, g, v)
    g["feat"] = torch.ones(3000, 8)
    sp = _splatter(g, v, cuda, f3, filter2d="antialias", n_features=8)
    a = sp.render_features(0)
    (a["features"].sum() + a["image"].sum()).backward()
    for q in NAMES + ("feat",):
        assert bool(torch.isfinite(getattr(sp.gaussian_3ds, q).grad).all()), q
    with torch.no_grad():
        b = sp.render_maps(0)
    assert abs_err(a["image"], b["image"]) < 1e-6
    assert abs_err(a["features"][..., 3], b["alpha"]) < 1e-5


@pytest.mark.parametrize("mode", ["none", "antialias"])
@pytest.mark.parametrize("sh_dim", [3, 48])
def test_zero_filter_is_bit_identical(gs, cuda, mode, sh_dim):
    """An all-zero filter renders and differentiates exactly as a context without one (plain and batched)."""
    import renderer
    g, v, cam = scene(4000, 128, 96, k=1, sh_dim=sh_dim)
    res = []
    for f in (None, torch.zeros(4000, device=cuda)):
        rctx = gs[0].RenderContext()
        rctx.set_sh_eval(renderer.SH_EVAL["gaussian"])
        rctx.set_filter2d(renderer.FILTER2D[mode], 0.3)
        rctx.set_filter3d(f)
        prm = {q: t.to(cuda).clone().requires_grad_(True) for q, t in g.items()}
        img, dep, alp, _ = renderer.render_frame_aux(rctx, *(prm[q] for q in NAMES), v.width, v.height, v.fx, v.fy,
                                                     v.rot, v.tran, v.near, 0.05, "abs", background=BG, final=True)
        (img.sum() + alp.sum()).backward()
        bi, _, ba, _ = renderer.render_frame_batch(rctx, *(t.detach() for t in (prm[q] for q in NAMES)), v.width,
                                                  v.height, [v.fx, v.fx], [v.fy, v.fy],
                                                  torch.stack([torch.as_tensor(v.rot)] * 2),
                                                  torch.stack([torch.as_tensor(v.tran)] * 2), v.near, 0.05, "abs",
                                                  final=True)
        res.append([img, alp, bi, ba] + [prm[q].grad for q in NAMES])
    for a, b in zip(*res):
        assert torch.equal(a, b)


def test_extreme_scales_give_finite_outputs(gs, cuda):
    import renderer
    g, v, cam = scene(3000, 128, 96, k=1)
    raw = g["scale"].abs().log()
    raw[::5] = -200.0          # exp underflows to 0: opacity 0, zero gradients
    raw[1::5] = 4.0            # huge
    raw[2::5, 0] = -60.0       # needles
    g["scale"] = raw
    f3 = _scene_filter(gs, cuda, g, v)
    rctx = gs[0].RenderContext()
    rctx.set_filter2d(renderer.FILTER2D["antialias"], 0.3)
    rctx.set_filter3d(f3.to(cuda))
    prm = {q: t.to(cuda).clone().requires_grad_(True) for q, t in g.items()}
    img, _ = renderer.render_frame_final(rctx, *(prm[q] for q in NAMES), v.width, v.height, v.fx, v.fy, v.rot, v.tran,
                                         v.near, 0.05, "exp")
    img.sum().backward()
    assert bool(torch.isfinite(img).all())
    for q in NAMES:
        assert bool(torch.isfinite(prm[q].grad).all()), q
    assert float(prm["opa"].grad[::5].abs().max()) == 0.0


def test_densify_stats_max_radius_uses_the_filtered_covariance(gs, cuda):
    g, v, cam = scene(4000, 128, 96, k=1, sigma_px=(0.2, 2.0))
    f3 = _scene_filter(gs, cuda, g, v)
    sp = _splatter(g, v, cuda, f3, filter2d="dilate", densify_stats="grad")
    sp(0).sum().backward()
    got = sp.densify_stats.max_radius.cpu()
    # expected: the dilated 2-D covariance of the filtered scale, from the oracle's projection in fp64
    nq, ns, _, _ = O.preactivate(g["quat"].double(), g["scale"].double(), g["opa"].double(), g["rgb"].double())
    sf, _ = F3.filtered(ns, torch.ones(4000, dtype=torch.float64), f3.double())
    rp, rc, mask = O.global_culling(g["pos"].double(), nq, sf, cam.rot.double(), cam.tran.double(), cam.near,
                                    cam.half_w, cam.half_h)
    ex, ey = F.filter_eps(cam, 0.3)
    a = (rc[:, 0, 0] + ex) * cam.fx ** 2
    d = (rc[:, 1, 1] + ey) * cam.fy ** 2
    b = rc[:, 0, 1] * cam.fx * cam.fy
    lmax = 0.5 * (a + d) + torch.sqrt((0.5 * (a - d)) ** 2 + b * b)
    exp_r = torch.ceil(3 * torch.sqrt(lmax))
    counted = sp.densify_stats.count.cpu() > 0
    assert int(counted.sum()) > 1000
    assert float((got[counted] - exp_r[counted].float()).abs().max()) <= 1.0
    # and the unfiltered radius would be smaller for the Gaussians the filter widened
    rp0, rc0, _ = O.global_culling(g["pos"].double(), nq, ns, cam.rot.double(), cam.tran.double(), cam.near,
                                   cam.half_w, cam.half_h)
    assert bool((got[counted] >= torch.ceil(3 * torch.sqrt(rc0[counted, 0, 0] * cam.fx ** 2)).float() - 1).all())
    assert float((got[counted] - torch.ceil(3 * torch.sqrt((rc0[counted, 0, 0] + ex) * cam.fx ** 2)).float()).max()) > 1


def test_gradient_push_on_one_gpu_bucket(gs, cuda):
    """One backward with a world-2 push configured on one device: the floats of rank 0's slice land in the bucket, the
    others in rank 1's staging slot 0; reassembled they are the plain backward's gradients bit for bit."""
    import renderer
    g, v, cam = scene(3000, 128, 96, k=1)
    f3 = _scene_filter(gs, cuda, g, v)
    plain, pushed = None, None
    for push in (False, True):
        rctx = gs[0].RenderContext()
        rctx.set_filter2d(renderer.FILTER2D["antialias"], 0.3)
        rctx.set_filter3d(f3.to(cuda))
        prm = {q: t.to(cuda).clone().requires_grad_(True) for q, t in g.items()}
        state = {}
        if push:
            def alloc(numel, dev):
                per = (numel + 7) // 8 * 4
                state["per"] = per
                state["bucket"] = torch.zeros(2 * per, device=dev)
                state["st"] = [torch.zeros(2 * per, device=dev) for _ in range(2)]
                return state["bucket"], (state["bucket"].data_ptr(), [s.data_ptr() for s in state["st"]], per, 0)
            renderer.set_flat_grad_allocator(alloc)
        try:
            img, _ = renderer.render_frame_final(rctx, *(prm[q] for q in NAMES), v.width, v.height, v.fx, v.fy,
                                                 v.rot, v.tran, v.near, 0.05, "abs")
            img.sum().backward()
            torch.cuda.synchronize()
        finally:
            renderer.set_flat_grad_allocator(None)
        flat = torch.cat([prm[q].grad.reshape(-1) for q in NAMES])
        if push:
            per = state["per"]
            full = torch.cat([state["bucket"][:per], state["st"][1][:per]])
            segs, o = [], 0
            for q in NAMES:
                k = prm[q].numel()
                segs.append(full[o:o + k])
                o += (k + 3) // 4 * 4
            pushed = torch.cat(segs)
        else:
            plain = flat
    assert torch.equal(plain, pushed)


def test_refusals_launch_nothing(gs, cuda):
    import renderer
    g, v, cam = scene(500, 64, 48, k=1)
    rctx = gs[0].RenderContext()
    with pytest.raises(Exception, match="filter3d"):
        rctx.set_filter3d(torch.zeros(500))                       # a CPU tensor
    with pytest.raises(Exception, match="filter3d"):
        rctx.set_filter3d(torch.zeros(500, 1, device=cuda))
    rctx.set_filter3d(torch.zeros(499, device=cuda))
    prm = {q: t.to(cuda) for q, t in g.items()}
    torch.cuda.synchronize()
    before = gs[0].kernel_launches()
    with pytest.raises(RuntimeError, match="3-D filter is sized for another n"):
        renderer.render_frame_final(rctx, *(prm[q] for q in NAMES), v.width, v.height, v.fx, v.fy, v.rot, v.tran,
                                    v.near, 0.05, "abs")
    with pytest.raises(RuntimeError, match="3-D filter is sized for another n"):
        renderer.render_frame_batch(rctx, *(prm[q] for q in NAMES), v.width, v.height, [v.fx], [v.fy],
                                    torch.as_tensor(v.rot)[None], torch.as_tensor(v.tran)[None], v.near, 0.05, "abs")
    c = _cams_of([v])
    for kw in (dict(variance=0.0), dict(margin=-1.0), dict(variance=float("nan"))):
        a = dict(near=0.3, margin=0.15, variance=0.2)
        a.update(kw)
        with pytest.raises(RuntimeError, match="gs_filter3d_compute"):
            gs[0].filter3d_compute(rctx, prm["pos"], c["size"], c["focal"], c["rot"], c["tran"], a["near"],
                                   a["margin"], a["variance"])
    assert gs[0].kernel_launches() == before
    rctx.set_filter3d(None)                                        # off again: the frame renders
    renderer.render_frame_final(rctx, *(prm[q] for q in NAMES), v.width, v.height, v.fx, v.fy, v.rot, v.tran, v.near,
                                0.05, "abs")


def test_training_through_splatter(gs, cuda, tmp_path):
    """200 Mip-Splatting-configured steps (antialias, variance 0.1, the filter recomputed every 100 steps and after a
    densification at step 100); a resume from the checkpoint of step 150 reproduces steps 150..199 bit for bit; the
    baked parameters rendered without a 3-D filter match the filtered frame."""
    import checkpoint
    import optim
    import splatter
    w, h = 128, 96
    teacher = S.make_gaussians(3000, w, h, seed=0)
    views = [S.make_view(w, h, k) for k in range(4)]
    vd = [dict(width=v.width, height=v.height, focal_x=v.fx, focal_y=v.fy, rot=v.rot, tran=v.tran) for v in views]
    with torch.no_grad():
        gts = [splatter.Splatter.from_tensors(teacher, vd, device=cuda)(k).clone() for k in range(4)]
    student = {k: t.clone() for k, t in teacher.items()}
    student["opa"] = torch.full_like(student["opa"], -1.0)
    kw = dict(filter2d="antialias", filter3d=True, filter3d_variance=0.1, densify_stats="grad")

    def make_opt(sp):
        gg = sp.gaussian_3ds
        return optim.FlatAdam([{"params": gg.opa, "lr": 0.03}, {"params": gg.rgb, "lr": 0.03},
                               {"params": gg.pos, "lr": 0.003}, {"params": gg.scale, "lr": 0.003},
                               {"params": gg.quat, "lr": 0.003}], betas=(0.9, 0.99))

    def run(sp, opt, start, stop, ckpt_at=None):
        for it in range(start, stop):
            if it % 100 == 0:
                sp.compute_filter3d()
            opt.zero_grad(set_to_none=True)
            img = sp(it % 4)
            (img - gts[it % 4]).abs().mean().backward()
            opt.step()
            if it == 100:
                n0 = sp.gaussian_3ds.pos.shape[0]
                sp.adaptive_control_screen(0.01, 10.0, grad_thresh=1e-7)
                assert sp.gaussian_3ds.pos.shape[0] != n0
                assert sp.filter3d.numel() == sp.gaussian_3ds.pos.shape[0]
                opt = make_opt(sp)
            if ckpt_at is not None and it == ckpt_at - 1:
                sp.save_checkpoint(str(tmp_path / "c.pth"), opt, iteration=it + 1)
        return opt

    torch.manual_seed(0)
    sp = splatter.Splatter.from_tensors(student, vd, device=cuda, **kw)
    opt = run(sp, make_opt(sp), 0, 200, ckpt_at=150)
    final = {q: getattr(sp.gaussian_3ds, q).detach().clone() for q in NAMES}
    f_end = sp.filter3d.clone()
    assert bool((f_end > 0).any())

    sp2 = splatter.Splatter.from_tensors(student, vd, device=cuda, **kw)
    checkpoint.load_checkpoint(str(tmp_path / "c.pth"), sp2)
    opt2 = make_opt(sp2)
    checkpoint.load_checkpoint(str(tmp_path / "c.pth"), None, opt2)
    run(sp2, opt2, 150, 200)
    for q in NAMES:
        assert torch.equal(getattr(sp2.gaussian_3ds, q).detach(), final[q]), q
    assert torch.equal(sp2.filter3d, f_end)

    # bake: the folded parameters rendered with no 3-D filter give the filtered frame
    with torch.no_grad():
        ref = sp(1)
        opa, scale = sp.bake_filter3d()
        g = {q: getattr(sp.gaussian_3ds, q).detach().clone() for q in NAMES}
        g["opa"], g["scale"] = opa, scale
        baked = splatter.Splatter.from_tensors({k: t.cpu() for k, t in g.items()}, vd, device=cuda,
                                               filter2d="antialias")(1)
    assert abs_err(baked, ref) < 1e-5
