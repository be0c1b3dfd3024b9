"""Camera lenses on the fused frame path (gs_ctx_set_lens, RenderContext.set_lens, `Splatter(camera_model="colmap")`)
against the fp64 oracle of tests/lens_oracle.py: frames and their five gradients, the culling mask, the image-centre
pinhole's bit identity with a frame without a lens, a principal point as a crop of a wider frame, COLMAP's pixel
convention, aux maps and camera gradients, batched frames, the densification statistics, the refusals and a short
COLMAP training run."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

import gs_oracle as O
import lens_oracle as L
from helpers import abs_err, rel_err, scene

pytestmark = pytest.mark.gpu

IMG_ATOL = 1e-4
GRAD_RTOL = 1e-3
NAMES = ("pos", "rgb", "opa", "quat", "scale")
LENSES = {
    "pinhole-offset": dict(model="PINHOLE", dcx=5.5, dcy=-3.25, k=[0.0] * 4),
    "opencv": dict(model="OPENCV", dcx=2.0, dcy=1.5, k=[-0.12, 0.03, 0.002, -0.001]),
    "fisheye": dict(model="FISHEYE", dcx=-1.5, dcy=2.5, k=[0.05, -0.02, 0.004, -0.0005]),
    # rho_max = sqrt(1 / 4.5) = 0.471 lies inside the test scenes: the fold-back limit culls Gaussians whose distorted
    # mean would still be in the image
    "opencv-fold": dict(model="OPENCV", dcx=-2.5, dcy=1.0, k=[-1.5, 0.0, 0.0, 0.0]),
}


def _lens(name, w, h):
    d = LENSES[name]
    return dict(model=d["model"], cx=w / 2 + d["dcx"], cy=h / 2 + d["dcy"], k=list(d["k"]))


def _set(rctx, lenses):
    if lenses is None:
        rctx.set_lens(None, None)
        return
    rctx.set_lens([L.MODELS[ln["model"]] for ln in lenses],
                  torch.tensor([[ln["cx"], ln["cy"], *ln["k"]] for ln in lenses], dtype=torch.float32))


def _ctx(gs, filter2d="none", sh_eval="pixel"):
    import renderer
    rctx = gs[0].RenderContext()
    rctx.set_sh_eval(renderer.SH_EVAL[sh_eval])
    rctx.set_filter2d(renderer.FILTER2D[filter2d], 0.3)
    return rctx


def _dev(g, dev):
    return {q: t.to(dev).contiguous().requires_grad_(True) for q, t in g.items()}


def _depth_keys(g, cam, dev):
    """fp32 |p_c| as the device computes it, for every Gaussian in front of the near plane (no frustum test)."""
    import renderer
    nq, ns, _, _ = O.preactivate(g["quat"], g["scale"], g["opa"], g["rgb"])
    rp, _, _ = renderer.global_culling(g["pos"].to(dev), nq.to(dev).contiguous(), ns.to(dev).contiguous(),
                                       cam.rot.to(dev), cam.tran.to(dev), cam.near, 1e30, 1e30)
    return rp[:, 2].detach().cpu()


def _stable(g, cam, lens, eps=1e-5):
    """The Gaussians whose culling and tile rectangle do not change under a relative perturbation eps of the stored
    mean, the covariance and rho (fp32 and fp64 agree on them: no tie at rho_max, the frustum or a tile edge)."""
    p = {q: t.double() for q, t in g.items()}
    nq, ns, _, _ = O.preactivate(p["quat"], p["scale"], p["opa"], p["rgb"])
    ox, oy = L.offsets(lens, cam.width, cam.height, cam.fx, cam.fy)
    rp, rc, mask = L.global_culling_lens(p["pos"], nq, ns, cam.rot.double(), cam.tran.double(), cam.near, cam.half_w,
                                         cam.half_h, lens, ox, oy)
    pc = p["pos"] @ cam.rot.double().T + cam.tran.double()
    rho = (pc[:, :2] / pc[:, 2:3]).norm(dim=-1)
    rm = L.rho_max(lens["model"], lens["k"])
    keep = (rho - rm).abs() > eps * max(1.0, rm if math.isfinite(rm) else 1.0)
    keep &= ((rp[:, 0].abs() - cam.half_w).abs() > eps) & ((rp[:, 1].abs() - cam.half_h).abs() > eps)
    base = O.tile_rects(rp[:, :2], rc, 0.05, cam.tile_lx, cam.tile_ly, cam.ntx, cam.nty, cam.leftmost, cam.topmost)
    for s in (1 - eps, 1 + eps):
        for pos2d, cov in ((rp[:, :2] * s, rc), (rp[:, :2] + eps * cam.tile_lx, rc * s),
                           (rp[:, :2] - eps * cam.tile_lx, rc)):
            r = O.tile_rects(pos2d, cov, 0.05, cam.tile_lx, cam.tile_ly, cam.ntx, cam.nty, cam.leftmost, cam.topmost)
            for a, b in zip(base, r):
                keep &= (a == b) | ~mask.bool()
    idx = torch.nonzero(keep).squeeze(-1)
    return {q: t[idx].contiguous() for q, t in g.items()}


def _upstream(h, w, seed=0):
    gen = torch.Generator().manual_seed(seed)
    return torch.rand(h, w, 3, generator=gen, dtype=torch.float64) * 2 - 1


def _render_final(gs, rctx, p, cam, v):
    import renderer
    return renderer.render_frame_final(rctx, p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], v.width, v.height,
                                       v.fx, v.fy, v.rot, v.tran, v.near, 0.05, "abs")


# (colour width, sh_eval): RGB logits, and per-Gaussian SH of degree 3
COLOURS = {"rgb": (3, "pixel"), "sh48-gauss": (48, "gaussian")}


@pytest.mark.parametrize("colour", list(COLOURS))
@pytest.mark.parametrize("filter2d", ["none", "antialias"])
@pytest.mark.parametrize("lens", list(LENSES))
def test_lens_frame_vs_oracle(gs, cuda, lens, filter2d, colour):
    """A frame through each lens against the oracle, RGB and per-Gaussian SH of degree 3: image 1e-4 abs, all five
    gradients 1e-3 relative, culling mask equal (with a finite rho_max too, which must cull some Gaussians)."""
    import sh_gaussian_oracle as G
    sh_dim, sh_eval = COLOURS[colour]
    g0, v, cam = scene(3000, 128, 96, k=1, sh_dim=sh_dim, opa_range=(0.05, 0.9))
    ln = _lens(lens, v.width, v.height)
    g = _stable(g0, cam, ln)
    p = {q: t.double().clone().requires_grad_(True) for q, t in g.items()}
    dk = _depth_keys(g, cam, cuda)
    rgb = p["rgb"] if sh_dim == 3 else G.gaussian_logits(p["pos"], p["rgb"], cam)
    if filter2d == "none":
        ref, aux = L.render(p["pos"], rgb, p["opa"], p["quat"], p["scale"], cam, ln, depth_key=dk)
    else:
        # the oracle's 2-D filter acts on the covariance the lens produced: route gs_oracle.global_culling through it
        ref, aux = _render_filtered(dict(p, rgb=rgb), cam, ln, filter2d, dk)
    if lens == "opencv-fold":
        rm = L.rho_max(ln["model"], ln["k"])
        pc = g["pos"].double() @ cam.rot.double().T + cam.tran.double()
        past = (pc[:, :2] / pc[:, 2:3]).norm(dim=-1) >= rm
        assert math.isfinite(rm) and int(past.sum()) > 20 and not bool(aux["mask"][past].any())
    go = _upstream(v.height, v.width)
    ref.backward(go)
    rctx = _ctx(gs, filter2d, sh_eval)
    _set(rctx, [ln])
    d = _dev(g, cuda)
    img, mask = _render_final(gs, rctx, d, cam, v)
    img.backward(go.float().to(cuda))
    torch.cuda.synchronize()
    assert torch.equal(mask.cpu(), aux["mask"].cpu())
    assert abs_err(img, ref) < IMG_ATOL
    for q in NAMES:
        assert bool(torch.isfinite(d[q].grad).all()), q
        assert rel_err(d[q].grad, p[q].grad) < GRAD_RTOL, (q, rel_err(d[q].grad, p[q].grad))


def _render_filtered(p, cam, ln, mode, dk):
    """L.render with the 2-D filter of filter_oracle applied after the lens."""
    import filter_oracle as F
    orig = O.global_culling

    def culled(pos, nq, ns, rot, tran, near, hw, hh):
        ox, oy = L.offsets(ln, cam.width, cam.height, cam.fx, cam.fy)
        return L.global_culling_lens(pos, nq, ns, rot, tran, near, hw, hh, ln, ox, oy)

    O.global_culling = culled
    try:
        img, aux = F.render(p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], cam, mode, return_aux=True,
                            depth_key=dk)
    finally:
        O.global_culling = orig
    return img, aux


@pytest.mark.parametrize("sh", [3, 48])
def test_lens_centre_pinhole_is_bit_identical(gs, cuda, sh):
    """A PINHOLE lens at (W/2, H/2) renders and differentiates the bits of a frame without a lens: image, aux maps,
    parameter gradients and the camera gradient."""
    import renderer
    g, v, cam = scene(3000, 120, 88, k=1, sh_dim=sh)
    sh_eval = "gaussian" if sh != 3 else "pixel"
    out = []
    for lenses in (None, [dict(model="PINHOLE", cx=v.width / 2, cy=v.height / 2, k=[0.0] * 4)]):
        rctx = _ctx(gs, sh_eval=sh_eval)
        _set(rctx, lenses)
        d = _dev(g, cuda)
        rot = v.rot.to(cuda).requires_grad_(True)
        tran = v.tran.to(cuda).requires_grad_(True)
        img, depth, alpha, mask = renderer.render_frame_cam(rctx, d["pos"], d["rgb"], d["opa"], d["quat"], d["scale"],
                                                            v.width, v.height, v.fx, v.fy, rot, tran, v.near, 0.05,
                                                            "abs", background=(0.2, 0.3, 0.4), final=True)
        gen = torch.Generator().manual_seed(3)
        ups = [torch.rand(t.shape, generator=gen).to(cuda) * 2 - 1 for t in (img, depth, alpha)]
        torch.autograd.backward([img, depth, alpha], ups)
        torch.cuda.synchronize()
        out.append([img, depth, alpha, mask, rot.grad, tran.grad] + [d[q].grad for q in NAMES])
    for a, b in zip(*out):
        assert torch.equal(a, b)


@pytest.mark.parametrize("axis", ["x", "y"])
def test_lens_principal_point_is_a_crop(gs, cuda, axis):
    """A principal point 32 px off the centre equals a crop of the centred frame 64 px wider (or taller): image within
    1e-5 abs, gradients within 1e-4 relative under a gradient on the shared pixels only."""
    import renderer
    W, H = (128, 96) if axis == "x" else (96, 128)
    g, v, cam = scene(3000, 96, 96, k=0)
    fx = v.fx
    gn = torch.Generator().manual_seed(2)
    up = _upstream(H, W, 4).float()
    res = []
    for wide in (False, True):
        w = W + 64 if (wide and axis == "x") else W
        h = H + 64 if (wide and axis == "y") else H
        rctx = _ctx(gs)
        _set(rctx, None if wide else [dict(model="PINHOLE", cx=W / 2 + (32 if axis == "x" else 0),
                                           cy=H / 2 + (32 if axis == "y" else 0), k=[0.0] * 4)])
        d = _dev(g, cuda)
        img, _ = renderer.render_frame_final(rctx, d["pos"], d["rgb"], d["opa"], d["quat"], d["scale"], w, h, fx, fx,
                                             v.rot, v.tran, v.near, 0.05, "abs")
        upw = torch.zeros(h, w, 3)
        upw[:H, :W] = up
        img.backward(upw.to(cuda))
        torch.cuda.synchronize()
        res.append((img[:H, :W].detach().cpu(), {q: d[q].grad.cpu() for q in NAMES}))
    assert abs_err(res[0][0], res[1][0]) < 1e-5
    for q in NAMES:
        assert rel_err(res[0][1][q], res[1][1][q]) < 1e-4, q


def _colmap_project(pt, rot, tran, fx, fy, ln):
    """COLMAP's world-to-image of one point, independently of the oracle's map (numpy fp64)."""
    pc = np.asarray(rot, np.float64) @ np.asarray(pt, np.float64) + np.asarray(tran, np.float64)
    u, w = pc[0] / pc[2], pc[1] / pc[2]
    k = ln["k"]
    if ln["model"] == "OPENCV":
        r2 = u * u + w * w
        rad = 1 + k[0] * r2 + k[1] * r2 * r2
        du = u * rad + 2 * k[2] * u * w + k[3] * (r2 + 2 * u * u)
        dw = w * rad + k[2] * (r2 + 2 * w * w) + 2 * k[3] * u * w
        u, w = du, dw
    elif ln["model"] == "FISHEYE":
        r = math.hypot(u, w)
        if r > 1e-12:
            th = math.atan(r)
            thd = th * (1 + k[0] * th ** 2 + k[1] * th ** 4 + k[2] * th ** 6 + k[3] * th ** 8)
            u, w = u * thd / r, w * thd / r
    return fx * u + ln["cx"], fy * w + ln["cy"]


@pytest.mark.parametrize("where", ["centre", "corner"])
@pytest.mark.parametrize("lens", ["pinhole-offset", "opencv", "fisheye"])   # the corner lies past opencv-fold's rho_max
def test_lens_pixel_convention(gs, cuda, lens, where):
    """A small isotropic Gaussian renders its alpha-weighted centroid within 0.05 px of COLMAP's projection."""
    import renderer
    W, H = 160, 128
    v = scene(1, W, H, k=0)[1]
    ln = _lens(lens, W, H)
    target = (W / 2 + 3.3, H / 2 - 2.6) if where == "centre" else (W * 0.85, H * 0.82)
    # the point on the ray of the undistorted position whose COLMAP projection is the target (solved on the oracle map
    # by Newton; the check below projects it with the independent restatement)
    a = torch.tensor([(target[0] - ln["cx"]) / v.fx], dtype=torch.float64)
    b = torch.tensor([(target[1] - ln["cy"]) / v.fy], dtype=torch.float64)
    ua, ub = a.clone(), b.clone()
    for _ in range(50):
        ad, bd = L.lens_map(ua, ub, ln["model"], ln["k"])
        J = L.lens_jacobian(ua, ub, ln["model"], ln["k"])[0]
        step = torch.linalg.solve(J, torch.stack([ad - a, bd - b]).reshape(2))
        ua, ub = ua - step[0], ub - step[1]
    z = 3.0
    pc = torch.tensor([float(ua) * z, float(ub) * z, z], dtype=torch.float64)
    R, t = v.rot.double(), v.tran.double()
    pw = torch.linalg.solve(R, pc - t)
    want = _colmap_project(pw.numpy(), R.numpy(), t.numpy(), v.fx, v.fy, ln)
    # 1.2 px: wide enough that the pixel samples' centroid is the Gaussian's mean (a sub-pixel one is pulled towards
    # the nearest pixel centre)
    s = 1.2 * z / v.fx
    g = dict(pos=pw.float().reshape(1, 3), rgb=torch.full((1, 3), 8.0), opa=torch.full((1,), 0.0),
             quat=torch.tensor([[1.0, 0.0, 0.0, 0.0]]), scale=torch.full((1, 3), s))
    rctx = _ctx(gs)
    _set(rctx, [ln])
    d = _dev(g, cuda)
    img, _, alpha, _ = renderer.render_frame_aux(rctx, d["pos"], d["rgb"], d["opa"], d["quat"], d["scale"], W, H,
                                                 v.fx, v.fy, v.rot, v.tran, v.near, 0.05, "abs", final=True)
    al = alpha.detach().double().cpu()
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    cx = float((al * (xs + 0.5)).sum() / al.sum())
    cy = float((al * (ys + 0.5)).sum() / al.sum())
    assert abs(cx - want[0]) < 0.05 and abs(cy - want[1]) < 0.05, (cx, cy, want)


def test_lens_aux_and_camera_grads_vs_oracle(gs, cuda):
    """The image and the camera gradient of render_frame_cam through a fisheye lens against the oracle."""
    import renderer
    g0, v, cam = scene(3000, 128, 96, k=1)
    ln = _lens("fisheye", v.width, v.height)
    g = _stable(g0, cam, ln)
    dk = _depth_keys(g, cam, cuda)
    # oracle: the depth map is sum w |p_c| and alpha sum w; the camera enters through rot / tran
    p = {q: t.double().clone().requires_grad_(True) for q, t in g.items()}
    rot = cam.rot.double().clone().requires_grad_(True)
    tran = cam.tran.double().clone().requires_grad_(True)
    cam2 = O.Camera(cam.width, cam.height, cam.fx, cam.fy, rot, tran, cam.near)
    ref, aux = L.render(p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], cam2, ln, depth_key=dk)
    go = _upstream(v.height, v.width)
    ref.backward(go)
    rctx = _ctx(gs)
    _set(rctx, [ln])
    d = _dev(g, cuda)
    drot = v.rot.to(cuda).requires_grad_(True)
    dtran = v.tran.to(cuda).requires_grad_(True)
    img, depth, alpha, mask = renderer.render_frame_cam(rctx, d["pos"], d["rgb"], d["opa"], d["quat"], d["scale"],
                                                        v.width, v.height, v.fx, v.fy, drot, dtran, v.near, 0.05,
                                                        "abs", final=True)
    img.backward(go.float().to(cuda))
    torch.cuda.synchronize()
    assert abs_err(img, ref) < IMG_ATOL
    for q in NAMES:
        assert rel_err(d[q].grad, p[q].grad) < GRAD_RTOL, q
    assert rel_err(drot.grad, rot.grad) < GRAD_RTOL
    assert rel_err(dtran.grad, tran.grad) < GRAD_RTOL
    assert float(alpha.detach().max()) > 0 and bool(torch.isfinite(depth).all())


def test_lens_batch_matches_single_views(gs, cuda):
    """B = 3 views with three different lenses equal three single-view frames (images, masks, summed gradients);
    a lens count other than 1 or B is refused."""
    import renderer
    g, v, cam = scene(3000, 128, 96, k=1)
    names = ["pinhole-offset", "opencv", "fisheye"]
    vs = [scene(1, 128, 96, k=k)[1] for k in (0, 1, 2)]
    lenses = [_lens(nm, v.width, v.height) for nm in names]
    up = [_upstream(v.height, v.width, s).float().to(cuda) for s in range(3)]
    singles, sgrads = [], {q: 0 for q in NAMES}
    for vi, ln, u in zip(vs, lenses, up):
        rctx = _ctx(gs)
        _set(rctx, [ln])
        d = _dev(g, cuda)
        img, _ = _render_final(gs, rctx, d, cam, vi)
        img.backward(u)
        singles.append(img.detach())
        for q in NAMES:
            sgrads[q] = sgrads[q] + d[q].grad
    rctx = _ctx(gs)
    _set(rctx, lenses)
    d = _dev(g, cuda)
    rots = torch.stack([x.rot for x in vs]).to(cuda)
    trans = torch.stack([x.tran for x in vs]).to(cuda)
    img, depth, alpha, mask = renderer.render_frame_batch(rctx, d["pos"], d["rgb"], d["opa"], d["quat"], d["scale"],
                                                          v.width, v.height, [x.fx for x in vs], [x.fy for x in vs],
                                                          rots, trans, v.near, 0.05, "abs", final=True)
    img.backward(torch.stack(up))
    torch.cuda.synchronize()
    for b in range(3):
        assert abs_err(img[b], singles[b]) < 1e-6, b
    for q in NAMES:
        assert rel_err(d[q].grad, sgrads[q]) < 1e-5, q
    _set(rctx, lenses[:2])
    with pytest.raises(RuntimeError):
        renderer.render_frame_batch(rctx, d["pos"], d["rgb"], d["opa"], d["quat"], d["scale"], v.width, v.height,
                                    [x.fx for x in vs], [x.fy for x in vs], rots, trans, v.near, 0.05, "abs")


def test_lens_densify_stats_max_radius(gs, cuda):
    """The densification statistics' max_radius follows the lensed covariance: a strong barrel lens shrinks it."""
    import splatter
    g, v, cam = scene(2000, 128, 96, k=1)
    radii = []
    for lens in (None, dict(model="OPENCV", cx=64.0, cy=48.0, k=[-0.3, 0.0, 0.0, 0.0])):
        vd = dict(width=v.width, height=v.height, focal_x=v.fx, focal_y=v.fy, rot=v.rot, tran=v.tran)
        if lens:
            vd["lens"] = lens
        sp = splatter.Splatter.from_tensors(g, [vd], device=cuda, densify_stats="grad")
        sp(0).sum().backward()
        torch.cuda.synchronize()
        radii.append(sp.densify_stats.max_radius.detach().cpu().clone())
    seen = (radii[0] > 0) & (radii[1] > 0)
    assert int(seen.sum()) > 100
    assert bool((radii[1][seen] <= radii[0][seen]).all()) and bool((radii[1][seen] < radii[0][seen]).any())


def test_lens_refusals_launch_nothing(gs, cuda):
    """Per-pixel SH with a distortion is refused before any launch; a principal point alone renders."""
    import renderer
    g, v, cam = scene(500, 64, 64, k=0, sh_dim=27)
    rctx = _ctx(gs)
    _set(rctx, [_lens("opencv", 64, 64)])
    d = _dev(g, cuda)
    lib = ctypes.CDLL(os.path.join(os.path.dirname(gs[0].__file__), "libgs_b200.so"))
    lib.gs_kernel_launches.restype = ctypes.c_ulonglong
    torch.cuda.synchronize()
    before = lib.gs_kernel_launches()
    with pytest.raises(RuntimeError, match="principal point"):
        _render_final(gs, rctx, d, cam, v)
    assert lib.gs_kernel_launches() == before
    _set(rctx, [_lens("pinhole-offset", 64, 64)])
    img, _ = _render_final(gs, rctx, d, cam, v)
    img.sum().backward()
    torch.cuda.synchronize()
    assert bool(torch.isfinite(d["pos"].grad).all())


def test_lens_splatter_colmap_fisheye_trains(gs, cuda, tmp_path):
    """Splatter(camera_model="colmap", filter3d=True) on a COLMAP dataset with OPENCV_FISHEYE cameras: 200 steps lower
    the loss, the parameters stay finite, and the 3-D filter is computed through the lenses."""
    import cv2
    import colmap_io
    import splatter
    W, H = 96, 80
    fx = W / (2 * math.tan(math.radians(35)))
    k = [0.04, -0.01, 0.0, 0.0]
    g_true, _, _ = scene(800, W, H, seed=7, k=0)
    cams = {1: colmap_io.Camera(1, "OPENCV_FISHEYE", W, H, np.array([fx, fx, W / 2 + 2.0, H / 2 - 1.5, *k]))}
    (tmp_path / "images").mkdir()
    pts = {}
    for i in range(len(g_true["pos"])):
        pts[i + 1] = colmap_io.Point3D(i + 1, g_true["pos"][i].double().numpy(), np.array([128, 128, 128]), 0.0)
    views, infos = [], {}
    for j, kk in enumerate((0, 1, 7)):
        v = scene(1, W, H, k=kk)[1]
        infos[j + 1] = colmap_io.Image(j + 1, colmap_io.rotmat_to_qvec(v.rot.double().numpy()), v.tran.double().numpy(),
                                       1, f"{j}.png")
        views.append(v)
    colmap_io.write_cameras_binary(str(tmp_path / "cameras.bin"), cams)
    colmap_io.write_images_binary(str(tmp_path / "images.bin"), infos)
    colmap_io.write_points3d_binary(str(tmp_path / "points3D.bin"), pts)
    # ground truth rendered through the same lens from the true scene
    ln = dict(model="FISHEYE", cx=W / 2 + 2.0, cy=H / 2 - 1.5, k=k)
    rctx = _ctx(gs)
    _set(rctx, [ln])
    gt = {q: t.to(cuda) for q, t in g_true.items()}
    for j, v in enumerate(views):
        with torch.no_grad():
            img, _ = _render_final(gs, rctx, gt, None, v)
        cv2.imwrite(str(tmp_path / "images" / f"{j}.png"),
                    cv2.cvtColor((img.clamp(0, 1) * 255).round().byte().cpu().numpy(), cv2.COLOR_RGB2BGR))
    sp = splatter.Splatter(str(tmp_path), str(tmp_path / "images"), device=cuda, camera_model="colmap",
                           filter3d=True)
    assert sp.views[0]["lens"]["model"] == "FISHEYE"
    opt = torch.optim.Adam(sp.parameters(), lr=2e-3)
    losses = []
    for step in range(200):
        i = step % 3
        out = sp(i)
        loss = (out - sp.ground_truth.float()).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    assert np.mean(losses[-15:]) < 0.8 * np.mean(losses[:15])
    for q in NAMES:
        assert bool(torch.isfinite(getattr(sp.gaussian_3ds, q)).all()), q
    assert sp.filter3d is not None and bool(torch.isfinite(sp.filter3d).all()) and bool((sp.filter3d > 0).any())


def _patched_culling(ln, cam):
    """A context in which gs_oracle.global_culling projects through `ln` (for the oracles built on it)."""
    import contextlib

    @contextlib.contextmanager
    def ctx():
        orig = O.global_culling

        def culled(pos, nq, ns, rot, tran, near, hw, hh):
            ox, oy = L.offsets(ln, cam.width, cam.height, cam.fx, cam.fy)
            return L.global_culling_lens(pos, nq, ns, rot, tran, near, hw, hh, ln, ox, oy)

        O.global_culling = culled
        try:
            yield
        finally:
            O.global_culling = orig
    return ctx()


@pytest.mark.parametrize("lens", ["opencv", "fisheye"])
def test_lens_aux_maps_vs_oracle(gs, cuda, lens):
    """Depth and alpha maps over a background through a lens against the oracle: the three maps 1e-4 abs, and all five
    gradients 1e-3 relative under depth-only and alpha-only upstream gradients."""
    import filter_oracle as F
    import renderer
    bg = (0.2, 0.5, 0.9)
    g0, v, cam = scene(3000, 128, 96, k=1)
    ln = _lens(lens, v.width, v.height)
    g = _stable(g0, cam, ln)
    p = {q: t.double().clone().requires_grad_(True) for q, t in g.items()}
    with _patched_culling(ln, cam):
        o = F.render_maps(*(p[q] for q in NAMES), cam, "none", background=bg, depth_key=_depth_keys(g, cam, cuda))
    gen = torch.Generator().manual_seed(5)
    gd = torch.rand(o["depth"].shape, generator=gen, dtype=torch.float64) * 2 - 1
    ga = torch.rand(o["depth"].shape, generator=gen, dtype=torch.float64) * 2 - 1
    rctx = _ctx(gs)
    _set(rctx, [ln])
    for which, upstream in (("depth", gd), ("alpha", ga)):
        ref = torch.autograd.grad(o[which], [p[q] for q in NAMES], upstream, retain_graph=True, allow_unused=True)
        ref = [torch.zeros_like(p[q]) if r is None else r for q, r in zip(NAMES, ref)]   # alpha: no colour term
        d = _dev(g, cuda)
        img, depth, alpha, _ = renderer.render_frame_aux(rctx, *(d[q] for q in NAMES), v.width, v.height, v.fx, v.fy,
                                                         v.rot, v.tran, v.near, 0.05, "abs", background=bg, final=True)
        assert abs_err(img, o["image"]) < IMG_ATOL
        assert abs_err(depth, o["depth"]) < IMG_ATOL * float(o["depth"].detach().abs().max())
        assert abs_err(alpha, o["alpha"]) < IMG_ATOL
        out = depth if which == "depth" else alpha
        out.backward(upstream.float().to(cuda))
        torch.cuda.synchronize()
        for q, r in zip(NAMES, ref):
            assert rel_err(d[q].grad, r) < GRAD_RTOL, (which, q, rel_err(d[q].grad, r))


def test_lens_per_pixel_sh_principal_point_vs_oracle(gs, cuda):
    """SH colour evaluated per pixel with an off-centre principal point (its rays shift with it) against the oracle."""
    g0, v, cam = scene(2500, 112, 80, k=1, sh_dim=27)
    ln = _lens("pinhole-offset", v.width, v.height)
    g = _stable(g0, cam, ln)
    p = {q: t.double().clone().requires_grad_(True) for q, t in g.items()}
    ref, aux = L.render(p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], cam, ln, use_sh_coeff=True,
                        depth_key=_depth_keys(g, cam, cuda))
    go = _upstream(v.height, v.width, 2)
    ref.backward(go)
    rctx = _ctx(gs)
    _set(rctx, [ln])
    d = _dev(g, cuda)
    img, mask = _render_final(gs, rctx, d, cam, v)
    img.backward(go.float().to(cuda))
    torch.cuda.synchronize()
    assert torch.equal(mask.cpu(), aux["mask"].cpu())
    assert abs_err(img, ref) < IMG_ATOL
    for q in NAMES:
        assert rel_err(d[q].grad, p[q].grad) < GRAD_RTOL, (q, rel_err(d[q].grad, p[q].grad))


@pytest.mark.parametrize("sh", [3, 48])
def test_lens_batch_camera_grads_match_single_views(gs, cuda, sh):
    """A batch of 3 views with 3 lenses and per-view camera gradients (render_frame_batch_cam) against 3 single-view
    render_frame_cam frames: per-view rot / tran gradients and the summed parameter gradients, with parameters and
    camera only."""
    import renderer
    g, v, cam = scene(3000, 128, 96, k=1, sh_dim=sh)
    sh_eval = "gaussian" if sh != 3 else "pixel"
    vs = [scene(1, 128, 96, k=k)[1] for k in (0, 1, 2)]
    lenses = [_lens(nm, v.width, v.height) for nm in ("pinhole-offset", "opencv", "fisheye")]
    up = [_upstream(v.height, v.width, s).float().to(cuda) for s in range(3)]
    for cam_only in (False, True):
        single_rt, sgrads = [], {q: 0 for q in NAMES}
        for vi, ln, u in zip(vs, lenses, up):
            rctx = _ctx(gs, sh_eval=sh_eval)
            _set(rctx, [ln])
            d = {q: t.to(cuda).contiguous().requires_grad_(not cam_only) for q, t in g.items()}
            rot = vi.rot.to(cuda).requires_grad_(True)
            tran = vi.tran.to(cuda).requires_grad_(True)
            img, _, _, _ = renderer.render_frame_cam(rctx, *(d[q] for q in NAMES), v.width, v.height, vi.fx, vi.fy,
                                                     rot, tran, v.near, 0.05, "abs", final=True)
            img.backward(u)
            single_rt.append((rot.grad.clone(), tran.grad.clone()))
            if not cam_only:
                for q in NAMES:
                    sgrads[q] = sgrads[q] + d[q].grad
        rctx = _ctx(gs, sh_eval=sh_eval)
        _set(rctx, lenses)
        d = {q: t.to(cuda).contiguous().requires_grad_(not cam_only) for q, t in g.items()}
        rots = torch.stack([x.rot for x in vs]).to(cuda).requires_grad_(True)
        trans = torch.stack([x.tran for x in vs]).to(cuda).requires_grad_(True)
        img, _, _, _ = renderer.render_frame_batch_cam(rctx, *(d[q] for q in NAMES), v.width, v.height,
                                                       [x.fx for x in vs], [x.fy for x in vs], rots, trans, v.near,
                                                       0.05, "abs", final=True)
        img.backward(torch.stack(up))
        torch.cuda.synchronize()
        for b in range(3):
            assert rel_err(rots.grad[b], single_rt[b][0]) < 1e-5, (cam_only, b)
            assert rel_err(trans.grad[b], single_rt[b][1]) < 1e-5, (cam_only, b)
        if not cam_only:
            for q in NAMES:
                assert rel_err(d[q].grad, sgrads[q]) < 1e-5, q


def test_lens_feature_maps_follow_the_lens(gs, cuda):
    """Feature maps use the lensed frame's weights: with the colours as the first three feature channels, those channels
    equal the image (no background), and both differ from the frame without a lens."""
    import renderer
    g, v, cam = scene(3000, 128, 96, k=1)
    feat = torch.zeros(g["pos"].shape[0], 8)
    feat[:, :3] = torch.sigmoid(g["rgb"])
    out = []
    for lenses in ([_lens("fisheye", v.width, v.height)], None):
        rctx = _ctx(gs)
        _set(rctx, lenses)
        d = _dev(g, cuda)
        fd = feat.to(cuda).contiguous().requires_grad_(True)
        img, fm, depth, alpha, _ = renderer.render_frame_feat(rctx, *(d[q] for q in NAMES), fd, v.width, v.height,
                                                              v.fx, v.fy, v.rot, v.tran, v.near, 0.05, "abs",
                                                              final=True)
        (fm.sum() + img.sum()).backward()
        torch.cuda.synchronize()
        assert abs_err(fm[..., :3], img) < 1e-5
        assert bool(torch.isfinite(fd.grad).all()) and bool(torch.isfinite(d["pos"].grad).all())
        out.append(fm.detach())
    assert abs_err(out[0], out[1]) > 0.05


def test_lens_densify_stats_batch_matches_single_views(gs, cuda):
    """The batched densification statistics through per-view lenses equal those of the single-view frames."""
    import splatter
    g, v, cam = scene(2000, 128, 96, k=1)
    vds = []
    for k, nm in zip((0, 1), ("opencv", "fisheye")):
        vi = scene(1, 128, 96, k=k)[1]
        vds.append(dict(width=vi.width, height=vi.height, focal_x=vi.fx, focal_y=vi.fy, rot=vi.rot, tran=vi.tran,
                        lens=_lens(nm, vi.width, vi.height)))
    sp1 = splatter.Splatter.from_tensors(g, vds, device=cuda, densify_stats="grad")
    for i in range(2):
        sp1(i).sum().backward()
    sp2 = splatter.Splatter.from_tensors(g, vds, device=cuda, densify_stats="grad")
    sp2.render_batch([0, 1])["image"].sum().backward()
    torch.cuda.synchronize()
    a, b = sp1.densify_stats, sp2.densify_stats
    assert torch.equal(a.count, b.count) and torch.equal(a.max_radius, b.max_radius)
    assert int((a.count == 2).sum()) > 100
    assert rel_err(b.grad2d, a.grad2d) < 1e-5


def test_lens_gradient_push_refused_before_any_launch(gs, cuda):
    """A backward of a lens frame with a gradient push configured is refused (GS_ERR_UNSUPPORTED) and launches nothing."""
    g, v, cam = scene(500, 64, 64, k=0)
    rctx = _ctx(gs)
    _set(rctx, [_lens("opencv", 64, 64)])
    d = _dev(g, cuda)
    img, _ = _render_final(gs, rctx, d, cam, v)
    per = 4096                                                  # 2 ranks x 4096 floats hold the 500 Gaussians' rows
    bucket = torch.zeros(2 * per, device=cuda)
    staging = [torch.zeros(2 * per, device=cuda) for _ in range(2)]
    push = (bucket.data_ptr(), [t.data_ptr() for t in staging], per, 0)
    lib = ctypes.CDLL(os.path.join(os.path.dirname(gs[0].__file__), "libgs_b200.so"))
    lib.gs_kernel_launches.restype = ctypes.c_ulonglong
    renderer = gs[1]
    renderer.set_flat_grad_allocator(lambda numel, dev: (bucket[:numel], push))
    try:
        torch.cuda.synchronize()
        before = lib.gs_kernel_launches()
        with pytest.raises(RuntimeError, match="gradient push"):
            img.sum().backward()
        assert lib.gs_kernel_launches() == before
    finally:
        renderer.set_flat_grad_allocator(None)


def _f3_views(w, h, k_views):
    import synthetic as S
    out = []
    for k in range(k_views):
        v = S.make_view(w, h, k % 8)
        tran = (np.asarray(v.tran, dtype=np.float64) * (0.6 + 0.1 * k)).astype(np.float32)
        out.append(S.View(w, h, v.fx, v.fy, v.rot, torch.from_numpy(tran), v.near))
    return out


def test_lens_filter3d_compute_vs_oracle(gs, cuda):
    """gs_filter3d_compute through per-view lenses (PINHOLE off-centre, OPENCV with a fold-back limit, FISHEYE) against
    the fp64 oracle: within 2 ulp, the same seen set, and different from the filter without lenses."""
    import synthetic as S
    n = 50_000
    pos = S.make_gaussians(n, 640, 360, seed=1)["pos"] * 1.6
    pos[: n // 50] += torch.tensor([0.0, 1000.0, 0.0])         # some Gaussians no view sees
    views = _f3_views(640, 360, 6)
    names = ["pinhole-offset", "opencv-fold", "fisheye", "opencv", "fisheye", "pinhole-offset"]
    lenses = [_lens(nm, 640, 360) for nm in names]
    cams = [dict(width=v.width, height=v.height, focal_x=v.fx, focal_y=v.fy, rot=np.asarray(v.rot),
                 tran=np.asarray(v.tran), near=0.3) for v in views]
    tie = L.sampling_ties_lens(pos.numpy(), cams, lenses)
    assert int(tie.sum()) < n // 100
    pos = pos[torch.from_numpy(~tie)].contiguous()
    ref, seen = L.sampling_filter_lens(pos.numpy(), cams, lenses)
    assert seen.any() and not seen.all()
    size = torch.tensor([[v.width, v.height] for v in views])
    focal = torch.tensor([[v.fx, v.fy] for v in views], dtype=torch.float32)
    rot = torch.stack([torch.as_tensor(v.rot, dtype=torch.float32) for v in views])
    tran = torch.stack([torch.as_tensor(v.tran, dtype=torch.float32) for v in views])
    rctx = gs[0].RenderContext()
    _set(rctx, lenses)
    pd = pos.to(cuda)
    got = gs[0].filter3d_compute(rctx, pd, size, focal, rot, tran, 0.3, 0.15, 0.2).cpu()
    spacing = torch.from_numpy(np.spacing(np.abs(np.float32(ref)))).double()
    ulp = float(((got.double() - torch.from_numpy(ref)).abs() / spacing.clamp_min(1e-45)).max())
    assert ulp <= 2.0, ulp
    assert bool((got[torch.from_numpy(~seen)] == got.max()).all())
    _set(rctx, None)
    plain = gs[0].filter3d_compute(rctx, pd, size, focal, rot, tran, 0.3, 0.15, 0.2).cpu()
    assert not torch.equal(plain, got)
    # a lens count other than 1 or n_cams is refused
    _set(rctx, lenses[:2])
    with pytest.raises(RuntimeError):
        gs[0].filter3d_compute(rctx, pd, size, focal, rot, tran, 0.3, 0.15, 0.2)
