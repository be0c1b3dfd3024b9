"""Camera pose gradients on the fused frame path (renderer.render_frame_cam, gs_render_backward_cam,
Splatter.render_at_pose) against the fp64 oracle, which differentiates through rot / tran when they are leaves of
O.Camera; bit-level agreement with the aux backward, the camera-only mode, edge cases, the C3 size and a pose
refinement run end to end."""
import math

import pytest
import torch

import aux_oracle as A
import gs_oracle as O
import sh_gaussian_oracle as G
import synthetic as S
from helpers import abs_err, device_depth_keys, rel_err, scene

pytestmark = pytest.mark.gpu

IMG_ATOL = 1e-4
GRAD_RTOL = 1e-3
BG = (0.2, 0.5, 0.9)
NAMES = ("pos", "rgb", "opa", "quat", "scale")
# (colour width, n, w, h, view, opacity range): RGB scenes of the aux tests and the per-Gaussian SH scenes
SCENES = [(3, 2000, 128, 96, 0, (0.005, 0.05)), (3, 8000, 200, 120, 2, (0.05, 0.9)),
          (3, 5000, 96, 64, 0, (0.6, 0.98)), (27, 2500, 112, 80, 1, (0.05, 0.9)), (48, 2500, 112, 80, 1, (0.05, 0.9))]
SCENE_IDS = ["rgb-safe", "rgb-k2", "rgb-opaque", "sh27", "sh48"]


def _intr(v):
    return (v.width, v.height, v.fx, v.fy)


def _ctx(gs, sh):
    import renderer
    rctx = gs[0].RenderContext()
    rctx.set_sh_eval(renderer.SH_EVAL["gaussian" if sh else "pixel"])
    return rctx


def _frame(rctx, g, v, cuda, final, background=BG, params_grad=True, rot=None, tran=None):
    import renderer
    d = {q: t.to(cuda).clone().requires_grad_(params_grad) for q, t in g.items()}
    rot = (v.rot if rot is None else rot).to(cuda).clone().requires_grad_(True)
    tran = (v.tran if tran is None else tran).to(cuda).clone().requires_grad_(True)
    img, dep, alp, mask = renderer.render_frame_cam(rctx, *(d[q] for q in NAMES), *_intr(v), rot, tran, v.near, 0.05,
                                                    "abs", background=background, final=final)
    return (img, dep, alp, mask), d, rot, tran


def _upstreams(shape, seed=5):
    gen = torch.Generator().manual_seed(seed)
    h, w = shape
    return {"image": (torch.rand(h, w, 3, generator=gen, dtype=torch.float64) * 2 - 1, 0),
            "depth": (torch.rand(h, w, generator=gen, dtype=torch.float64) * 2 - 1, 1),
            "alpha": (torch.rand(h, w, generator=gen, dtype=torch.float64) * 2 - 1, 2)}


@pytest.mark.parametrize("final", [True, False], ids=["final", "padded"])
@pytest.mark.parametrize("sh_dim,n,w,h,k,opa", SCENES, ids=SCENE_IDS)
def test_cam_grad_vs_oracle(gs, cuda, sh_dim, n, w, h, k, opa, final):
    """dL/drot and dL/dtran (and the five parameter gradients) against the fp64 oracle under image-only, depth-only
    and alpha-only upstream gradients over a non-black background: 1e-3 of max|ref|, each tensor on its own."""
    sh = sh_dim != 3
    g, v, cam = scene(n, w, h, k=k, sh_dim=sh_dim, opa_range=opa)
    p = {q: t.double().clone().requires_grad_(True) for q, t in g.items()}
    rot, tran = v.rot.double().clone().requires_grad_(True), v.tran.double().clone().requires_grad_(True)
    ocam = O.Camera(w, h, v.fx, v.fy, rot, tran, v.near)
    o = (G if sh else A).render_maps(*(p[q] for q in NAMES), ocam, background=BG,
                                     depth_key=device_depth_keys(g, cam, cuda))
    outs = (o["image"], o["depth"], o["alpha"]) if final else (o["padded_image"], o["padded_depth"],
                                                               o["padded_alpha"])
    rctx = _ctx(gs, sh)
    for case, (up, which) in _upstreams(outs[1].shape).items():
        ref = torch.autograd.grad(outs[which], [p[q] for q in NAMES] + [rot, tran], up, retain_graph=True,
                                  allow_unused=True)
        (img, dep, alp, _), d, drot, dtran = _frame(rctx, g, v, cuda, final)
        assert abs_err(img, outs[0]) < IMG_ATOL
        (img, dep, alp)[which].backward(up.float().to(cuda))
        assert float(ref[5].abs().max()) > 0 and float(ref[6].abs().max()) > 0, case
        assert rel_err(drot.grad, ref[5]) < GRAD_RTOL, (case, "rot", rel_err(drot.grad, ref[5]))
        assert rel_err(dtran.grad, ref[6]) < GRAD_RTOL, (case, "tran", rel_err(dtran.grad, ref[6]))
        for q, r in zip(NAMES, ref):
            r = torch.zeros_like(p[q]) if r is None else r
            assert rel_err(d[q].grad, r) < GRAD_RTOL, (case, q)


def test_cam_grad_packed_path_vs_oracle(gs, cuda):
    """The packed path (gs_tune("gather", 0)), which renders no maps: RenderContext.forward_final, then
    backward_cam_into without aux, full and camera only."""
    g, v, cam = scene(8000, 200, 120, k=2, opa_range=(0.05, 0.9))
    p = {q: t.double().clone().requires_grad_(True) for q, t in g.items()}
    rot, tran = v.rot.double().clone().requires_grad_(True), v.tran.double().clone().requires_grad_(True)
    ocam = O.Camera(200, 120, v.fx, v.fy, rot, tran, v.near)
    oimg = O.render(*(p[q] for q in NAMES), ocam, depth_key=device_depth_keys(g, cam, cuda))
    up = _upstreams((120, 200))["image"][0]
    ref = torch.autograd.grad(oimg, [p[q] for q in NAMES] + [rot, tran], up)
    d = {q: t.to(cuda).contiguous() for q, t in g.items()}
    rctx = gs[0].RenderContext()
    gs[0].tune("gather", 0)
    try:
        fin, raw, _ = rctx.forward_final(*(d[q] for q in NAMES), *_intr(v), v.rot, v.tran, v.near, 0.05, 0)
        grads = [torch.empty_like(d[q]) for q in NAMES]
        cam_full, cam_only = torch.empty(12, device=cuda), torch.empty(12, device=cuda)
        gi = up.float().to(cuda)
        rctx.backward_cam_into(*(d[q] for q in NAMES), raw, gi, True, None, None, *grads, cam_full)
        rctx.backward_cam_into(*(d[q] for q in NAMES), raw, gi, True, None, None, None, None, None, None, None,
                               cam_only)
        torch.cuda.synchronize()
    finally:
        gs[0].tune("gather", 1)
    assert abs_err(fin, oimg) < IMG_ATOL
    assert rel_err(cam_full[:9].view(3, 3), ref[5]) < GRAD_RTOL
    assert rel_err(cam_full[9:], ref[6]) < GRAD_RTOL
    assert torch.equal(cam_full, cam_only)
    for q, got, r in zip(NAMES, grads, ref):
        assert rel_err(got, r) < GRAD_RTOL, q


@pytest.mark.parametrize("sh_dim", [3, 48])
@pytest.mark.parametrize("with_aux", [False, True], ids=["image", "image+maps"])
def test_params_match_aux_backward_and_camera_only(gs, cuda, sh_dim, with_aux):
    """For one forward: the parameter gradients of gs_render_backward_cam equal gs_render_backward_aux's bit for bit,
    and the camera-only call (five NULL gradients) writes the same grad_cam bits as the full call."""
    sh = sh_dim != 3
    g, v, _ = scene(8000, 200, 120, k=1, sh_dim=sh_dim, opa_range=(0.05, 0.9))
    rctx = _ctx(gs, sh)
    d = {q: t.to(cuda).contiguous() for q, t in g.items()}
    fin, raw, aux, aux_fin, _ = rctx.forward_aux(*(d[q] for q in NAMES), *_intr(v), v.rot, v.tran, v.near, 0.05, 0,
                                                 list(BG), True)
    frame = rctx.frame_id()
    gen = torch.Generator().manual_seed(9)
    gi = (torch.rand(fin.shape, generator=gen) * 2 - 1).to(cuda)
    ga = (torch.rand(aux_fin.shape, generator=gen) * 2 - 1).to(cuda) if with_aux else None

    def bufs():
        return [torch.full_like(d[q], float("nan")) for q in NAMES]

    plain = bufs()
    rctx.backward_aux_into(*(d[q] for q in NAMES), raw, gi, True, aux, ga, *plain, frame)
    full, cam_full, cam_only = bufs(), torch.full((12,), float("nan"), device=cuda), torch.full(
        (12,), float("nan"), device=cuda)
    rctx.backward_cam_into(*(d[q] for q in NAMES), raw, gi, True, aux, ga, *full, cam_full, frame)
    rctx.backward_cam_into(*(d[q] for q in NAMES), raw, gi, True, aux, ga, None, None, None, None, None, cam_only,
                           frame)
    torch.cuda.synchronize()
    for q, a, b in zip(NAMES, plain, full):
        assert torch.equal(a, b), q
    assert bool(torch.isfinite(cam_full).all()) and float(cam_full.abs().max()) > 0
    assert torch.equal(cam_full, cam_only)
    with pytest.raises(RuntimeError, match="all five parameter gradients or none"):
        rctx.backward_cam_into(*(d[q] for q in NAMES), raw, gi, True, aux, ga, full[0], None, None, None, None,
                               cam_only, frame)


@pytest.mark.parametrize("what", ["empty", "culled"])
def test_empty_frame_writes_zeros(gs, cuda, what):
    g, v, _ = scene(0 if what == "empty" else 500, 80, 48)
    if what == "culled":
        g["pos"][:, 2] = -10.0                       # behind the camera
    rctx = gs[0].RenderContext()
    for final in (True, False):
        # an empty parameter set has no gradient buffers to write: camera only there
        (img, dep, alp, mask), d, rot, tran = _frame(rctx, g, v, cuda, final, params_grad=what == "culled")
        assert int(mask.sum()) == 0
        (img.sum() + dep.sum() + alp.sum()).backward()
        assert torch.equal(rot.grad, torch.zeros_like(rot)) and torch.equal(tran.grad, torch.zeros_like(tran))
        if what == "culled":
            for q in NAMES:
                assert torch.equal(d[q].grad, torch.zeros_like(d[q].grad)), q


def test_unsupported_and_bad_inputs_are_refused(gs, cuda):
    import renderer
    g, v, _ = scene(2000, 96, 64, k=1)
    g27, _, _ = scene(2000, 96, 64, k=1, sh_dim=27)
    (img, _, _, _), _, _, _ = _frame(_ctx(gs, False), g27, v, cuda, True)       # per-pixel SH: no camera gradient
    with pytest.raises(RuntimeError, match="per pixel"):
        img.sum().backward()

    world = 2

    def alloc(numel, device):
        per = (numel + world * 4 - 1) // (world * 4) * 4
        flat = torch.zeros(world * per, device=device)
        staging = [torch.zeros(world * per, device=device) for _ in range(world)]
        alloc.keep = staging
        return flat, (flat.data_ptr(), [s.data_ptr() for s in staging], per, 0)

    renderer.set_flat_grad_allocator(alloc)
    try:
        (img, _, _, _), _, _, _ = _frame(gs[0].RenderContext(), g, v, cuda, True)
        with pytest.raises(RuntimeError, match="push"):
            img.sum().backward()
    finally:
        renderer.set_flat_grad_allocator(None)

    d = {q: t.to(cuda) for q, t in g.items()}
    rctx = gs[0].RenderContext()
    good_r, good_t = v.rot.to(cuda), v.tran.to(cuda)
    for rot, tran in ((v.rot, good_t), (good_r, v.tran), (good_r.double(), good_t), (good_r, good_t[:2]),
                      (good_r.reshape(9), good_t), (good_r.tolist(), good_t)):
        with pytest.raises(ValueError, match="render_frame_cam"):
            renderer.render_frame_cam(rctx, *(d[q] for q in NAMES), *_intr(v), rot, tran, v.near, 0.05, "abs")
    # the context still renders
    (img, _, alp, _), _, rot, _ = _frame(rctx, g, v, cuda, True)
    img.sum().backward()
    assert bool(torch.isfinite(rot.grad).all()) and float(alp.max()) > 0


def test_c3_deterministic_translation_identity_and_launches(gs, cuda):
    """C3 (2.4 M Gaussians, 1080p): two backwards give bit-identical camera gradients; dL/dt = R sum_i dL/dpos_i holds
    on our own outputs to 1e-5 of sum_i |dL/dpos_i|; the frame launches one kernel more than the aux frame."""
    import renderer
    n, w, h = 2_400_000, 1920, 1080
    g = {q: t.to(cuda) for q, t in S.make_gaussians(n, w, h, 0).items()}
    v = S.make_view(w, h, 1)
    gen = torch.Generator().manual_seed(3)
    go = (torch.rand(h, w, 3, generator=gen) * 2 - 1).to(cuda)
    gd = (torch.rand(h, w, generator=gen) * 2 - 1).to(cuda) * 1e-2
    rctx = gs[0].RenderContext()
    args = (*_intr(v),)

    def cam_frame():
        d = {q: t.clone().requires_grad_(True) for q, t in g.items()}
        rot, tran = v.rot.to(cuda).requires_grad_(True), v.tran.to(cuda).requires_grad_(True)
        l0 = gs[0].kernel_launches()
        img, dep, _, _ = renderer.render_frame_cam(rctx, *(d[q] for q in NAMES), *args, rot, tran, v.near, 0.05,
                                                   "abs", background=BG)
        torch.autograd.backward([img, dep], [go, gd])
        torch.cuda.synchronize()
        return rot.grad, tran.grad, d["pos"].grad, gs[0].kernel_launches() - l0

    cam_frame()                                    # the first frame of a context also fills its index table
    r1, t1, gp1, l1 = cam_frame()
    r2, t2, gp2, l2 = cam_frame()
    assert torch.equal(r1, r2) and torch.equal(t1, t2) and torch.equal(gp1, gp2)
    gpd = gp1.double()
    want = v.rot.double().to(cuda) @ gpd.sum(0)
    tol = 1e-5 * float(gpd.norm(dim=1).sum())
    assert float((t1.double() - want).abs().max()) <= tol, (t1, want, tol)
    assert float(t1.abs().max()) > tol

    d = {q: t.clone().requires_grad_(True) for q, t in g.items()}
    l0 = gs[0].kernel_launches()
    img, dep, _, _ = renderer.render_frame_aux(rctx, *(d[q] for q in NAMES), *args, v.rot, v.tran, v.near, 0.05,
                                               "abs", background=BG)
    torch.autograd.backward([img, dep], [go, gd])
    torch.cuda.synchronize()
    assert l1 == l2 == gs[0].kernel_launches() - l0 + 1


def _skew(x):
    z = torch.zeros((), dtype=x.dtype, device=x.device)
    return torch.stack([torch.stack([z, -x[2], x[1]]), torch.stack([x[2], z, -x[0]]),
                        torch.stack([-x[1], x[0], z])])


def test_pose_refinement_end_to_end(gs, cuda):
    """A frozen synthetic scene rendered at a known pose; Splatter.render_at_pose starts from a pose off by 3 degrees
    and ~3 % of the camera distance, parameterised as a learnable se(3) correction (R = exp([w]x) R_p,
    t = exp([w]x) t_p + rho), and Adam on the L1 image loss (camera-only backward) brings both errors down to a
    quarter of their initial values within 150 steps."""
    import splatter
    torch.manual_seed(0)
    w, h = 96, 64
    v = S.make_view(w, h, 0)
    g = S.make_gaussians(800, w, h, 1, opa_range=(0.3, 0.9), sigma_px=(1.5, 6.0))
    views = [dict(width=w, height=h, focal_x=v.fx, focal_y=v.fy, rot=v.rot, tran=v.tran)]
    sp = splatter.Splatter.from_tensors(g, views, device=cuda)
    for prm in sp.gaussian_3ds.parameters():
        prm.requires_grad_(False)                 # the scene is frozen: camera-only backward
    R0, t0 = v.rot.to(cuda), v.tran.to(cuda)
    with torch.no_grad():
        target = sp.render_at_pose(R0, t0, camera_id=0)["image"].clone()
    axis = torch.tensor([0.3, 1.0, -0.5], device=cuda)
    axis = axis / axis.norm()
    Rp = torch.linalg.matrix_exp(_skew(axis * math.radians(3.0))) @ R0
    tp = t0 + torch.tensor([0.06, -0.05, 0.1], device=cuda)
    xi = torch.zeros(6, device=cuda, requires_grad=True)
    opt = torch.optim.Adam([xi], lr=5e-3)

    def errors(R, t):
        c = ((R @ R0.T).trace() - 1) / 2
        return float(torch.acos(c.clamp(-1, 1))), float((t - t0).norm())

    e0 = errors(Rp, tp)
    for _ in range(150):
        dR = torch.linalg.matrix_exp(_skew(xi[:3]))
        R, t = dR @ Rp, dR @ tp + xi[3:]
        out = sp.render_at_pose(R, t)
        loss = (out["image"] - target).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
    assert sp.n_tile_gaussians > 0 and sp.culling_mask is not None
    e1 = errors(R.detach(), t.detach())
    assert e1[0] <= e0[0] / 4 and e1[1] <= e0[1] / 4, (e0, e1)
