"""Per-view camera pose gradients of a batched frame (renderer.render_frame_batch_cam, gs_render_backward_batch_cam,
Splatter.render_batch_at_poses): a one-view batch equals render_frame_cam bit for bit; with several views each view's
camera gradient matches a single-view camera backward of that view, the parameter gradients and densification
statistics are the plain batched backward's, camera only writes the same bits; the fp64 oracle, identical views,
determinism, the launch count, B = 64, the C3 size, the refusals, and a mini-batch pose refinement run end to end."""
import math

import pytest
import torch

import aux_oracle as A
import gs_oracle as O
import sh_gaussian_oracle as G
import synthetic as S
from helpers import abs_err, device_depth_keys, rel_err, scene

pytestmark = pytest.mark.gpu

NAMES = ("pos", "rgb", "opa", "quat", "scale")
BG = (0.2, 0.5, 0.9)
GRAD_RTOL = 1e-3


def _view(w, h, k=0, focal=1.0, tran=None):
    v = S.make_view(w, h, k)
    return dict(fx=v.fx * focal, fy=v.fy * focal * (1.1 if focal != 1.0 else 1.0), rot=v.rot,
                tran=v.tran if tran is None else torch.tensor(tran), near=v.near)


def _hetero_views(w, h):
    """four poses and focal lengths: a plain one, a zoomed orbit view, one looking away from the scene (no instances),
    one shifted so that part of the scene is culled"""
    return [_view(w, h, 0), _view(w, h, 1, focal=1.3), _view(w, h, 0, tran=(0.0, 0.0, -4.0)),
            _view(w, h, 2, focal=0.8, tran=(1.6, 0.4, 4.0))]


def _ctx(gs, sh_dim, filt="none"):
    gaussian, renderer = gs
    rctx = gaussian.RenderContext()
    if sh_dim != 3:
        rctx.set_sh_eval(renderer.SH_EVAL["gaussian"])
    rctx.set_filter2d(renderer.FILTER2D[filt], 0.3)
    return rctx


def _shape(w, h, final):
    return (h, w) if final else (int(math.ceil(h / 16)) * 16, int(math.ceil(w / 16)) * 16)


def _upstream(b, rows, cols, seed):
    gen = torch.Generator().manual_seed(seed)
    return ((torch.rand(b, rows, cols, 3, generator=gen) * 2 - 1), (torch.rand(b, rows, cols, generator=gen) * 2 - 1),
            (torch.rand(b, rows, cols, generator=gen) * 2 - 1))


def _forward_batch(rctx, d, w, h, views, final):
    focal = torch.tensor([[vw["fx"], vw["fy"]] for vw in views], dtype=torch.float64)
    rot = torch.stack([vw["rot"] for vw in views])
    tran = torch.stack([vw["tran"] for vw in views])
    return rctx.forward_batch(*(d[q] for q in NAMES), w, h, focal, rot, tran, views[0]["near"], 0.05, 0, list(BG),
                              final)


def _nan_grads(d):
    return [torch.full_like(d[q], float("nan")) for q in NAMES]


def _batch_cam_frame(gs, rctx, g, w, h, views, final, up, cuda, maps, params_grad=True):
    """render_frame_batch_cam with rot / tran as leaves: (outputs, parameter leaves, rot, tran)"""
    _, renderer = gs
    d = {q: t.to(cuda).clone().requires_grad_(params_grad) for q, t in g.items()}
    rot = torch.stack([vw["rot"] for vw in views]).to(cuda).requires_grad_(True)
    tran = torch.stack([vw["tran"] for vw in views]).to(cuda).requires_grad_(True)
    img, dep, alp, mask = renderer.render_frame_batch_cam(
        rctx, *(d[q] for q in NAMES), w, h, [vw["fx"] for vw in views], [vw["fy"] for vw in views], rot, tran,
        views[0]["near"], 0.05, "abs", background=BG, final=final)
    ys = [img, dep, alp] if maps else [img]
    torch.autograd.backward(ys, [u.to(cuda) for u in up][:len(ys)])
    return (img, dep, alp, mask), d, rot, tran


CONFIGS = [(sh, filt, final, maps) for sh in (3, 48) for filt in ("none", "antialias") for final in (True, False)
           for maps in (False, True)]
CONFIG_IDS = [f"{'rgb' if sh == 3 else 'sh48'}-{filt}-{'final' if final else 'padded'}-{'maps' if maps else 'image'}"
              for sh, filt, final, maps in CONFIGS]


@pytest.mark.parametrize("sh_dim,filt,final,maps", CONFIGS, ids=CONFIG_IDS)
def test_one_view_equals_render_frame_cam_bitwise(gs, cuda, sh_dim, filt, final, maps):
    _, renderer = gs
    w, h = 200, 120
    g, _, _ = scene(6000, w, h, k=0, sh_dim=sh_dim)
    vw = _view(w, h, 1, focal=1.2)
    up = _upstream(1, *_shape(w, h, final), 3)
    rctx = _ctx(gs, sh_dim, filt)
    (img_b, _, _, _), db, rot_b, tran_b = _batch_cam_frame(gs, rctx, g, w, h, [vw], final, up, cuda, maps)
    d = {q: t.to(cuda).clone().requires_grad_(True) for q, t in g.items()}
    rot, tran = vw["rot"].to(cuda).requires_grad_(True), vw["tran"].to(cuda).requires_grad_(True)
    img, dep, alp, _ = renderer.render_frame_cam(rctx, *(d[q] for q in NAMES), w, h, vw["fx"], vw["fy"], rot, tran,
                                                 vw["near"], 0.05, "abs", background=BG, final=final)
    ys = [img, dep, alp] if maps else [img]
    torch.autograd.backward(ys, [u[0].to(cuda) for u in up][:len(ys)])
    assert torch.equal(img_b[0], img)
    assert float(rot.grad.abs().max()) > 0
    assert torch.equal(rot_b.grad[0], rot.grad) and torch.equal(tran_b.grad[0], tran.grad)
    for q in NAMES:
        assert torch.equal(db[q].grad, d[q].grad), q


@pytest.mark.parametrize("sh_dim,filt,final,maps", CONFIGS, ids=CONFIG_IDS)
def test_views_match_single_view_camera_backwards(gs, cuda, sh_dim, filt, final, maps):
    """Several views with different poses and focal lengths, one of which sees nothing: each view's camera gradient
    against backward_cam_into after a single-view forward of that view (1e-5 of the view's max), the parameter
    gradients against backward_batch_into bit for bit, camera only against the full call bit for bit."""
    w, h = 184, 120
    g, _, _ = scene(8000, w, h, k=0, sh_dim=sh_dim)
    views = _hetero_views(w, h)
    b = len(views)
    rctx = _ctx(gs, sh_dim, filt)
    d = {q: t.to(cuda).contiguous() for q, t in g.items()}
    fin, raw, aux, aux_fin, mask = _forward_batch(rctx, d, w, h, views, final)
    frame = rctx.frame_id()
    assert int(mask[2].sum()) == 0 and all(int(mask[v].sum()) > 0 for v in (0, 1, 3))
    gi, gd, ga_ = _upstream(b, *_shape(w, h, final), 7)
    gi = gi.to(cuda)
    ga = torch.stack([gd, ga_], -1).to(cuda) if maps else None
    plain, full = _nan_grads(d), _nan_grads(d)
    cams_full = torch.full((b, 12), float("nan"), device=cuda)
    cams_only = torch.full((b, 12), float("nan"), device=cuda)
    rctx.backward_batch_into(*(d[q] for q in NAMES), raw, gi, final, aux, ga, *plain, frame)
    rctx.backward_batch_cam_into(*(d[q] for q in NAMES), raw, gi, final, aux, ga, *full, cams_full, frame)
    rctx.backward_batch_cam_into(*(d[q] for q in NAMES), raw, gi, final, aux, ga, None, None, None, None, None,
                                 cams_only, frame)
    torch.cuda.synchronize()
    for q, a, c in zip(NAMES, plain, full):
        assert torch.equal(a, c), q
    assert torch.equal(cams_full, cams_only)
    assert torch.equal(cams_full[2], torch.zeros(12, device=cuda))
    single = _ctx(gs, sh_dim, filt)
    for v, vw in enumerate(views):
        sf, sraw, saux, _, _ = single.forward_aux(*(d[q] for q in NAMES), w, h, vw["fx"], vw["fy"], vw["rot"],
                                                  vw["tran"], vw["near"], 0.05, 0, list(BG), final)
        assert torch.equal(sraw, raw[v])
        cam = torch.full((12,), float("nan"), device=cuda)
        single.backward_cam_into(*(d[q] for q in NAMES), sraw, gi[v], final, saux, None if ga is None else ga[v],
                                 None, None, None, None, None, cam, single.frame_id())
        torch.cuda.synchronize()
        if v == 2:
            assert torch.equal(cam, torch.zeros_like(cam))
            continue
        scale = float(cam.abs().max())
        assert scale > 0, v
        assert float((cams_full[v] - cam).abs().max()) <= 1e-5 * scale, (v, cams_full[v], cam)


@pytest.mark.parametrize("sh_dim", [3, 48])
def test_views_vs_oracle(gs, cuda, sh_dim):
    """Every view's dL/drot and dL/dtran against the fp64 oracle with rot / tran as autograd leaves, under image, depth
    and alpha upstream gradients over a non-black background: 1e-3 of max|ref| per view and tensor."""
    w, h = 128, 96
    g, _, _ = scene(3000, w, h, k=0, sh_dim=sh_dim)
    views = [_view(w, h, 0), _view(w, h, 1, focal=1.25), _view(w, h, 7, focal=0.9)]
    up = _upstream(len(views), h, w, 11)
    rctx = _ctx(gs, sh_dim)
    (img, _, _, _), _, rot, tran = _batch_cam_frame(gs, rctx, g, w, h, views, True, up, cuda, True, params_grad=False)
    p = {q: t.double() for q, t in g.items()}
    for v, vw in enumerate(views):
        r, t = vw["rot"].double().clone().requires_grad_(True), vw["tran"].double().clone().requires_grad_(True)
        ocam = O.Camera(w, h, vw["fx"], vw["fy"], r, t, vw["near"])
        kcam = O.Camera(w, h, vw["fx"], vw["fy"], vw["rot"], vw["tran"], vw["near"])
        o = (G if sh_dim != 3 else A).render_maps(*(p[q] for q in NAMES), ocam, background=BG,
                                                  depth_key=device_depth_keys(g, kcam, cuda))
        assert abs_err(img[v], o["image"]) < 1e-4, v
        ref = torch.autograd.grad([o["image"], o["depth"], o["alpha"]], [r, t],
                                  [up[0][v].double(), up[1][v].double(), up[2][v].double()])
        assert float(ref[0].abs().max()) > 0, v
        assert rel_err(rot.grad[v], ref[0]) < GRAD_RTOL, (v, "rot", rel_err(rot.grad[v], ref[0]))
        assert rel_err(tran.grad[v], ref[1]) < GRAD_RTOL, (v, "tran", rel_err(tran.grad[v], ref[1]))


@pytest.mark.parametrize("sh_dim", [3, 48])
def test_identical_views_give_identical_rows(gs, cuda, sh_dim):
    w, h = 160, 96
    g, _, _ = scene(5000, w, h, k=0, sh_dim=sh_dim)
    b = 5
    views = [_view(w, h, 1, focal=1.1)] * b
    one = _upstream(1, h, w, 4)
    up = tuple(u.expand(b, *u.shape[1:]).contiguous() for u in one)
    rctx = _ctx(gs, sh_dim)
    _, _, rot, tran = _batch_cam_frame(gs, rctx, g, w, h, views, True, up, cuda, True)
    assert float(rot.grad.abs().max()) > 0
    for v in range(1, b):
        assert torch.equal(rot.grad[v], rot.grad[0]) and torch.equal(tran.grad[v], tran.grad[0]), v


def test_determinism_launch_count_and_64_views(gs, cuda):
    """Two backwards are bit-identical; the launch count is render_frame_batch's + 1 for B = 2, 8 and 64; a 64-view
    batch at a small size gives finite gradients that agree with its first view's single-view camera gradient."""
    gaussian, renderer = gs
    w, h = 96, 64
    g, _, _ = scene(3000, w, h, k=0)
    rctx = _ctx(gs, 3)

    def run(views, cam, up=None):
        up = _upstream(len(views), h, w, 1) if up is None else up
        d = {q: t.to(cuda).clone().requires_grad_(True) for q, t in g.items()}
        rot = torch.stack([vw["rot"] for vw in views]).to(cuda).requires_grad_(cam)
        tran = torch.stack([vw["tran"] for vw in views]).to(cuda).requires_grad_(cam)
        fn = renderer.render_frame_batch_cam if cam else renderer.render_frame_batch
        torch.cuda.synchronize()
        k0 = gaussian.kernel_launches()
        img, dep, alp, _ = fn(rctx, *(d[q] for q in NAMES), w, h, [vw["fx"] for vw in views],
                              [vw["fy"] for vw in views], rot, tran, views[0]["near"], 0.05, "abs", background=BG)
        torch.autograd.backward([img, dep, alp], [u.to(cuda) for u in up])
        torch.cuda.synchronize()
        return gaussian.kernel_launches() - k0, rot.grad, tran.grad, [d[q].grad for q in NAMES]

    for b in (2, 8, 64):
        views = [_view(w, h, k % 8, focal=1.0 + 0.01 * k) for k in range(b)]
        run(views, True)                                   # warm-up: workspaces and the depth sort's index table
        run(views, False)
        l_plain = run(views, False)[0]
        l1, r1, t1, p1 = run(views, True)
        l2, r2, t2, p2 = run(views, True)
        assert l1 == l2 == l_plain + 1, (b, l1, l2, l_plain)
        assert torch.equal(r1, r2) and torch.equal(t1, t2)
        for a, c in zip(p1, p2):
            assert torch.equal(a, c)
        assert bool(torch.isfinite(r1).all()) and bool(torch.isfinite(t1).all())
        if b == 64:
            assert float(r1[0].abs().max()) > 0 and float(r1[63].abs().max()) > 0
            _, rs, ts, _ = run(views[:1], True, tuple(u[:1] for u in _upstream(b, h, w, 1)))
            for got, want in ((r1[0], rs[0]), (t1[0], ts[0])):
                assert float((got - want).abs().max()) <= 1e-5 * float(want.abs().max())


def test_c3_eight_views_finite(gs, cuda):
    """The C3 scene (2.4 M Gaussians), 8 views at 480x270: finite camera and parameter gradients."""
    _, renderer = gs
    n, w, h = 2_400_000, 480, 270
    g = {q: t.to(cuda) for q, t in S.make_gaussians(n, w, h, 0).items()}
    views = [_view(w, h, k % 8, focal=1.0 + 0.02 * k) for k in range(8)]
    up = _upstream(8, h, w, 2)
    rctx = _ctx(gs, 3)
    (img, _, _, _), d, rot, tran = _batch_cam_frame(gs, rctx, g, w, h, views, True, up, cuda, True)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(rot.grad).all()) and bool(torch.isfinite(tran.grad).all())
    assert all(float(rot.grad[v].abs().max()) > 0 for v in range(8))
    for q in NAMES:
        assert bool(torch.isfinite(d[q].grad).all()), q


def test_densify_stats_with_parameters_and_untouched_camera_only(gs, cuda):
    w, h = 184, 120
    n = 8000
    g, _, _ = scene(n, w, h, k=0)
    views = _hetero_views(w, h)
    b = len(views)
    rctx = _ctx(gs, 3)
    st = [torch.zeros(n, device=cuda), torch.zeros(n, dtype=torch.int32, device=cuda), torch.zeros(n, device=cuda)]
    rctx.set_densify_stats(*st, None)
    d = {q: t.to(cuda).contiguous() for q, t in g.items()}
    fin, raw, aux, _, _ = _forward_batch(rctx, d, w, h, views, True)
    frame = rctx.frame_id()
    gi = _upstream(b, h, w, 5)[0].to(cuda)
    cams = torch.empty(b, 12, device=cuda)
    rctx.backward_batch_into(*(d[q] for q in NAMES), raw, gi, True, aux, None, *_nan_grads(d), frame)
    torch.cuda.synchronize()
    want = [t.clone() for t in st]
    assert int(want[1].max()) >= 2
    for t in st:
        t.zero_()
    rctx.backward_batch_cam_into(*(d[q] for q in NAMES), raw, gi, True, aux, None, *_nan_grads(d), cams, frame)
    torch.cuda.synchronize()
    for a, c in zip(st, want):
        assert torch.equal(a, c)
    for t in st:
        t.zero_()
    rctx.backward_batch_cam_into(*(d[q] for q in NAMES), raw, gi, True, aux, None, None, None, None, None, None, cams,
                                 frame)
    torch.cuda.synchronize()
    for t in st:
        assert not bool(t.any())


def _expect_refused(gaussian, fn, exc, text):
    torch.cuda.synchronize()
    k0 = gaussian.kernel_launches()
    with pytest.raises(exc, match=text):
        fn()
    assert gaussian.kernel_launches() == k0


def test_refusals_leave_the_context_usable(gs, cuda):
    gaussian, renderer = gs
    w, h = 96, 64
    g, _, _ = scene(2000, w, h, k=0)
    g27, _, _ = scene(2000, w, h, k=0, sh_dim=27)
    views = [_view(w, h, 0), _view(w, h, 1)]
    rctx = gaussian.RenderContext()
    d = {q: t.to(cuda) for q, t in g.items()}
    rot = torch.stack([vw["rot"] for vw in views]).to(cuda)
    tran = torch.stack([vw["tran"] for vw in views]).to(cuda)
    fx, fy = [vw["fx"] for vw in views], [vw["fy"] for vw in views]

    def frame(params=d, r=rot, t=tran, f=(fx, fy)):
        return renderer.render_frame_batch_cam(rctx, *(params[q] for q in NAMES), w, h, *f, r, t, 0.3, 0.05, "abs",
                                               background=BG)

    def usable():
        p = {q: t.clone().requires_grad_(True) for q, t in d.items()}
        r, t = rot.clone().requires_grad_(True), tran.clone().requires_grad_(True)
        img, _, _, _ = frame(p, r, t)
        img.sum().backward()
        torch.cuda.synchronize()
        assert bool(torch.isfinite(r.grad).all()) and float(r.grad.abs().max()) > 0

    # per-pixel SH colour: the batched forward refuses it
    d27 = {q: t.to(cuda) for q, t in g27.items()}
    _expect_refused(gaussian, lambda: frame(d27), RuntimeError, "per pixel")
    usable()
    # a data-parallel gradient push
    world = 2

    def alloc(numel, device):
        per = (numel + world * 4 - 1) // (world * 4) * 4
        flat = torch.zeros(world * per, device=device)
        staging = [torch.zeros(world * per, device=device) for _ in range(world)]
        alloc.keep = staging
        return flat, (flat.data_ptr(), [s.data_ptr() for s in staging], per, 0)

    renderer.set_flat_grad_allocator(alloc)
    try:
        p = {q: t.clone().requires_grad_(True) for q, t in d.items()}
        img, _, _, _ = frame(p, rot.clone().requires_grad_(True), tran)
        _expect_refused(gaussian, lambda: img.sum().backward(), RuntimeError, "push")
    finally:
        renderer.set_flat_grad_allocator(None)
        rctx.clear_grad_push()
    usable()
    # wrong shape, dtype or device of rot / tran, and more than 64 views
    for r, t in ((rot.cpu(), tran), (rot, tran.cpu()), (rot.double(), tran), (rot, tran.double()), (rot[0], tran),
                 (rot, tran[:1]), (rot.reshape(2, 9), tran), (rot, tran[:, :2]), (rot.tolist(), tran),
                 (rot[:, :2], tran)):
        _expect_refused(gaussian, lambda: frame(r=r, t=t), ValueError, "render_frame_batch_cam")
    big = 65
    _expect_refused(gaussian, lambda: frame(r=rot[:1].repeat(big, 1, 1), t=tran[:1].repeat(big, 1),
                                            f=([fx[0]] * big, [fy[0]] * big)), ValueError, "1 .. 64")
    usable()
    # single-view and batched calls mixed
    fin, raw, aux, _, _ = _forward_batch(rctx, d, w, h, views, True)
    outs = [torch.empty_like(d[q]) for q in NAMES]
    _expect_refused(gaussian, lambda: rctx.backward_cam_into(*(d[q] for q in NAMES), raw[0], torch.zeros_like(fin[0]),
                                                             True, aux[0], None, *outs, torch.zeros(12, device=cuda),
                                                             -1), RuntimeError, r"\(-1\).*batched")
    sfin, sraw, saux, _, _ = rctx.forward_aux(*(d[q] for q in NAMES), w, h, fx[0], fy[0], views[0]["rot"],
                                              views[0]["tran"], 0.3, 0.05, 0, list(BG), True)
    _expect_refused(gaussian, lambda: rctx.backward_batch_cam_into(*(d[q] for q in NAMES), raw, torch.zeros_like(fin),
                                                                   True, aux, None, *outs,
                                                                   torch.zeros(2, 12, device=cuda), -1),
                    RuntimeError, r"\(-1\).*not batched")
    usable()


def _skew(x):
    """[..., 3] -> [..., 3, 3] cross-product matrices"""
    z = torch.zeros_like(x[..., 0])
    return torch.stack([torch.stack([z, -x[..., 2], x[..., 1]], -1), torch.stack([x[..., 2], z, -x[..., 0]], -1),
                        torch.stack([-x[..., 1], x[..., 0], z], -1)], -2)


def test_mini_batch_pose_refinement_end_to_end(gs, cuda):
    """A frozen synthetic scene seen from 4 views whose poses are off by 3 degrees and ~3 % of the camera distance;
    a learnable se(3) correction per view (R = exp([w]x) R_p, t = exp([w]x) t_p + rho) trained through
    Splatter.render_batch_at_poses with Adam on the L1 image loss (camera-only backward) brings every view's rotation
    and translation errors down to a quarter of their initial values within 150 steps."""
    import splatter
    torch.manual_seed(0)
    w, h = 96, 64
    base = [S.make_view(w, h, k) for k in (0, 1, 7, 0)]
    g = S.make_gaussians(800, w, h, 1, opa_range=(0.3, 0.9), sigma_px=(1.5, 6.0))
    views = [dict(width=w, height=h, focal_x=v.fx, focal_y=v.fy, rot=v.rot, tran=v.tran) for v in base]
    sp = splatter.Splatter.from_tensors(g, views, device=cuda)
    for prm in sp.gaussian_3ds.parameters():
        prm.requires_grad_(False)                 # the scene is frozen: camera-only backward
    ids = [0, 1, 2, 3]
    R0 = torch.stack([v.rot for v in base]).to(cuda)
    t0 = torch.stack([v.tran for v in base]).to(cuda)
    with torch.no_grad():
        target = sp.render_batch_at_poses(R0, t0, ids)["image"].clone()
    axes = torch.tensor([[0.3, 1.0, -0.5], [1.0, -0.2, 0.4], [-0.6, 0.3, 1.0], [0.2, 0.8, 0.9]], device=cuda)
    axes = axes / axes.norm(dim=1, keepdim=True)
    Rp = torch.linalg.matrix_exp(_skew(axes * math.radians(3.0))) @ R0
    tp = t0 + torch.tensor([[0.06, -0.05, 0.1], [-0.08, 0.06, 0.06], [0.05, 0.09, -0.06], [-0.07, -0.07, 0.07]],
                           device=cuda)
    xi = torch.zeros(4, 6, device=cuda, requires_grad=True)
    opt = torch.optim.Adam([xi], lr=5e-3)

    def errors(R, t):
        c = ((R @ R0.transpose(1, 2)).diagonal(dim1=1, dim2=2).sum(-1) - 1) / 2
        return torch.acos(c.clamp(-1, 1)).cpu(), (t - t0).norm(dim=1).cpu()

    e0 = errors(Rp, tp)
    assert float(e0[0].min()) > math.radians(2.5) and float(e0[1].min()) > 0.09
    for _ in range(150):
        dR = torch.linalg.matrix_exp(_skew(xi[:, :3]))
        R, t = dR @ Rp, (dR @ tp.unsqueeze(-1)).squeeze(-1) + xi[:, 3:]
        out = sp.render_batch_at_poses(R, t, ids)
        loss = (out["image"] - target).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
    assert out["image"].shape == (4, h, w, 3) and out["culling_mask"].shape == (4, 800)
    assert sp.n_tile_gaussians > 0 and torch.equal(sp.culling_mask, out["culling_mask"].sum(0))
    e1 = errors(R.detach(), t.detach())
    assert bool((e1[0] <= e0[0] / 4).all()) and bool((e1[1] <= e0[1] / 4).all()), (e0, e1)
