"""2D Gaussian surfels on the GPU (gs_render_forward_surfel / gs_render_backward_surfel through
renderer.render_frame_surfel) against the fp64 oracle tests/surfel_oracle.py: image and maps <= 1e-4 abs (depth-like
maps relative to their scale), each gradient <= 1e-3 max|ref| (a gradient that is exactly zero: the fp32 noise floor).  Also bit-determinism, the
3DGS frame after a surfel frame, and the refusals that need a real context."""
import pytest
import torch

import helpers as H
import surfel_oracle as SO

pytestmark = pytest.mark.gpu

MAPS = ("alpha", "depth", "median", "distortion", "normal")
KEYS = ("pos", "rgb", "opa", "quat", "scale")
BG = [0.2, 0.5, 0.1]


def _mods():
    import gaussian
    import renderer
    return gaussian, renderer


def _scene(n=400, w=80, h=64, seed=0, sh=0, extra=True):
    g, _, cam = H.scene(n, w, h, seed=seed, sh_dim=3 * sh if sh else 3)
    g = {k: v.clone() for k, v in g.items()}
    if extra:
        gen = torch.Generator().manual_seed(seed + 100)
        R, t = cam.rot.float(), cam.tran.float()

        def add(pc, quat, s, opa):
            m = len(pc)
            pos = (torch.tensor(pc, dtype=torch.float32) - t) @ R          # p = R^T (p_c - t)
            g["pos"] = torch.cat([g["pos"], pos])
            g["quat"] = torch.cat([g["quat"], torch.tensor(quat, dtype=torch.float32)])
            g["scale"] = torch.cat([g["scale"], torch.tensor([[a, b, 0.0] for a, b in s], dtype=torch.float32)])
            g["opa"] = torch.cat([g["opa"], torch.tensor(opa, dtype=torch.float32)])
            g["rgb"] = torch.cat([g["rgb"], torch.randn(m, g["rgb"].shape[1], generator=gen)])

        z0 = float((g["pos"] @ R.T + t)[:, 2].median())
        # edge-on surfels (normal perpendicular to the view ray: h2 -> 0 across the disk)
        add([[0.1 * z0, 0.05 * z0, z0], [-0.1 * z0, 0.1 * z0, z0]], [[0.7071, 0.7071, 0.0, 0.0], [0.7071, 0.0, 0.7071, 0.0]],
            [(0.05 * z0, 0.05 * z0)] * 2, [1.0, 1.0])
        # sub-pixel surfels: the low-pass branch wins
        add([[0.02 * z0 * k, -0.03 * z0, z0 * 0.9] for k in range(-3, 4)], [[1.0, 0.1, 0.2, 0.0]] * 7,
            [(1e-4 * z0, 1e-4 * z0)] * 7, [3.0] * 7)
        # crossing the near plane: the disk reaches the camera plane (no instances)
        add([[0.0, 0.0, cam.near * 1.5]], [[0.7071, 0.7071, 0.0, 0.0]], [(5.0, 5.0)], [2.0])
        # at the 0.99 clamp, and nearly transparent (alpha < 1/255 over most of the disk)
        add([[-0.15 * z0, -0.1 * z0, 0.8 * z0], [0.15 * z0, -0.12 * z0, 0.8 * z0]], [[1.0, 0.0, 0.0, 0.0]] * 2,
            [(0.04 * z0, 0.03 * z0)] * 2, [8.0, -6.0])
        # a saturated tile: a stack of opaque surfels in front of everything
        add([[0.2 * z0, 0.2 * z0, 0.5 * z0 + 0.01 * k] for k in range(12)], [[1.0, 0.0, 0.0, 0.0]] * 12,
            [(0.03 * z0, 0.03 * z0)] * 12, [6.0] * 12)
    return SO.without_branch_ties(g, cam), cam


def _device(g, dev):
    return {k: v.to(dev).contiguous().requires_grad_(True) for k, v in g.items()}


def _run(g, cam, sh=0, background=None, final=True, maps=True, weights=None, rctx=None, act="abs"):
    """GPU frame + backward of sum_k <weights[k], output k>; -> (image, maps, grads, rctx)"""
    gaussian, renderer = _mods()
    dev = torch.device("cuda", 0)
    rctx = rctx or gaussian.RenderContext()
    if sh:
        rctx.set_sh_eval(gaussian.SH_EVAL_GAUSSIAN)
    p = _device(g, dev)
    img, mp, _ = renderer.render_frame_surfel(rctx, p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], cam.width,
                                              cam.height, cam.fx, cam.fy, cam.rot, cam.tran, cam.near, 0.05, act,
                                              background, final, maps)
    loss = 0
    for k, w in (weights or {}).items():
        out = img if k == "image" else mp[k]
        loss = loss + (out * w.to(dev)).sum()
    if weights:
        loss.backward()
    torch.cuda.synchronize()
    grads = {k: p[k].grad.detach().cpu().double() if p[k].grad is not None else None for k in KEYS}
    return img.detach().cpu().double(), {k: v.detach().cpu().double() for k, v in mp.items()}, grads, rctx


def _oracle(g, cam, background=None, final=True, weights=None, act="abs"):
    p = {k: v.double().clone().requires_grad_(True) for k, v in g.items()}
    img, mp, info = SO.render(p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], cam, background=background,
                              scale_activation=act)
    if final:
        img = cam.crop(img.clamp(0, 1))
        mp = {k: cam.crop(v[..., None] if v.dim() == 2 else v) for k, v in mp.items()}
        mp = {k: (v[..., 0] if k != "normal" else v) for k, v in mp.items()}
    loss = 0
    for k, w in (weights or {}).items():
        out = img if k == "image" else mp[k]
        loss = loss + (out * w.double()).sum()
    if weights:
        loss.backward()
    grads = {k: p[k].grad for k in KEYS}
    return img.detach(), {k: v.detach() for k, v in mp.items()}, grads, info


def _weights(shape, which, seed=0):
    gen = torch.Generator().manual_seed(seed)
    w = {}
    for k in which:
        s = tuple(shape) + ((3,) if k in ("image", "normal") else ())
        w[k] = torch.randn(s, generator=gen) * (1.0 if k in ("image", "alpha", "normal") else 0.2)
    return w


def _check(gpu, ref, maps=True):
    img, mp, grads = gpu
    rimg, rmp, rgrads = ref
    assert H.abs_err(img, rimg) <= 1e-4
    if maps:
        for k in MAPS:
            scale = max(1.0, float(rmp[k].abs().max())) if k in ("depth", "median") else 1.0
            assert H.abs_err(mp[k], rmp[k]) <= 1e-4 * scale, k
    # each gradient <= 1e-3 max|ref|.  Only a parameter whose exact gradient is zero (the median depth does not move
    # when a disk is stretched in its own plane: the fp64 reference is rounding noise, 1e-16 of the frame's largest
    # gradient) is held instead to the fp32 noise floor of the frame's largest gradient
    top = max(float(rgrads[k].abs().max()) for k in KEYS if rgrads[k] is not None)
    for k in KEYS:
        if rgrads[k] is None:
            continue
        ref = float(rgrads[k].abs().max())
        bound = 1e-3 * ref if ref > 1e-12 * top else 1e-6 * top
        assert H.abs_err(grads[k], rgrads[k]) <= bound, (k, H.rel_err(grads[k], rgrads[k]))


@pytest.mark.parametrize("sh", [0, 16])
@pytest.mark.parametrize("background", [None, BG])
def test_frame_and_gradients_match_the_oracle(sh, background):
    g, cam = _scene(seed=1 + sh, sh=sh)
    w = _weights((cam.height, cam.width), ("image",) + MAPS, seed=3)
    img, mp, grads, _ = _run(g, cam, sh=sh, background=background, weights=w)
    rimg, rmp, rgrads, _ = _oracle(g, cam, background=background, weights=w)
    _check((img, mp, grads), (rimg, rmp, rgrads))
    assert float(grads["scale"][:, 2].abs().max()) == 0.0


@pytest.mark.parametrize("which", MAPS)
def test_each_map_gradient_alone(which):
    g, cam = _scene(seed=5)
    w = _weights((cam.height, cam.width), (which,), seed=4)
    gpu = _run(g, cam, background=BG, weights=w)[:3]
    ref = _oracle(g, cam, background=BG, weights=w)[:3]
    _check(gpu, ref)


def test_padded_outputs_and_gradient():
    g, cam = _scene(seed=6, w=72, h=56)                       # not a multiple of 16: padding and a crop
    w = _weights((cam.Hp, cam.Wp), ("image",) + MAPS, seed=5)
    gpu = _run(g, cam, background=BG, final=False, weights=w)[:3]
    ref = _oracle(g, cam, background=BG, final=False, weights=w)[:3]
    _check(gpu, ref)


def test_without_maps_matches_the_image_of_the_oracle():
    g, cam = _scene(seed=7)
    w = _weights((cam.height, cam.width), ("image",), seed=6)
    img, mp, grads, _ = _run(g, cam, maps=False, weights=w)
    assert mp == {}
    rimg, _, rgrads, _ = _oracle(g, cam, weights=w)
    _check((img, {}, grads), (rimg, {}, rgrads), maps=False)


def test_a_tile_longer_than_a_staging_chunk():
    # 300 overlapping faint surfels on one region: every tile there holds more than one forward (64) and backward (32)
    # chunk, and the stop is never reached
    g, cam = _scene(n=10, seed=8, extra=False)
    n = 300
    gen = torch.Generator().manual_seed(9)
    R, t = cam.rot.float(), cam.tran.float()
    pc = torch.stack([torch.randn(n, generator=gen) * 0.05, torch.randn(n, generator=gen) * 0.05,
                      3.0 + torch.rand(n, generator=gen)], -1)
    extra = dict(pos=(pc - t) @ R, quat=torch.randn(n, 4, generator=gen),
                 scale=torch.cat([torch.rand(n, 2, generator=gen) * 0.2 + 0.1, torch.zeros(n, 1)], -1),
                 opa=torch.full((n,), -3.5), rgb=torch.randn(n, 3, generator=gen))
    g = SO.without_branch_ties({k: torch.cat([g[k], extra[k]]) for k in KEYS}, cam)
    w = _weights((cam.height, cam.width), ("image",) + MAPS, seed=7)
    gpu = _run(g, cam, background=BG, weights=w)[:3]
    ref, info = _oracle(g, cam, background=BG, weights=w)[:3], None
    acc = SO.render(*[g[k].double() for k in KEYS], cam)[2]["accum"]
    assert int((acc[1:] - acc[:-1]).max()) > 64
    _check(gpu, ref)


def test_two_runs_are_bit_equal_and_a_3dgs_frame_after_is_unchanged():
    gaussian, renderer = _mods()
    g, cam = _scene(seed=10)
    w = _weights((cam.height, cam.width), ("image",) + MAPS, seed=8)
    a = _run(g, cam, background=BG, weights=w)
    b = _run(g, cam, background=BG, weights=w, rctx=a[3])
    assert torch.equal(a[0], b[0])
    for k in MAPS:
        assert torch.equal(a[1][k], b[1][k])
    for k in KEYS:
        assert torch.equal(a[2][k], b[2][k])
    dev = torch.device("cuda", 0)

    def frame(rctx):
        p = _device(g, dev)
        img, _ = renderer.render_frame_final(rctx, p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], cam.width,
                                             cam.height, cam.fx, cam.fy, cam.rot, cam.tran, cam.near, 0.05, "abs")
        img.backward(torch.ones_like(img))
        torch.cuda.synchronize()
        return img.detach().cpu(), [p[k].grad.cpu() for k in KEYS]

    used, fresh = frame(a[3]), frame(gaussian.RenderContext())
    assert torch.equal(used[0], fresh[0])
    for x, y in zip(used[1], fresh[1]):
        assert torch.equal(x, y)


def test_refusals_that_need_a_context():
    gaussian, renderer = _mods()
    dev = torch.device("cuda", 0)
    g, cam = _scene(n=50, seed=11, extra=False)
    p = {k: v.to(dev).contiguous() for k, v in g.items()}
    args = (cam.width, cam.height, cam.fx, cam.fy, cam.rot, cam.tran, cam.near, 0.05, 0)
    grads = [torch.zeros_like(p[k]) for k in KEYS]
    rctx = gaussian.RenderContext()
    fin, raw, m, mf, mask = rctx.forward_surfel(*[p[k] for k in KEYS], *args, None, True, True)
    with pytest.raises(RuntimeError, match="surfels"):       # a 3DGS backward after a surfel forward
        rctx.backward_final_into(*[p[k] for k in KEYS], raw, torch.zeros_like(fin), *grads, -1)
    fin, raw, mask = rctx.forward_final(*[p[k] for k in KEYS], *args)
    with pytest.raises(RuntimeError, match="did not render surfels"):
        rctx.backward_surfel_into(*[p[k] for k in KEYS], raw, torch.zeros_like(fin), True, None, *grads, -1)
    fin, raw, m, mf, mask = rctx.forward_surfel(*[p[k] for k in KEYS], *args, None, False, True)
    with pytest.raises(RuntimeError, match="wrote no maps"):
        rctx.backward_surfel_into(*[p[k] for k in KEYS], raw, torch.zeros_like(fin), True,
                                  torch.zeros(cam.height, cam.width, 8, device=dev), *grads, -1)
    sh = {k: v.to(dev).contiguous() for k, v in _scene(n=50, seed=12, sh=16, extra=False)[0].items()}
    with pytest.raises(RuntimeError, match="per pixel"):
        rctx.forward_surfel(*[sh[k] for k in KEYS], *args, None, True, True)
    rctx.set_filter2d(gaussian.FILTER2D_ANTIALIAS, 0.3)
    with pytest.raises(RuntimeError, match="filters"):
        rctx.forward_surfel(*[p[k] for k in KEYS], *args, None, True, True)
    rctx.set_filter2d(gaussian.FILTER2D_NONE, 0.3)
    with pytest.raises(RuntimeError, match="dist_near"):
        rctx.forward_surfel(*[p[k] for k in KEYS], *args, None, True, True, 1.0, 0.5)


def test_frame_stats_and_visible_report_the_surfel_frame():
    gaussian, renderer = _mods()
    g, cam = _scene(seed=13)
    _, _, _, rctx = _run(g, cam)
    info = SO.render(*[g[k].double() for k in KEYS], cam)[2]
    assert rctx.last_instances() == int(info["accum"][-1])
    mask = torch.zeros(g["pos"].shape[0], dtype=torch.uint8, device="cuda")
    rctx.visible_into(mask, False)
    tx0, tx1, ty0, ty1 = info["rects"]
    assert torch.equal(mask.cpu().bool(), ((tx1 - tx0) * (ty1 - ty0)) > 0)


def test_every_context_refusal():
    """Forward: a lens, the 3-D filter, densification statistics, a gradient push, the packed path.  Backward: a push
    or statistics set after the forward.  Every 3DGS backward after a surfel forward."""
    gaussian, renderer = _mods()
    dev = torch.device("cuda", 0)
    g, cam = _scene(n=50, seed=14, extra=False)
    n = g["pos"].shape[0]
    p = {k: v.to(dev).contiguous() for k, v in g.items()}
    P = [p[k] for k in KEYS]
    args = (cam.width, cam.height, cam.fx, cam.fy, cam.rot, cam.tran, cam.near, 0.05, 0)
    grads = [torch.zeros_like(p[k]) for k in KEYS]
    rctx = gaussian.RenderContext()

    def refused(match):
        with pytest.raises(RuntimeError, match=match):
            rctx.forward_surfel(*P, *args, None, True, True)

    lens = torch.tensor([[cam.width / 2, cam.height / 2, 0.1, 0.0, 0.0, 0.0]])
    rctx.set_lens([1], lens)                                      # OPENCV, k1 = 0.1
    refused("lenses")
    rctx.set_lens(None, None)
    rctx.set_filter3d(torch.zeros(n, device=dev))
    refused("filters")
    rctx.set_filter3d(None)
    stats = (torch.zeros(n, device=dev), torch.zeros(n, dtype=torch.int32, device=dev), torch.zeros(n, device=dev))
    rctx.set_densify_stats(*stats, None)
    refused("densification")
    rctx.clear_densify_stats()
    bucket = torch.zeros(64, device=dev)
    staging = [torch.zeros(64, device=dev) for _ in range(2)]
    rctx.set_grad_push(bucket.data_ptr(), [s.data_ptr() for s in staging], 32, 0)
    refused("gradient push")
    rctx.clear_grad_push()
    gaussian.tune("gather", 0)
    try:
        refused("packed path")
    finally:
        gaussian.tune("gather", 1)

    fin, raw, m, mf, mask = rctx.forward_surfel(*P, *args, None, True, True)
    gi = torch.zeros_like(fin)
    rctx.set_grad_push(bucket.data_ptr(), [s.data_ptr() for s in staging], 32, 0)
    with pytest.raises(RuntimeError, match="gradient push"):
        rctx.backward_surfel_into(*P, raw, gi, True, None, *grads, -1)
    rctx.clear_grad_push()
    rctx.set_densify_stats(*stats, None)
    with pytest.raises(RuntimeError, match="densification"):
        rctx.backward_surfel_into(*P, raw, gi, True, None, *grads, -1)
    rctx.clear_densify_stats()

    aux = torch.zeros(cam.Hp, cam.Wp, 2, device=dev)
    with pytest.raises(RuntimeError, match="surfels"):
        rctx.backward_into(*P, raw, torch.zeros_like(raw), *grads, -1)
    with pytest.raises(RuntimeError, match="surfels"):
        rctx.backward_aux_into(*P, raw, gi, True, aux, None, *grads, -1)
    with pytest.raises(RuntimeError, match="surfels"):
        rctx.backward_cam_into(*P, raw, gi, True, None, None, *grads, torch.zeros(12, device=dev), -1)
    feat = torch.zeros(n, 8, device=dev)
    fmap = torch.zeros(cam.Hp, cam.Wp, 8, device=dev)
    with pytest.raises(RuntimeError, match="surfels"):
        rctx.backward_feat_into(P[0], P[1], P[2], P[3], P[4], feat, raw, gi, True, aux, None, fmap, None, *grads,
                                torch.zeros_like(feat), -1)
    # a batched forward records the batch shape; a surfel forward after it makes every batched backward refuse
    focal = torch.tensor([[cam.fx, cam.fy]] * 2)
    rots, trans = torch.stack([cam.rot.float()] * 2), torch.stack([cam.tran.float()] * 2)
    out = rctx.forward_batch(*P, cam.width, cam.height, focal, rots, trans, cam.near, 0.05, 0, None, True)
    fin, raw, m, mf, mask = rctx.forward_surfel(*P, *args, None, True, True)
    braw, baux = torch.zeros_like(out[1]), torch.zeros_like(out[2])
    with pytest.raises(RuntimeError, match="surfels"):
        rctx.backward_batch_into(*P, braw, torch.zeros_like(out[0]), True, baux, None, *grads, -1)
    with pytest.raises(RuntimeError, match="surfels"):
        rctx.backward_batch_cam_into(*P, braw, torch.zeros_like(out[0]), True, baux, None, *grads,
                                     torch.zeros(2, 12, device=dev), -1)


def test_exp_scale_activation_matches_the_oracle():
    g, cam = _scene(seed=15)
    g["scale"] = torch.log(g["scale"].abs() + 1e-4)           # the same sizes as raw log-scales
    w = _weights((cam.height, cam.width), ("image",) + MAPS, seed=9)
    img, mp, grads, _ = _run(g, cam, background=BG, weights=w, act="exp")
    rimg, rmp, rgrads, _ = _oracle(g, cam, background=BG, weights=w, act="exp")
    _check((img, mp, grads), (rimg, rmp, rgrads))
