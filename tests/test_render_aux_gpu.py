"""Depth / alpha maps and background colour on the fused frame path (renderer.render_frame_aux,
gs_render_forward_aux / gs_render_backward_aux) against the fp64 oracle of tests/aux_oracle.py, plus the
properties that must hold when the maps are rendered but unused, edge cases and the full C3 size."""
import pytest
import torch

import aux_oracle as A
import synthetic as S
from helpers import abs_err, device_depth_keys, rel_err, scene

pytestmark = pytest.mark.gpu

IMG_ATOL = 1e-4
GRAD_RTOL = 1e-3
BG = (0.2, 0.5, 0.9)
NAMES = ("pos", "rgb", "opa", "quat", "scale")


def _args(v):
    return (v.width, v.height, v.fx, v.fy, v.rot, v.tran, v.near, 0.05, "abs")


def _upstream(shape, seed):
    gen = torch.Generator().manual_seed(seed)
    h, w = shape
    gi = (torch.rand(h, w, 3, generator=gen) * 2 - 1).double()
    gd = (torch.rand(h, w, generator=gen) * 2 - 1).double()
    ga = (torch.rand(h, w, generator=gen) * 2 - 1).double()
    return {"depth": (None, gd, None), "alpha": (None, None, ga), "all": (gi, gd, ga)}


def _check_vs_oracle(gs, cuda, g, v, cam, final, sh_tc=-1):
    sh = g["rgb"].shape[1] != 3
    p = {q: t.double().clone().requires_grad_(True) for q, t in g.items()}
    o = A.render_maps(p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], cam, background=BG, use_sh_coeff=sh,
                      depth_key=device_depth_keys(g, cam, cuda))
    oi, od, oa = (o["image"], o["depth"], o["alpha"]) if final else (o["padded_image"], o["padded_depth"],
                                                                      o["padded_alpha"])
    rctx = gs[0].RenderContext()
    gs[0].tune("sh_tc", sh_tc)
    try:
        _compare(rctx, g, v, final, oi, od, oa, p)
    finally:
        gs[0].tune("sh_tc", -1)


@pytest.mark.parametrize("final", [True, False], ids=["final", "padded"])
@pytest.mark.parametrize("n,w,h,k,opa", [
    (2000, 128, 96, 0, (0.005, 0.05)),
    (10000, 256, 256, 0, (0.05, 0.9)),
    (8000, 200, 120, 2, (0.05, 0.9)),
    (5000, 96, 64, 0, (0.6, 0.98)),
])
def test_aux_frame_vs_oracle(gs, cuda, n, w, h, k, opa, final):
    g, v, cam = scene(n, w, h, k=k, opa_range=opa)
    _check_vs_oracle(gs, cuda, g, v, cam, final)


@pytest.mark.parametrize("final", [True, False], ids=["final", "padded"])
@pytest.mark.parametrize("sh_dim,sh_tc", [(27, 0), (27, 3), (48, 3)], ids=["sh27-scalar", "sh27-tc", "sh48-tc"])
def test_aux_frame_sh_vs_oracle(gs, cuda, sh_dim, sh_tc, final):
    """Per-pixel SH colour: the scalar kernels (blend_sh.cu, the default at D = 27) and the one-pixel-per-thread
    tensor-core kernels (blend_sh_tc.cu, the default at D = 48)."""
    g, v, cam = scene(2500, 112, 80, k=1, sh_dim=sh_dim, opa_range=(0.05, 0.9))
    _check_vs_oracle(gs, cuda, g, v, cam, final, sh_tc)


def _compare(rctx, g, v, final, oi, od, oa, p):
    import renderer
    cuda = torch.device("cuda", 0)
    for case, (gi, gd, ga) in _upstream(od.shape, 5).items():
        d = {q: t.to(cuda).clone().requires_grad_(True) for q, t in g.items()}
        img, dep, alp, _ = renderer.render_frame_aux(rctx, d["pos"], d["rgb"], d["opa"], d["quat"], d["scale"],
                                                     *_args(v), background=BG, final=final)
        assert abs_err(img, oi) < IMG_ATOL
        assert abs_err(alp, oa) < 1e-4
        assert abs_err(dep, od) < 1e-4 * float(od.abs().max())
        outs = [(t, u) for t, u in ((oi, gi), (od, gd), (oa, ga)) if u is not None]
        ref = torch.autograd.grad([t for t, _ in outs], [p[q] for q in NAMES], [u for _, u in outs],
                                  retain_graph=True, allow_unused=True)
        douts = [t for t, u in zip((img, dep, alp), (gi, gd, ga)) if u is not None]
        torch.autograd.backward(douts, [u.float().to(cuda) for u in (gi, gd, ga) if u is not None])
        for q, r in zip(NAMES, ref):
            r = torch.zeros_like(p[q]) if r is None else r
            assert rel_err(d[q].grad, r) < GRAD_RTOL, (case, q)


def test_aux_unused_matches_plain_frame(gs, cuda):
    import renderer
    g, v, cam = scene(10000, 256, 256, opa_range=(0.05, 0.9))
    go = S.make_grad_output(256, 256, 0).to(cuda) * (256 * 256)
    rctx = gs[0].RenderContext()
    grads = {}
    for mode in ("plain", "aux-no-grad", "aux-zero-grad"):
        d = {q: t.to(cuda).clone().requires_grad_(True) for q, t in g.items()}
        if mode == "plain":
            img, _ = renderer.render_frame_final(rctx, d["pos"], d["rgb"], d["opa"], d["quat"], d["scale"], *_args(v))
            img.backward(go)
            plain = img.detach()
        else:
            img, dep, alp, _ = renderer.render_frame_aux(rctx, d["pos"], d["rgb"], d["opa"], d["quat"], d["scale"],
                                                         *_args(v))
            assert torch.equal(img.detach(), plain)
            if mode == "aux-no-grad":
                img.backward(go)
            else:
                torch.autograd.backward([img, dep, alp], [go, torch.zeros_like(dep), torch.zeros_like(alp)])
        grads[mode] = {q: d[q].grad.clone() for q in NAMES}
    for mode in ("aux-no-grad", "aux-zero-grad"):
        for q in NAMES:
            assert rel_err(grads[mode][q], grads["plain"][q]) < 1e-6, (mode, q)


@pytest.mark.parametrize("what", ["empty", "culled"])
def test_aux_empty_frame_is_background(gs, cuda, what):
    import renderer
    g, v, cam = scene(0 if what == "empty" else 500, 80, 48)
    if what == "culled":
        g["pos"][:, 2] = -10.0                       # behind the camera
    d = {q: t.to(cuda).clone().requires_grad_(True) for q, t in g.items()}
    rctx = gs[0].RenderContext()
    for final in (True, False):
        img, dep, alp, mask = renderer.render_frame_aux(rctx, d["pos"], d["rgb"], d["opa"], d["quat"], d["scale"],
                                                        *_args(v), background=BG, final=final)
        assert int(mask.sum()) == 0
        assert torch.equal(img, torch.tensor(BG, device=cuda).expand_as(img))
        assert torch.equal(dep, torch.zeros_like(dep)) and torch.equal(alp, torch.zeros_like(alp))
        if what == "culled":                         # (an empty parameter set has no gradient buffers to write)
            (img.sum() + dep.sum() + alp.sum()).backward()
            for q in NAMES:
                assert torch.equal(d[q].grad, torch.zeros_like(d[q].grad)), q
            d = {q: t.detach().clone().requires_grad_(True) for q, t in d.items()}


def test_aux_unsupported_paths_raise(gs, cuda):
    import renderer
    g, v, cam = scene(2000, 96, 64)
    g27, _, _ = scene(2000, 96, 64, sh_dim=27)
    rctx = gs[0].RenderContext()

    def run(gg, **kw):
        d = {q: t.to(cuda) for q, t in gg.items()}
        return renderer.render_frame_aux(rctx, d["pos"], d["rgb"], d["opa"], d["quat"], d["scale"], *_args(v), **kw)

    gs[0].tune("sh_tc", 7)                         # two-pixel tensor-core backward: no aux variant
    try:
        with pytest.raises(RuntimeError, match="aux kernel"):
            run(g27)
    finally:
        gs[0].tune("sh_tc", -1)
    for knob, value in (("gather", 0), ("fwd_px", 8), ("fwd_ch", 64), ("bwd_minb", 16), ("bwd_ch", 64)):
        gs[0].tune(knob, value)
        try:
            with pytest.raises(RuntimeError, match="aux kernel"):
                run(g)
        finally:
            gs[0].tune(knob, {"gather": 1, "fwd_px": 4, "fwd_ch": 128, "bwd_minb": 10, "bwd_ch": 32}[knob])
    with pytest.raises(RuntimeError, match="finite"):
        run(g, background=(0.0, float("nan"), 0.0))
    # the plain path still works, and so does the aux path
    d = {q: t.to(cuda).clone().requires_grad_(True) for q, t in g.items()}
    img, _ = renderer.render_frame_final(rctx, d["pos"], d["rgb"], d["opa"], d["quat"], d["scale"], *_args(v))
    img.sum().backward()
    assert torch.isfinite(d["pos"].grad).all()
    img, dep, alp, _ = run(g, background=BG)
    assert float(alp.max()) > 0


def test_aux_full_size_deterministic(gs, cuda):
    """C3 (2.4 M Gaussians, 1080p): aux forward + backward are bit-deterministic, 0 <= alpha <= 1, and the frame
    launches as many of our kernels as the plain frame."""
    import renderer
    n, w, h = 2_400_000, 1920, 1080
    g = {q: t.to(cuda) for q, t in S.make_gaussians(n, w, h, 0).items()}
    v = S.make_view(w, h, 0)
    gen = torch.Generator().manual_seed(3)
    go = (torch.rand(h, w, 3, generator=gen) * 2 - 1).to(cuda)
    gd = (torch.rand(h, w, generator=gen) * 2 - 1).to(cuda) * 1e-2
    ga = (torch.rand(h, w, generator=gen) * 2 - 1).to(cuda)
    rctx = gs[0].RenderContext()
    d = {q: t.clone().requires_grad_(True) for q, t in g.items()}
    img, _ = renderer.render_frame_final(rctx, d["pos"], d["rgb"], d["opa"], d["quat"], d["scale"], *_args(v))
    img.backward(go)                               # the first frame of a context also fills its index table
    runs, launches = [], []
    for _ in range(2):
        d = {q: t.clone().requires_grad_(True) for q, t in g.items()}
        l0 = gs[0].kernel_launches()
        img, dep, alp, _ = renderer.render_frame_aux(rctx, d["pos"], d["rgb"], d["opa"], d["quat"], d["scale"],
                                                     *_args(v), background=BG)
        torch.autograd.backward([img, dep, alp], [go, gd, ga])
        torch.cuda.synchronize()
        launches.append(gs[0].kernel_launches() - l0)
        runs.append([img.detach(), dep.detach(), alp.detach()] + [d[q].grad for q in NAMES])
    for a, b in zip(*runs):
        assert torch.equal(a, b)
    alp = runs[0][2]
    assert float(alp.min()) >= 0.0 and float(alp.max()) <= 1.0
    d = {q: t.clone().requires_grad_(True) for q, t in g.items()}
    l0 = gs[0].kernel_launches()
    img, _ = renderer.render_frame_final(rctx, d["pos"], d["rgb"], d["opa"], d["quat"], d["scale"], *_args(v))
    img.backward(go)
    torch.cuda.synchronize()
    assert launches[0] == launches[1] == gs[0].kernel_launches() - l0
