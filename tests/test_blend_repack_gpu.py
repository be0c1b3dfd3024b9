"""Live-pixel repack of the shipped RGB backward blend (gs_tune("blend_repack", 1), the default) against the same
kernel without it (blend_repack = 0).  The repack only moves live pixels to other lanes, so the image is bit-identical,
every parameter gradient agrees within 1e-4 of its largest magnitude (the cross-pixel sums are added in another
order), and the repacked result is bit-deterministic.  Parity with the fp64 oracle is gated by the existing oracle
tests, which run the default."""
import pytest
import torch

import synthetic as S
from helpers import scene

pytestmark = pytest.mark.gpu

NAMES = ("pos", "rgb", "opa", "quat", "scale")
BOUND = 1e-4
BG = (0.2, 0.5, 0.9)


def _args(v):
    return (v.width, v.height, v.fx, v.fy, v.rot, v.tran, v.near, 0.05, "abs")


def _frame(gs, g, v, repack, mode, ups):
    """One forward + backward with the knob set; mode: "final" / "padded" (plain kernels), "aux-final" /
    "aux-padded" (aux kernels); ups: upstream gradients (image[, depth, alpha])."""
    import renderer
    gs[0].tune("blend_repack", repack)
    try:
        rctx = gs[0].RenderContext()
        d = {q: t.clone().requires_grad_(True) for q, t in g.items()}
        if mode == "final":
            outs = [renderer.render_frame_final(rctx, *(d[q] for q in NAMES), *_args(v))[0]]
        elif mode == "padded":
            outs = [renderer.render_frame(rctx, *(d[q] for q in NAMES), *_args(v))[0]]
        else:
            outs = list(renderer.render_frame_aux(rctx, *(d[q] for q in NAMES), *_args(v), background=BG,
                                                  final=mode == "aux-final")[:3])
        used = [(o, u) for o, u in zip(outs, ups) if u is not None]
        torch.autograd.backward([o for o, _ in used], [u for _, u in used])
        torch.cuda.synchronize()
        return [o.detach() for o in outs], {q: d[q].grad.clone() for q in NAMES}
    finally:
        gs[0].tune("blend_repack", 1)


def _upstream(mode, v, cam, cuda, what="image"):
    h, w = (v.height, v.width) if mode.endswith("final") else (cam.Hp, cam.Wp)
    gen = torch.Generator().manual_seed(7)
    gi = (torch.rand(h, w, 3, generator=gen) * 2 - 1).to(cuda)
    gd = (torch.rand(h, w, generator=gen) * 2 - 1).to(cuda) * 1e-2
    ga = (torch.rand(h, w, generator=gen) * 2 - 1).to(cuda)
    return {"image": (gi,), "depth": (None, gd, None), "alpha": (None, None, ga), "all": (gi, gd, ga)}[what]


def _check(gs, g, v, mode, ups):
    outs0, grads0 = _frame(gs, g, v, 0, mode, ups)
    outs1, grads1 = _frame(gs, g, v, 1, mode, ups)
    outs2, grads2 = _frame(gs, g, v, 1, mode, ups)
    for a, b, c in zip(outs0, outs1, outs2):
        assert torch.equal(a, b) and torch.equal(b, c)           # the forward is untouched by the knob
    for q in NAMES:
        assert torch.equal(grads1[q], grads2[q]), q               # repacked backward is bit-deterministic
        assert bool(torch.isfinite(grads1[q]).all()), q
        ref = float(grads0[q].abs().max())
        assert float((grads1[q] - grads0[q]).abs().max()) <= BOUND * ref, (q, ref)


SCENES = {
    "small": (10000, 256, 256, 0, (0.05, 0.9)),
    "border": (8000, 200, 120, 2, (0.05, 0.9)),        # rotated view, size not a multiple of 16: border tiles
    "opaque": (20000, 256, 192, 0, (0.5, 0.99)),       # pixels saturate early and at different instances
    # deep, nearly opaque tiles: the live count of most tiles falls below 32 long before their list ends, which
    # takes the slot count down to 1
    "deep-opaque": (120000, 256, 192, 0, (0.9, 0.99)),
}


@pytest.mark.parametrize("mode", ["final", "padded"])
@pytest.mark.parametrize("name", sorted(SCENES))
def test_repack_matches_unpacked(gs, cuda, name, mode):
    n, w, h, k, opa = SCENES[name]
    g, v, cam = scene(n, w, h, k=k, opa_range=opa)
    g = {q: t.to(cuda) for q, t in g.items()}
    _check(gs, g, v, mode, _upstream(mode, v, cam, cuda))


@pytest.mark.parametrize("mode", ["aux-final", "aux-padded"])
@pytest.mark.parametrize("what", ["depth", "alpha", "all"])
def test_repack_matches_unpacked_aux(gs, cuda, what, mode):
    n, w, h, k, opa = SCENES["opaque"]
    g, v, cam = scene(n, w, h, k=k, opa_range=opa)
    g = {q: t.to(cuda) for q, t in g.items()}
    _check(gs, g, v, mode, _upstream(mode, v, cam, cuda, what))


@pytest.mark.parametrize("n", [500_000, 2_400_000], ids=["C2", "C3"])
def test_repack_matches_unpacked_full_size(gs, cuda, n):
    w, h = 1920, 1080
    g = {q: t.to(cuda) for q, t in S.make_gaussians(n, w, h, 0).items()}
    v = S.make_view(w, h, 0)
    go = (S.make_grad_output(h, w, 0) * (h * w)).to(cuda)
    _check(gs, g, v, "final", (go,))
