"""The data-parallel gradient push and the peer all-reduce kernels (dp.SymmetricGradBucket's "push" and "p2p"
exchanges) on one GPU.

Every pointer these kernels take can be an ordinary allocation on one device, and the exchange has no device-side wait
(dp.py orders it with host barriers), so W ranks are emulated one after another in one process.  The buffers are laid
out as dp.SymmetricGradBucket lays them out - bucket length o from renderer._flat_grads, slices of
per = ceil(o / 4 / W) * 4 floats, one [W][per] staging buffer per owner - inside one arena with guard floats around
every buffer.  Each rank renders its own view through the real autograd path, `renderer.set_flat_grad_allocator`
handing it its bucket and push configuration.  Checked, bit for bit unless stated otherwise:

- routing: every gradient float of rank p lands exactly once, in bucket p if p owns it, else in staging[owner][p],
  with the value a plain (W = 0) backward of the same frame on a fresh context computes; no other float of any
  bucket, staging slot, pad or guard changes;
- gs_allreduce_push_finish_f32 and gs_allreduce_p2p_f32 leave every bucket holding the fp32 sum g0 + g1 + ... in rank
  order (the kernels' own order), including slices that are empty for the high ranks;
- a second step on the same buffers, with views that change which Gaussians are visible: no stale float survives;
- every world size x colour layout x depth gradient x 2-D filter, with rows straddling slice boundaries;
- the summed gradient against the fp64 oracle once per colour mode, the densification statistics, and the refusals of
  a bad push configuration before any launch."""
import ctypes
import os

import pytest
import torch

import filter_oracle as F
import gs_oracle as O
import sh_gaussian_oracle as G
import synthetic as S
from helpers import device_depth_keys, rel_err

pytestmark = pytest.mark.gpu

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "3d-gaussian-splatting_b200")
NAMES = ("pos", "rgb", "opa", "quat", "scale")
WIDTH, HEIGHT = 128, 80
BG = (0.2, 0.5, 0.9)
SENT = 0x7FC0BEEF        # a quiet NaN: a float nobody has written
GUARD = 0x7FC0F00D       # a quiet NaN around every buffer
NG = 8                   # guard floats on each side of a buffer (keeps every buffer 16-byte aligned)
# colour layouts: parameter width d and where SH colour is evaluated
LAYOUTS = {"rgb": (3, "pixel"), "sh27": (27, "pixel"), "sh48": (48, "pixel"), "gsh9": (27, "gaussian"),
           "gsh16": (48, "gaussian")}


def _view(k=0, focal=1.0, tran=None):
    v = S.make_view(WIDTH, HEIGHT, k)
    return dict(fx=v.fx * focal, fy=v.fy * focal, rot=v.rot, tran=v.tran if tran is None else torch.tensor(tran),
                near=v.near)


# rank r renders VIEWS[r] in a first step and VIEWS[(r + 2) % 8] in a second: view 2 looks away from the scene (every
# Gaussian has no instance), view 3 culls part of it
VIEWS = [_view(0), _view(1, focal=1.3), _view(0, tran=(0.0, 0.0, -4.0)), _view(2, focal=0.8, tran=(1.6, 0.4, 4.0)),
         _view(3), _view(5, focal=1.1), _view(6), _view(1, tran=(-1.2, 0.0, 4.0))]


def _upstream(v, dev):
    """gradients of view v's final image [H,W,3], depth and alpha [H,W]"""
    gen = torch.Generator().manual_seed(100 + v)
    return [(torch.rand(*s, generator=gen) * 2 - 1).to(dev) for s in ((HEIGHT, WIDTH, 3), (HEIGHT, WIDTH), (HEIGHT, WIDTH))]


def _layout(n, d):
    """[(start, row width)] of the five gradient segments and the bucket length o, as renderer._flat_grads lays them
    out (each segment padded to 4 floats)"""
    segs, o = [], 0
    for wd in (3, d, 1, 4, 3):
        segs.append((o, wd))
        o += (n * wd + 3) // 4 * 4
    return segs, o


def _pads(segs, n, o, dev):
    pad = torch.zeros(o, dtype=torch.bool, device=dev)
    for k, (s, wd) in enumerate(segs):
        end = segs[k + 1][0] if k + 1 < len(segs) else o
        pad[s + n * wd:end] = True
    return pad


def _straddled(segs, n, o, world, per):
    """row widths of which some row straddles a slice boundary (those rows take the element-wise store path)"""
    out = set()
    for b in range(per, min(world * per, o), per):
        for s, wd in segs:
            if wd > 1 and s < b < s + n * wd and (b - s) % wd:
                out.add(wd)
    return out


def _where(i, segs, n):
    for k in reversed(range(len(segs))):
        s, wd = segs[k]
        if i >= s:
            return f"{NAMES[k]}[{(i - s) // wd}][{(i - s) % wd}]" if i < s + n * wd else f"{NAMES[k]} pad"
    return "?"


class _Exchange:
    """The buffers of `world` emulated ranks in one arena: bucket r (o floats) and staging r ([world][per] floats), NG
    guard floats before and after each.  dest[p][i]: the arena index where rank p's gradient float i belongs."""

    def __init__(self, dev, n, d, world, per):
        self.segs, self.o = _layout(n, d)
        self.n, self.world, self.per, self.dev = n, world, per, dev
        o = self.o
        assert per % 4 == 0 and world * per >= o
        sizes = [o] * world + [world * per] * world
        offs, at = [], NG
        for s in sizes:
            offs.append(at)
            at += s + NG
        self.off_b, self.off_s = offs[:world], offs[world:]
        self.arena = torch.empty(at, dtype=torch.float32, device=dev)
        self.bits = self.arena.view(torch.int32)
        self.pad = _pads(self.segs, n, o, dev)
        i = torch.arange(o, device=dev)
        owner = i // per
        off_s = torch.tensor(self.off_s, device=dev)
        self.dest = [torch.where(owner == p, self.off_b[p] + i, off_s[owner] + p * per + (i - owner * per))
                     for p in range(world)]

    def sentinels(self):
        """guards GUARD, every bucket and staging float SENT, pads 0 (dp zeroes the staging buffers once; the backward
        zeroes the bucket pads and never pushes a pad)"""
        self.bits.fill_(GUARD)
        o, per = self.o, self.per
        pad_i = torch.nonzero(self.pad).squeeze(1)
        for r in range(self.world):
            self.bits[self.off_b[r]:self.off_b[r] + o] = SENT
            self.bits[self.off_b[r] + pad_i] = 0
            self.bits[self.off_s[r]:self.off_s[r] + self.world * per] = SENT
        for q in range(self.world):
            self.bits[self.dest[q][self.pad]] = 0
        return self

    def bucket(self, r):
        return self.arena[self.off_b[r]:self.off_b[r] + self.o]

    def staging_ptr(self, r):
        return self.arena[self.off_s[r]:].data_ptr()

    def push(self, r):
        return (self.bucket(r).data_ptr(), [self.staging_ptr(s) for s in range(self.world)], self.per, r)

    def allocator(self, r):
        def alloc(numel, device):
            assert numel == self.o and device == self.dev
            return self.bucket(r), self.push(r)
        return alloc


def _ctx(gs, sh_eval, filt):
    gaussian, renderer = gs
    rctx = gaussian.RenderContext()
    rctx.set_sh_eval(renderer.SH_EVAL[sh_eval])
    rctx.set_filter2d(renderer.FILTER2D[filt], 0.3)
    return rctx


def _render_backward(renderer, rctx, g, v, dt, alloc):
    """view v through render_frame_aux and its backward with `alloc` as the bucket allocator; dt: the depth and alpha
    maps get a gradient too (the projection backward's DT kernels)"""
    vw = VIEWS[v]
    p = {q: t.detach().requires_grad_(True) for q, t in g.items()}
    img, dep, alp, _ = renderer.render_frame_aux(rctx, p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], WIDTH,
                                                 HEIGHT, vw["fx"], vw["fy"], vw["rot"], vw["tran"], vw["near"], 0.05,
                                                 "abs", background=BG, final=True)
    up = _upstream(v, img.device)
    ys = [img, dep, alp] if dt else [img]
    renderer.set_flat_grad_allocator(alloc)
    try:
        torch.autograd.grad(ys, [p[q] for q in NAMES], up[:len(ys)])
    finally:
        renderer.set_flat_grad_allocator(None)


def _dense(gs, g, v, d, sh_eval, filt, dt, o):
    """the flat gradient bucket of a plain (W = 0) backward of view v on a fresh context"""
    flat = torch.full((o,), float("nan"), device=g["pos"].device)
    _render_backward(gs[1], _ctx(gs, sh_eval, filt), g, v, dt, lambda numel, device: flat)
    return flat


def _first_diff(a, b):
    ne = torch.nonzero(a != b)
    return int(ne.shape[0]), (int(ne[0]) if ne.shape[0] else -1)


def _step(gs, ex, ctxs, g, views, dt, dense, label):
    """one training step of the emulated ranks: each rank's backward (routing checked), then every owner's
    push-finish (the rank-order sum checked); returns the summed bucket"""
    gaussian, renderer = gs
    contribs = []
    for r, v in enumerate(views):
        before = ex.bits.clone()
        _render_backward(renderer, ctxs[r], g, v, dt, ex.allocator(r))
        dest = ex.dest[r]
        keep = torch.ones_like(ex.bits, dtype=torch.bool)
        keep[dest] = False
        cnt, i = _first_diff(ex.bits[keep], before[keep])
        assert cnt == 0, f"{label} rank {r}: {cnt} floats outside its destinations changed (first: arena {i})"
        got = ex.arena[dest]
        cnt, i = _first_diff(got.view(torch.int32), dense[v].view(torch.int32))
        assert cnt == 0, (f"{label} rank {r}: {cnt} gradient floats differ from the plain backward, first "
                          f"{_where(i, ex.segs, ex.n)}: {float(got[i])} != {float(dense[v][i])}")
        contribs.append(got)
    want = contribs[0].clone()
    for c in contribs[1:]:
        want = want + c
    before = ex.bits.clone()
    ptrs = [ex.bucket(r).data_ptr() for r in range(ex.world)]
    for s in range(ex.world):
        gaussian.allreduce_push_finish(ptrs, ex.staging_ptr(s), ex.o, ex.per, s, ex.world, ex.dev.index)
    expected = before
    for r in range(ex.world):
        expected[ex.off_b[r]:ex.off_b[r] + ex.o] = want.view(torch.int32)
    cnt, i = _first_diff(ex.bits, expected)
    assert cnt == 0, f"{label}: {cnt} floats differ from the rank-order sum after the push-finish (first: arena {i})"
    return want


def _scene(d, n, seed, dev):
    return {q: t.to(dev) for q, t in S.make_gaussians(n, WIDTH, HEIGHT, seed, d).items()}


@pytest.mark.parametrize("filt", ["none", "antialias"])
@pytest.mark.parametrize("dt", [False, True], ids=["image-grad", "depth-grad"])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_push_routing_and_finish(gs, cuda, layout, dt, filt):
    d, sh_eval = LAYOUTS[layout]
    li = list(LAYOUTS).index(layout)
    n = 1201 + (2 * li + 2 * dt + (filt != "none")) % 3          # n % 4 = 1, 2 or 3: padded segments
    g = _scene(d, n, li, cuda)
    segs, o = _layout(n, d)
    dense = {}
    straddled = set()
    # dp's slices at W = 2, 4, 8, and slices larger than needed: ranks 6 and 7 own nothing
    configs = [(w, (o // 4 + w - 1) // w * 4) for w in (2, 4, 8)] + [(8, ((o + 5) // 6 + 3) // 4 * 4)]
    assert 6 * configs[-1][1] >= o
    for world, per in configs:
        ex = _Exchange(cuda, n, d, world, per).sentinels()
        ctxs = [_ctx(gs, sh_eval, filt) for _ in range(world)]
        for step in range(2):                    # the second step reuses the buffers, as dp does: no re-zeroing
            views = [(r + 2 * step) % len(VIEWS) for r in range(world)]
            for v in views:
                if v not in dense:
                    dense[v] = _dense(gs, g, v, d, sh_eval, filt, dt, o)
            _step(gs, ex, ctxs, g, views, dt, dense, f"W={world} per={per} step {step}")
        straddled |= _straddled(segs, n, o, world, per)
    assert d in straddled, straddled             # colour rows crossing a slice boundary were exercised


def test_views_cover_culled_gaussians(gs, cuda):
    """the views the routing test renders: view 2 sees nothing, view 3 culls part of what view 0 sees"""
    gaussian, renderer = gs
    g = _scene(3, 1201, 0, cuda)
    masks = []
    for v in (0, 2, 3):
        vw = VIEWS[v]
        _, _, _, mask = renderer.render_frame_aux(_ctx(gs, "pixel", "none"), g["pos"], g["rgb"], g["opa"], g["quat"],
                                                  g["scale"], WIDTH, HEIGHT, vw["fx"], vw["fy"], vw["rot"], vw["tran"],
                                                  vw["near"], 0.05, "abs")
        masks.append(int(mask.sum()))
    assert masks[1] == 0 and 0 < masks[2] < masks[0], masks


def _exchange_arena(dev, world, n):
    offs = [NG + r * (n + NG) for r in range(world)]
    arena = torch.empty(NG + world * (n + NG), device=dev)
    arena.view(torch.int32).fill_(GUARD)
    return arena, offs


@pytest.mark.parametrize("kernel", ["p2p", "push_finish"])
@pytest.mark.parametrize("world", [2, 4, 8])
def test_exchange_kernels_sum_in_rank_order(gs, cuda, world, kernel):
    """gs_allreduce_p2p_f32 (each rank sums its slice of the W buckets) and gs_allreduce_push_finish_f32 (the owner
    sums its own bucket slice with the W-1 staged contributions) on W local buffers: afterwards every bucket holds the
    fp32 sum in rank order, bit for bit, and nothing else changed.  Lengths of 1 to 7 float4s leave the high ranks an
    empty slice; 2.4M float4s make every slice longer than one pass of the kernel's grid."""
    gaussian, _ = gs
    for n4 in (1, 2, 3, 4, 5, 7, 1001, 2_400_001):
        n = 4 * n4
        per = (n4 + world - 1) // world * 4
        gen = torch.Generator(device=cuda).manual_seed(n4 * world)
        vals = torch.randn(world, n, generator=gen, device=cuda)
        vals *= torch.pow(10.0, torch.randint(-4, 5, (world, n), generator=gen, device=cuda).float())
        want = vals[0].clone()
        for r in range(1, world):
            want = want + vals[r]
        if n4 > 1000 and world > 2:                    # the order matters at these values: the check can tell
            rev = vals[world - 1].clone()
            for r in reversed(range(world - 1)):
                rev = rev + vals[r]
            assert not torch.equal(rev, want)
        buckets, boffs = _exchange_arena(cuda, world, n)
        for r in range(world):
            buckets[boffs[r]:boffs[r] + n] = vals[r]
        ptrs = [buckets[o:].data_ptr() for o in boffs]
        if kernel == "p2p":
            before = buckets.view(torch.int32).clone()
            for r in range(world):
                gaussian.allreduce_p2p(ptrs, n, r, world, cuda.index)
        else:
            # owner s: its own slice in bucket s, rank p's part of it in staging[s][p]; its own slot is never read
            staging, soffs = _exchange_arena(cuda, world, world * per)
            for s in range(world):
                for p in range(world):
                    lo, hi = s * per, min((s + 1) * per, n)
                    if p != s and hi > lo:
                        staging[soffs[s] + p * per:soffs[s] + p * per + hi - lo] = vals[p, lo:hi]
                bucket_s = buckets[boffs[s]:boffs[s] + n]
                bucket_s[:s * per] = float("nan")       # only slice s of bucket s is rank s's own
                bucket_s[(s + 1) * per:] = float("nan")
            before = buckets.view(torch.int32).clone()
            sbefore = staging.view(torch.int32).clone()
            for s in range(world):
                gaussian.allreduce_push_finish(ptrs, staging[soffs[s]:].data_ptr(), n, per, s, world, cuda.index)
            assert torch.equal(staging.view(torch.int32), sbefore)
        for r in range(world):
            before[boffs[r]:boffs[r] + n] = want.view(torch.int32)
        cnt, i = _first_diff(buckets.view(torch.int32), before)
        assert cnt == 0, f"n = {n}: {cnt} floats differ from the rank-order sum (first: arena {i})"


TIE_VIEWS = [0, 1, 3, 4]


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_push_sum_vs_fp64_oracle(gs, cuda, layout):
    """W = 4: the exchanged bucket against the sum over the four views of the fp64 oracle's gradients (image, depth
    and alpha upstream, as test_batch_gpu.py::test_batch_vs_oracle)"""
    d, sh_eval = LAYOUTS[layout]
    n, world = 801, 4
    gc = S.make_gaussians(n, WIDTH, HEIGHT, 11, d)
    g = {q: t.to(cuda) for q, t in gc.items()}
    segs, o = _layout(n, d)
    dense = {v: _dense(gs, g, v, d, sh_eval, "none", True, o) for v in TIE_VIEWS}
    ex = _Exchange(cuda, n, d, world, (o // 4 + world - 1) // world * 4).sentinels()
    ctxs = [_ctx(gs, sh_eval, "none") for _ in range(world)]
    got = _step(gs, ex, ctxs, g, TIE_VIEWS, True, dense, layout).cpu()
    p = {q: t.double().clone().requires_grad_(True) for q, t in gc.items()}
    ref = None
    for v in TIE_VIEWS:
        vw = VIEWS[v]
        cam = O.Camera(WIDTH, HEIGHT, vw["fx"], vw["fy"], vw["rot"], vw["tran"], vw["near"])
        rgb = G.gaussian_logits(p["pos"], p["rgb"], cam) if sh_eval == "gaussian" else p["rgb"]
        out = F.render_maps(p["pos"], rgb, p["opa"], p["quat"], p["scale"], cam, mode="none", background=BG,
                            use_sh_coeff=sh_eval == "pixel" and d != 3, depth_key=device_depth_keys(gc, cam, cuda))
        up = [u.double().cpu() for u in _upstream(v, cuda)]
        gr = torch.autograd.grad([out["image"], out["depth"], out["alpha"]], [p[q] for q in NAMES], up,
                                 allow_unused=True)
        gr = [torch.zeros_like(p[q]) if t is None else t for q, t in zip(NAMES, gr)]
        ref = gr if ref is None else [a + b for a, b in zip(ref, gr)]
    for k, (q, (s, wd)) in enumerate(zip(NAMES, segs)):
        assert rel_err(got[s:s + n * wd], ref[k].reshape(-1)) < 1e-3, q


def test_densify_stats_unchanged_by_push(gs, cuda):
    """the densification statistics of a pushed backward are those of a plain one, bit for bit"""
    n, world, v = 1203, 4, 1
    g = _scene(3, n, 0, cuda)
    segs, o = _layout(n, 3)
    ex = _Exchange(cuda, n, 3, world, (o // 4 + world - 1) // world * 4).sentinels()
    stats = []
    for alloc in (ex.allocator(1), lambda numel, device: torch.empty(numel, device=device)):
        rctx = _ctx(gs, "pixel", "none")
        st = [torch.zeros(n, device=cuda), torch.zeros(n, dtype=torch.int32, device=cuda), torch.zeros(n, device=cuda)]
        rctx.set_densify_stats(*st, None)
        _render_backward(gs[1], rctx, g, v, True, alloc)
        stats.append(st)
    assert int(stats[0][1].sum()) > 0 and all(torch.equal(a, b) for a, b in zip(*stats))


class _Camera(ctypes.Structure):
    _fields_ = [("width", ctypes.c_int), ("height", ctypes.c_int), ("focal_x", ctypes.c_float),
                ("focal_y", ctypes.c_float), ("rot", ctypes.c_float * 9), ("tran", ctypes.c_float * 3),
                ("near_plane", ctypes.c_float), ("tile_thresh", ctypes.c_float)]


class _Push(ctypes.Structure):
    _fields_ = [("world", ctypes.c_int), ("rank", ctypes.c_int), ("per", ctypes.c_longlong),
                ("bucket", ctypes.c_void_p), ("staging", ctypes.c_void_p * 8)]


def _expect_refused(gaussian, fn, text):
    k0 = gaussian.kernel_launches()
    with pytest.raises(RuntimeError, match=text):
        fn()
    assert gaussian.kernel_launches() == k0


def test_push_refusals_before_any_launch(gs, cuda):
    gaussian, renderer = gs
    n, world = 1202, 2
    g = _scene(3, n, 0, cuda)
    segs, o = _layout(n, 3)
    per = (o // 4 + world - 1) // world * 4
    ex = _Exchange(cuda, n, 3, world, per).sentinels()
    b, st = ex.bucket(0).data_ptr(), [ex.staging_ptr(s) for s in range(world)]
    rctx = _ctx(gs, "pixel", "none")
    # gs_ctx_set_grad_push: world 1 or 3, rank out of range, per 0 / not a multiple of 4 / world * per >= 2^32, a null
    # or misaligned bucket or staging buffer, and (the binding) more than 8 ranks
    for cfg in ((b, st[:1], per, 0), (b, st + st[:1], per, 0), (b, st, per, 2), (b, st, per, -1), (b, st, 0, 0),
                (b, st, per + 2, 0), (b, st, 1 << 31, 0), (0, st, per, 0), (b + 4, st, per, 0), (b, [st[0], 0], per, 0),
                (b, [st[0], st[1] + 4], per, 0), (b, st * 5, per, 0)):
        _expect_refused(gaussian, lambda: rctx.set_grad_push(*cfg), "set_grad_push")

    # a backward whose gradient segments leave the push bucket [bucket, bucket + world * per): refused before the blend
    # backward runs, and the same frame still differentiates afterwards
    vw = VIEWS[0]
    args = (g["pos"], g["rgb"], g["opa"], g["quat"], g["scale"])
    fin, raw, aux, _, _ = rctx.forward_aux(*args, WIDTH, HEIGHT, vw["fx"], vw["fy"], vw["rot"], vw["tran"], vw["near"],
                                           0.05, 0, list(BG), True)
    grad_fin = _upstream(0, cuda)[0]
    views = [ex.bucket(0)[s:s + n * wd] for s, wd in segs]
    rctx.set_grad_push(*ex.push(0))
    outside = torch.empty(n, device=cuda)
    past_end = ex.arena[ex.off_b[0] + world * per - 3 * n + 4:][:3 * n]     # its last float lies past the slices
    for bad in ([views[0], views[1], outside, views[3], views[4]], [*views[:4], past_end]):
        _expect_refused(gaussian, lambda: rctx.backward_aux_into(*args, raw, grad_fin, True, aux, None, *bad, -1),
                        "not inside the push bucket")
    rctx.backward_aux_into(*args, raw, grad_fin, True, aux, None, *views, -1)
    ref_ctx = _ctx(gs, "pixel", "none")
    ref_ctx.forward_aux(*args, WIDTH, HEIGHT, vw["fx"], vw["fy"], vw["rot"], vw["tran"], vw["near"], 0.05, 0, list(BG),
                        True)
    ref = [torch.empty_like(t) for t in args]
    ref_ctx.backward_aux_into(*args, raw, grad_fin, True, aux, None, *ref, -1)
    flat_ref = torch.zeros(o, device=cuda)
    for (s, wd), t in zip(segs, ref):
        flat_ref[s:s + n * wd] = t.reshape(-1)
    assert torch.equal(ex.arena[ex.dest[0]].view(torch.int32), flat_ref.view(torch.int32))

    # grad_quat off a 16-byte bucket offset: the binding refuses a misaligned tensor itself, so call the C ABI
    lib = ctypes.CDLL(os.path.join(PKG, "libgs_b200.so"))
    lib.gs_last_error.restype = ctypes.c_char_p
    P, I = ctypes.c_void_p, ctypes.c_int
    lib.gs_ctx_create.argtypes = [ctypes.POINTER(P)]
    lib.gs_ctx_destroy.argtypes = [P]
    lib.gs_ctx_set_grad_push.argtypes = [P, ctypes.POINTER(_Push)]
    lib.gs_render_forward.argtypes = [P] * 6 + [I] * 3 + [ctypes.POINTER(_Camera), P, P, P]
    lib.gs_render_backward.argtypes = [P] * 14
    stream = torch.cuda.current_stream(cuda).cuda_stream
    cam = _Camera(WIDTH, HEIGHT, vw["fx"], vw["fy"], (ctypes.c_float * 9)(*vw["rot"].flatten().tolist()),
                  (ctypes.c_float * 3)(*vw["tran"].tolist()), vw["near"], 0.05)
    image = torch.empty_like(raw)
    mask = torch.empty(n, dtype=torch.int64, device=cuda)
    grad_img = _upstream(1, cuda)[0]
    grad_img = torch.nn.functional.pad(grad_img, (0, 0, 0, raw.shape[1] - WIDTH, 0, raw.shape[0] - HEIGHT)).contiguous()
    ptr = [t.data_ptr() for t in args]
    ctx = P()
    assert lib.gs_ctx_create(ctypes.byref(ctx)) == 0
    try:
        assert lib.gs_render_forward(ctx, *ptr, n, 3, 0, ctypes.byref(cam), image.data_ptr(), mask.data_ptr(),
                                     stream) == 0
        bp, sp, pr, rk = ex.push(0)
        push = _Push(world, rk, pr, bp, (P * 8)(*sp))
        assert lib.gs_ctx_set_grad_push(ctx, ctypes.byref(push)) == 0
        gp = [t.data_ptr() for t in views]
        gp[3] += 4
        k0 = gaussian.kernel_launches()
        assert lib.gs_render_backward(ctx, *ptr, image.data_ptr(), grad_img.data_ptr(), *gp, stream) == -1
        assert "16-byte bucket offset" in lib.gs_last_error().decode()
        assert gaussian.kernel_launches() == k0
        assert lib.gs_ctx_set_grad_push(ctx, None) == 0
        got = [torch.empty_like(t) for t in args]
        assert lib.gs_render_backward(ctx, *ptr, image.data_ptr(), grad_img.data_ptr(), *(t.data_ptr() for t in got),
                                      stream) == 0
        torch.cuda.synchronize()
    finally:
        lib.gs_ctx_destroy(ctx)
    ref_ctx = gaussian.RenderContext()
    ref_img, _ = ref_ctx.forward(*args, WIDTH, HEIGHT, vw["fx"], vw["fy"], vw["rot"], vw["tran"], vw["near"], 0.05, 0)
    ref = [torch.empty_like(t) for t in args]
    ref_ctx.backward_into(*args, ref_img, grad_img, *ref, -1)
    assert torch.equal(image, ref_img)
    for q, a, r in zip(NAMES, got, ref):
        assert torch.equal(a, r), q

    # the backwards that take no push: the camera gradient and the feature-map gradient, and a batched frame
    p = {q: t.detach().requires_grad_(True) for q, t in g.items()}
    rot, tran = vw["rot"].to(cuda), vw["tran"].to(cuda).requires_grad_(True)
    img, _, _, _ = renderer.render_frame_cam(rctx, *(p[q] for q in NAMES), WIDTH, HEIGHT, vw["fx"], vw["fy"], rot, tran,
                                             vw["near"], 0.05, "abs")
    renderer.set_flat_grad_allocator(ex.allocator(0))
    try:
        _expect_refused(gaussian, lambda: torch.autograd.grad(img, [p["pos"], tran], grad_fin), "push")
        feat = torch.rand(n, 8, device=cuda, requires_grad=True)
        img, fmap, _, _, _ = renderer.render_frame_feat(rctx, *(p[q] for q in NAMES), feat, WIDTH, HEIGHT, vw["fx"],
                                                        vw["fy"], vw["rot"], vw["tran"], vw["near"], 0.05, "abs")
        _expect_refused(gaussian, lambda: torch.autograd.grad([img, fmap], [p["pos"], feat],
                                                              [grad_fin, torch.ones_like(fmap)]), "push")
    finally:
        renderer.set_flat_grad_allocator(None)
    rctx.set_grad_push(*ex.push(0))
    _expect_refused(gaussian, lambda: renderer.render_frame_batch(
        rctx, *(p[q] for q in NAMES), WIDTH, HEIGHT, [vw["fx"]], [vw["fy"]], vw["rot"][None], vw["tran"][None],
        vw["near"], 0.05, "abs"), "push")
