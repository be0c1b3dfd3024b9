"""The fused L1 + SSIM loss (csrc/loss.cu) and the bilateral-grid slice (csrc/bilagrid.cu) on the edge fixtures of
tests/image_edges.py, against the fp64 oracles with the per-element comparators: every tile-position case of the
loss's inner band and last tile, flat / equal / checkerboard / impulse contents with float32 and float16 targets,
every call of the loss API, the no-gradient path, a non-contiguous image, a 4K frame's determinism; round-up knot
pixels, grids with more cells than pixels, empty row slices and the slice's launch splits.  Through the C ABI, every
output word is checked to be written over a NaN sentinel, and the grid rows of views outside the batch to keep it."""
import ctypes
import os

import pytest
import torch

import image_edges as E

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENT = 0x7FC0BEEF          # a quiet NaN nobody writes


def _lib():
    lib = ctypes.CDLL(os.path.join(ROOT, "3d-gaussian-splatting_b200", "libgs_b200.so"))
    vp, i, f, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_size_t
    lib.gs_last_error.restype = ctypes.c_char_p
    lib.gs_loss_workspace_bytes.restype = sz
    lib.gs_loss_workspace_bytes.argtypes = [i, i]
    lib.gs_loss_l1_ssim.argtypes = [vp, vp, i, i, i, f, f, f, vp, vp, vp, sz, vp]
    lib.gs_bilagrid_workspace_bytes.restype = sz
    lib.gs_bilagrid_workspace_bytes.argtypes = [i] * 7
    lib.gs_bilagrid_slice_fwd.argtypes = [vp, vp, vp] + [i] * 7 + [vp, vp]
    lib.gs_bilagrid_slice_bwd.argtypes = [vp, vp, vp] + [i] * 7 + [vp, vp, vp, vp, sz, vp]
    return lib


def _sentinel(n, dev):
    return torch.full((n,), SENT, dtype=torch.int32, device=dev)


def _sent_f32(shape, dev):
    return _sentinel(torch.Size(shape).numel(), dev).view(torch.float32).view(*shape)


def _is_sent(t):
    return t.contiguous().view(torch.int32) == SENT


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


# ------------------------------------------------------------------------------------------------------------- loss
LOSS_CASES = [(h, w, c, half) for (h, w) in E.LOSS_SHAPES for c in E.CONTENTS for half in (False, True)]


def _call(mode, x, y):
    import loss
    if mode == "ssim":
        return (loss.ssim(x, y),)
    if mode == "l1":
        return (loss.l1(x, y),)
    return loss.l1_ssim_loss(x, y, float(mode[2:]))


def _check_values(ref, mode, outs):
    v, bound = ref.value(mode)
    assert abs(float(outs[0]) - v) <= bound, (mode, float(outs[0]), v, bound)
    if len(outs) == 3:
        assert abs(float(outs[1]) - ref.l1) <= ref.l1_bound(), (mode, "l1")
        assert abs(float(outs[2]) - (1 - ref.ssim)) <= ref.ssim_bound() + E.C_VAL * E.EPS32, (mode, "ssim_loss")


def _run_loss_calls(x, y, ref):
    for mode in E.CALLS:
        xg = x.clone().requires_grad_(True)
        outs = _call(mode, xg, y)
        outs[0].backward()
        _check_values(ref, mode, outs)
        g, gb = ref.grad(mode)
        r = E.excess(xg.grad, g, gb)
        assert r <= 1.0, (mode, r)
        # the no-gradient path (grad_image NULL) gives the same value bits
        with torch.no_grad():
            plain = _call(mode, x, y)
        for a, b in zip(plain, outs):
            assert torch.equal(a, b.detach()), mode


@pytest.mark.parametrize("h,w,content,half", LOSS_CASES,
                         ids=[f"{h}x{w}-{c}-{'f16' if hf else 'f32'}" for h, w, c, hf in LOSS_CASES])
def test_loss_matches_oracle_per_element(gs, cuda, h, w, content, half):
    x, y = E.loss_pair(h, w, content, half)
    x, y = x.to(cuda), y.to(cuda)
    ref = E.LossRef(x, y)
    _run_loss_calls(x, y, ref)


@pytest.mark.parametrize("h,w", [(33, 42), (12, 16), (2000, 11)])
def test_loss_of_a_non_contiguous_image(gs, cuda, h, w):
    import loss
    x, y = E.loss_pair(h, w, "noise")
    x, y = x.to(cuda), y.to(cuda)
    xt = x.transpose(0, 1).contiguous().transpose(0, 1).requires_grad_(True)        # same values, column-major
    assert not xt.is_contiguous()
    xc = x.clone().requires_grad_(True)
    a, b = loss.l1_ssim_loss(xt, y, 0.1), loss.l1_ssim_loss(xc, y, 0.1)
    a[0].backward()
    b[0].backward()
    for p, q in zip(a, b):
        assert torch.equal(p.detach(), q.detach())
    assert torch.equal(xt.grad, xc.grad)


@pytest.mark.parametrize("half", [False, True], ids=["f32", "f16"])
def test_loss_uhd_frame_matches_oracle_and_is_deterministic(gs, cuda, half):
    import loss
    x, y = E.loss_pair(*E.UHD, "mixed", half)
    x, y = x.to(cuda), y.to(cuda)
    ref = E.LossRef(x, y)
    runs = []
    for _ in range(2):
        xg = x.clone().requires_grad_(True)
        outs = loss.l1_ssim_loss(xg, y, 0.1)
        outs[0].backward()
        runs.append((torch.stack([o.detach() for o in outs]), xg.grad))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    _check_values(ref, "w=0.1", runs[0][0])
    g, gb = ref.grad("w=0.1")
    assert E.excess(runs[0][1], g, gb) <= 1.0


def _abi_loss(lib, x, y, w_l1, w_ssim, bias, grad=True):
    h, w = x.shape[:2]
    nws = lib.gs_loss_workspace_bytes(h, w)
    ws = _sentinel(nws // 4, x.device)
    gi = _sent_f32((h, w, 3), x.device) if grad else None
    out3 = _sent_f32((3,), x.device)
    rc = lib.gs_loss_l1_ssim(x.data_ptr(), y.data_ptr(), int(y.dtype == torch.float16), h, w, w_l1, w_ssim, bias,
                             gi.data_ptr() if grad else None, out3.data_ptr(), ws.data_ptr(), nws, _stream())
    assert rc == 0, lib.gs_last_error()
    torch.cuda.synchronize()
    return out3, gi


@pytest.mark.parametrize("h,w", E.LOSS_SHAPES + [E.UHD])
@pytest.mark.parametrize("half", [False, True], ids=["f32", "f16"])
def test_loss_writes_every_gradient_word_over_nan(gs, cuda, h, w, half):
    """NaN-filled workspace, grad_image and out3: every word of grad_image and out3 is overwritten, finite, and equal
    to the binding's (whose buffers are fresh allocations); nothing the gradient pass reads is left unwritten."""
    gaussian, _ = gs
    lib = _lib()
    x, y = E.loss_pair(h, w, "impulse" if (h, w) != E.UHD else "mixed", half)
    x, y = x.to(cuda), y.to(cuda)
    out3, gi = _abi_loss(lib, x, y, 0.9, -0.1, 0.1)
    assert bool(torch.isfinite(gi).all()) and bool(torch.isfinite(out3).all())
    b_out3, b_gi = gaussian.loss_l1_ssim(x, y, 0.9, -0.1, 0.1, True)
    assert torch.equal(out3, b_out3) and torch.equal(gi, b_gi)
    out3_ng, _ = _abi_loss(lib, x, y, 0.9, -0.1, 0.1, grad=False)
    assert torch.equal(out3_ng, out3)


# --------------------------------------------------------------------------------------------------- bilateral grid
SLICE_CASES = list(E.SLICE_BUILDERS)


def _abi_slice(lib, case, dev):
    img, grids, go = case.image.to(dev), case.grids.to(dev), case.go.to(dev)
    b, h, w, _ = img.shape
    v, gh, gw, gl, _ = grids.shape
    ids = (ctypes.c_int * b)(*case.ids)
    out = _sent_f32(tuple(img.shape), dev)
    assert lib.gs_bilagrid_slice_fwd(img.data_ptr(), grids.data_ptr(), ids, b, h, w, v, gh, gw, gl, out.data_ptr(),
                                     _stream()) == 0, lib.gs_last_error()
    nws = lib.gs_bilagrid_workspace_bytes(b, h, w, v, gh, gw, gl)
    ws = _sentinel((nws + 3) // 4, dev)
    gi = _sent_f32(tuple(img.shape), dev)
    gg = _sent_f32(tuple(grids.shape), dev)
    assert lib.gs_bilagrid_slice_bwd(img.data_ptr(), grids.data_ptr(), ids, b, h, w, v, gh, gw, gl, go.data_ptr(),
                                     gi.data_ptr(), gg.data_ptr(), ws.data_ptr(), nws, _stream()) == 0, \
        lib.gs_last_error()
    torch.cuda.synchronize()
    return out, gi, gg


@pytest.mark.parametrize("name", SLICE_CASES)
def test_slice_matches_oracle_and_writes_exactly_its_rows(gs, cuda, name):
    gaussian, _ = gs
    case = E.SLICE_BUILDERS[name]()
    ref = E.SliceRef(case)
    out, gi, gg = _abi_slice(_lib(), case, cuda)
    assert bool(torch.isfinite(out).all()) and bool(torch.isfinite(gi).all())
    views = case.views
    others = [v for v in range(case.grids.shape[0]) if v not in views]
    assert bool(torch.isfinite(gg[views]).all())
    assert others and bool(_is_sent(gg[others]).all())
    r = E.slice_excess(ref, case, out.cpu(), gi.cpu(), gg.cpu())
    assert max(r) <= 1.0, r
    # the binding (fresh and zeroed buffers) computes the same bits
    img, grids, go = case.image.to(cuda), case.grids.to(cuda), case.go.to(cuda)
    assert torch.equal(gaussian.bilagrid_slice(img, grids, case.ids), out)
    b_gi, b_gg = gaussian.bilagrid_slice_backward(img, grids, case.ids, go, True, True)
    assert torch.equal(b_gi, gi) and torch.equal(b_gg[views], gg[views])
    assert torch.count_nonzero(b_gg[others]) == 0


def test_slice_refuses_seventeen_knots(gs, cuda):
    import bilagrid_oracle as BO
    gaussian, _ = gs
    px = torch.from_numpy(BO.knot_pixels(17, 16, seed=17)).reshape(1, 4, 4, 3).to(cuda)
    with pytest.raises(RuntimeError, match="grid dimensions"):
        gaussian.bilagrid_slice(px, BO.random_grids(1, 3, 3, 17, seed=1).float().to(cuda), [0])
