"""gs_ctx_set_filter3d / gs_filter3d_compute are declared and exported, and refuse bad arguments before any launch:
GS_ERR_INVALID_ARG comes back, gs_last_error names the reason and the launch counter does not move.  The context and
device pointers are fakes that a refused call never dereferences; no GPU is needed.  Splatter's filter3d_variance is
validated before anything touches a device."""
import ctypes
import math
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "3d-gaussian-splatting_b200")
HEADER = os.path.join(ROOT, "include", "gs_b200.h")
INVALID = -1
B = 0x1000          # a fake device pointer / context


class Camera(ctypes.Structure):
    _fields_ = [("width", ctypes.c_int), ("height", ctypes.c_int), ("focal_x", ctypes.c_float),
                ("focal_y", ctypes.c_float), ("rot", ctypes.c_float * 9), ("tran", ctypes.c_float * 3),
                ("near_plane", ctypes.c_float), ("tile_thresh", ctypes.c_float)]


def _lib():
    lib = ctypes.CDLL(os.path.join(PKG, "libgs_b200.so"))
    lib.gs_last_error.restype = ctypes.c_char_p
    lib.gs_kernel_launches.restype = ctypes.c_ulonglong
    P, I, F = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    lib.gs_ctx_set_filter3d.argtypes = [P, P, I]
    lib.gs_filter3d_compute.argtypes = [P, P, I, P, I, F, F, P, P]
    return lib


def _cams(k=2, **over):
    arr = (Camera * k)()
    for c in arr:
        c.width, c.height, c.focal_x, c.focal_y = 64, 48, 50.0, 50.0
        c.rot[0] = c.rot[4] = c.rot[8] = 1.0
        c.near_plane, c.tile_thresh = 0.3, 0.05
    for name, value in over.items():
        setattr(arr[k - 1], name, value)
    return arr


def _compute(lib, ctx=B, pos=B, n=10, cams="ok", n_cams=2, margin=0.15, variance=0.2, out=B, **cam_over):
    arr = _cams(max(n_cams, 1), **cam_over) if cams == "ok" else None
    before = lib.gs_kernel_launches()
    rc = lib.gs_filter3d_compute(ctx, pos, n, arr, n_cams, margin, variance, out, None)
    assert lib.gs_kernel_launches() == before, "a refused call must not launch"
    return rc, lib.gs_last_error().decode()


def test_entry_points_declared_and_abi_version_kept():
    text = open(HEADER).read()
    for fn in ("gs_ctx_set_filter3d", "gs_filter3d_compute"):
        assert re.search(r"\bint " + fn + r"\(", text), fn
    lib = _lib()
    lib.gs_abi_version.restype = ctypes.c_int
    assert lib.gs_abi_version() == 2          # additive: no signature changed


def test_set_filter3d_refusals():
    lib = _lib()
    assert lib.gs_ctx_set_filter3d(None, B, 10) == INVALID
    assert "null ctx" in lib.gs_last_error().decode()
    assert lib.gs_ctx_set_filter3d(None, None, 0) == INVALID
    assert lib.gs_ctx_set_filter3d(B, B, -1) == INVALID
    assert "n < 0" in lib.gs_last_error().decode()


def test_compute_refusals_need_no_gpu():
    lib = _lib()
    for kw in (dict(ctx=None), dict(pos=None), dict(out=None), dict(cams=None)):
        rc, msg = _compute(lib, **kw)
        assert rc == INVALID and "null argument" in msg, kw
    for kw in (dict(n=-1), dict(n_cams=0), dict(n_cams=-3)):
        rc, msg = _compute(lib, **kw)
        assert rc == INVALID and "n_cams" in msg, kw
    for v in (0.0, -0.1, math.nan, math.inf):
        rc, msg = _compute(lib, variance=v)
        assert rc == INVALID and "variance" in msg, v
    for m in (-0.01, math.nan, math.inf):
        rc, msg = _compute(lib, margin=m)
        assert rc == INVALID and "margin" in msg, m
    for kw in (dict(width=0), dict(height=-2), dict(focal_x=0.0), dict(focal_y=-1.0), dict(focal_x=math.nan),
               dict(focal_y=math.inf)):
        rc, msg = _compute(lib, **kw)
        assert rc == INVALID and "bad camera" in msg, kw
    for near in (math.nan, -0.5):
        rc, msg = _compute(lib, near_plane=near)
        assert rc == INVALID and "near_plane" in msg, near
    # margin 0 is allowed; n == 0 does nothing (empty tensors may have null pointers) and needs no device
    assert _compute(lib, n=0, margin=0.0)[0] == 0
    assert _compute(lib, n=0, pos=None, out=None)[0] == 0


@pytest.mark.parametrize("bad", [0.0, -1.0, math.nan, math.inf, "x"])
def test_splatter_refuses_a_bad_filter3d_variance(bad):
    import splatter
    views = [dict(width=32, height=32, focal_x=30.0, focal_y=30.0, rot=[[1, 0, 0], [0, 1, 0], [0, 0, 1]],
                  tran=[0, 0, 0])]
    import torch
    g = dict(pos=torch.zeros(2, 3), rgb=torch.zeros(2, 3), opa=torch.zeros(2), quat=torch.tensor([[1.0, 0, 0, 0]] * 2),
             scale=torch.full((2, 3), 0.01))
    with pytest.raises(ValueError, match="filter3d_variance"):
        splatter.Splatter.from_tensors(g, views, device="cpu", filter3d=True, filter3d_variance=bad)
