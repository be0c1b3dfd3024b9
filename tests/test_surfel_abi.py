"""gs_render_forward_surfel / gs_render_backward_surfel are declared and exported, gs_render_surfel matches its ctypes
mirror, and bad arguments are refused before any launch: the error code comes back, gs_last_error names the reason
and the launch counter does not move.  The context is a fake that these refusals never dereference; the refusals that
depend on the context's settings are tested on the GPU (tests/test_surfel_gpu.py).  No GPU is needed."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "3d-gaussian-splatting_b200")
HEADER = os.path.join(ROOT, "include", "gs_b200.h")
INVALID, UNSUPPORTED = -1, -2
B = 0x1000          # a fake context
P = ctypes.c_void_p


class Camera(ctypes.Structure):
    _fields_ = [("width", ctypes.c_int), ("height", ctypes.c_int), ("focal_x", ctypes.c_float),
                ("focal_y", ctypes.c_float), ("rot", ctypes.c_float * 9), ("tran", ctypes.c_float * 3),
                ("near_plane", ctypes.c_float), ("tile_thresh", ctypes.c_float)]


class Surfel(ctypes.Structure):
    _fields_ = [("background", P), ("maps", P), ("maps_final", P), ("dist_near", ctypes.c_float),
                ("dist_far", ctypes.c_float)]


def _lib():
    lib = ctypes.CDLL(os.path.join(PKG, "libgs_b200.so"))
    lib.gs_last_error.restype = ctypes.c_char_p
    lib.gs_kernel_launches.restype = ctypes.c_ulonglong
    lib.gs_render_forward_surfel.argtypes = [P] * 6 + [ctypes.c_int] * 3 + [ctypes.POINTER(Camera), P, P, P,
                                                                           ctypes.POINTER(Surfel), P]
    lib.gs_render_backward_surfel.argtypes = [P] * 8 + [ctypes.c_int] + [P] * 7
    return lib


def _cam(**over):
    c = Camera(64, 48, 50.0, 50.0)
    c.rot[0] = c.rot[4] = c.rot[8] = 1.0
    c.near_plane, c.tile_thresh = 0.2, 0.05
    for k, v in over.items():
        setattr(c, k, v)
    return c


def _fwd(lib, ctx=B, n=4, d=3, act=0, surfel="ok", image=0x2000, final=0x3000, **over):
    s = Surfel(None, 0x4000, 0x5000, 0.2, 100.0)
    for k, v in over.items():
        setattr(s, k, v)
    cam = _cam()
    before = lib.gs_kernel_launches()
    rc = lib.gs_render_forward_surfel(ctx, 0x10, 0x20, 0x30, 0x40, 0x50, n, d, act, ctypes.byref(cam), image, final,
                                      None, ctypes.byref(s) if surfel == "ok" else None, None)
    assert lib.gs_kernel_launches() == before, "a refused call must not launch"
    return rc, lib.gs_last_error().decode()


def test_entry_points_declared_and_abi_version_kept():
    text = open(HEADER).read()
    assert re.search(r"\bint gs_render_forward_surfel\(", text)
    assert re.search(r"\bint gs_render_backward_surfel\(", text)
    assert re.search(r"#define GS_SURFEL_MAP_CH 8\b", text)
    lib = _lib()
    lib.gs_abi_version.restype = ctypes.c_int
    assert lib.gs_abi_version() == 2


def test_gs_render_surfel_layout_matches_the_header():
    text = open(HEADER).read()
    body = re.search(r"typedef struct gs_render_surfel \{(.*?)\} gs_render_surfel;", text, re.S).group(1)
    fields = [f.strip() for f in re.sub(r"/\*.*?\*/", "", body, flags=re.S).split(";") if f.strip()]
    assert fields == ["const float* background", "float* maps", "float* maps_final", "float dist_near, dist_far"]
    assert ctypes.sizeof(Surfel) == 32 and Surfel.dist_near.offset == 24 and Surfel.dist_far.offset == 28


def test_forward_refusals():
    lib = _lib()
    rc, msg = _fwd(lib, ctx=None)
    assert rc == INVALID and "bad arguments" in msg
    rc, msg = _fwd(lib, n=-1)
    assert rc == INVALID
    rc, msg = _fwd(lib, d=12)
    assert rc == UNSUPPORTED and "colour width" in msg
    rc, msg = _fwd(lib, image=None)
    assert rc == INVALID and "null tensor" in msg
    rc, msg = _fwd(lib, act=7)
    assert rc == INVALID and "scale activation" in msg
    for near, far in ((0.0, 1.0), (2.0, 1.0), (0.2, float("inf")), (float("nan"), 1.0)):
        rc, msg = _fwd(lib, dist_near=near, dist_far=far)
        assert rc == INVALID and "dist_near" in msg
    rc, msg = _fwd(lib, maps=None)
    assert rc == INVALID and "maps_final needs maps" in msg
    rc, msg = _fwd(lib, final=None)
    assert rc == INVALID and "maps_final needs maps" in msg
    rc, msg = _fwd(lib, maps=0x4004, maps_final=None)
    assert rc == INVALID and "16-byte aligned" in msg
    bg = (ctypes.c_float * 3)(0.0, float("nan"), 0.0)
    rc, msg = _fwd(lib, background=ctypes.cast(bg, P))
    assert rc == INVALID and "background" in msg


def test_backward_refuses_a_null_context():
    lib = _lib()
    before = lib.gs_kernel_launches()
    rc = lib.gs_render_backward_surfel(None, *([0x10] * 7), 0, None, *([0x10] * 5), None)
    assert rc == INVALID and lib.gs_kernel_launches() == before
    assert "null ctx" in lib.gs_last_error().decode()

