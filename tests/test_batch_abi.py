"""The batched frame's C entry points (gs_render_forward_batch / gs_render_backward_batch) are declared and exported,
and refuse before touching the context or CUDA: a null context, null cameras, a view count outside 1 .. GS_MAX_VIEWS,
views that differ in width, height, near plane or tile threshold, more tile rows than the 16-bit row field of a tile
rectangle holds (B Hp / 16 > 65535), and B n >= 2^31 pairs."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "3d-gaussian-splatting_b200")
HEADER = os.path.join(ROOT, "include", "gs_b200.h")


class _Camera(ctypes.Structure):
    _fields_ = [("width", ctypes.c_int), ("height", ctypes.c_int), ("focal_x", ctypes.c_float),
                ("focal_y", ctypes.c_float), ("rot", ctypes.c_float * 9), ("tran", ctypes.c_float * 3),
                ("near_plane", ctypes.c_float), ("tile_thresh", ctypes.c_float)]


def test_batch_entry_points_declared():
    text = open(HEADER).read()
    assert re.search(r"#define GS_MAX_VIEWS 64\b", text)
    for fn in ("gs_render_forward_batch", "gs_render_backward_batch"):
        assert re.search(r"\bint " + fn + r"\(", text), fn


def test_batch_argument_validation_needs_no_gpu():
    lib = ctypes.CDLL(os.path.join(PKG, "libgs_b200.so"))
    lib.gs_last_error.restype = ctypes.c_char_p
    P, I = ctypes.c_void_p, ctypes.c_int

    def err():
        return lib.gs_last_error().decode()

    fwd = lib.gs_render_forward_batch
    fwd.argtypes = [P] * 6 + [I, I, I, I, P, P, P, P, P, P]
    bwd = lib.gs_render_backward_batch
    bwd.argtypes = [P] * 8 + [I] + [P] * 8
    cams = (_Camera * 65)()
    for c in cams:
        c.width, c.height, c.focal_x, c.focal_y = 64, 48, 50.0, 50.0
        c.rot[0] = c.rot[4] = c.rot[8] = 1.0
        c.tran[2] = 4.0
        c.near_plane, c.tile_thresh = 0.3, 0.05
    fake_ctx = P(0x1000)   # never dereferenced: the view count is checked first
    args = [0x2000] * 5

    assert fwd(None, *args, 10, 3, 0, 1, cams, 0x3000, None, None, None, None) == -1 and "null ctx" in err()
    assert fwd(fake_ctx, *args, 10, 3, 0, 1, None, 0x3000, None, None, None, None) == -1 and "cams" in err()
    for b in (0, -1, 65):
        assert fwd(fake_ctx, *args, 10, 3, 0, b, cams, 0x3000, None, None, None, None) == -1
        assert "n_views" in err()
    assert bwd(None, *([0x2000] * 7), 0, *([0x2000] * 7), None) == -1 and "null ctx" in err()


def test_batch_geometry_refusals_need_no_gpu():
    lib = ctypes.CDLL(os.path.join(PKG, "libgs_b200.so"))
    lib.gs_last_error.restype = ctypes.c_char_p
    P, I = ctypes.c_void_p, ctypes.c_int
    fwd = lib.gs_render_forward_batch
    fwd.argtypes = [P] * 6 + [I, I, I, I, P, P, P, P, P, P]
    fake_ctx = P(0x1000)   # never dereferenced: every check below comes first
    args = [0x2000] * 5

    def cams(b, **first):
        cs = (_Camera * b)()
        for c in cs:
            c.width, c.height, c.focal_x, c.focal_y = 64, 48, 50.0, 50.0
            c.rot[0] = c.rot[4] = c.rot[8] = 1.0
            c.tran[2] = 4.0
            c.near_plane, c.tile_thresh = 0.3, 0.05
        for k, v in first.items():
            setattr(cs[b - 1], k, v)
        return cs

    def call(cs, b, n=10):
        rc = fwd(fake_ctx, *args, n, 3, 0, b, cs, 0x3000, None, None, None, None)
        return rc, lib.gs_last_error().decode()

    for field, value in (("width", 80), ("height", 32), ("near_plane", 0.5), ("tile_thresh", 0.1)):
        rc, msg = call(cams(3, **{field: value}), 3)
        assert rc == -1 and "must share width, height, near_plane and tile_thresh" in msg, field
    tall = cams(64)
    for c in tall:
        c.height = 16 * 1024                                      # 1024 tile rows per view, 65,536 in the batch
    rc, msg = call(tall, 64)
    assert rc == -1 and "65535" in msg
    for c in tall:
        c.height = 16 * 1023 + 1                                  # still 1024 rows once padded
    assert call(tall, 64)[0] == -1
    rc, msg = call(cams(64), 64, n=(1 << 31) // 64)               # B n = 2^31
    assert rc == -1 and "2^31" in msg
