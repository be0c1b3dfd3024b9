"""gs_adam_step_visible and gs_frame_visible are declared and exported, and refuse bad arguments before any launch:
the documented code comes back, gs_last_error names the reason and the launch counter does not move.  The pointers are
fakes that a refused call never dereferences; no GPU is needed.  (gs_frame_visible's refusals that need a live context
- no forward yet, another n - are in tests/test_visible_adam_gpu.py.)"""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "3d-gaussian-splatting_b200")
HEADER = os.path.join(ROOT, "include", "gs_b200.h")
INVALID = -1


def _lib():
    lib = ctypes.CDLL(os.path.join(PKG, "libgs_b200.so"))
    lib.gs_last_error.restype = ctypes.c_char_p
    lib.gs_kernel_launches.restype = ctypes.c_ulonglong
    P, I, F, LL = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_longlong
    lib.gs_adam_step_visible.argtypes = [P, P, P, P, LL, P, P, P, I, I, P, F, F, F, I, P]
    lib.gs_frame_visible.argtypes = [P, P, I, I, P]
    return lib


def test_entry_points_declared_and_abi_version_kept():
    text = open(HEADER).read()
    for fn in ("gs_adam_step_visible", "gs_frame_visible"):
        assert re.search(r"\bint " + fn + r"\(", text), fn
    lib = _lib()
    lib.gs_abi_version.restype = ctypes.c_int
    assert lib.gs_abi_version() == 2          # additive: no signature changed


def _call(lib, n_flat=4000, starts=(0, 304, 2000), widths=(3, 16, 4), lrs=(0.1, 0.2, 0.3), n_seg=None, n_rows=100,
          step=1, bufs=0x1000, visible=0x2000, null=()):
    k = len(starts)
    a_s = (ctypes.c_longlong * max(k, 1))(*starts)
    a_w = (ctypes.c_int * max(len(widths), 1))(*widths)
    a_l = (ctypes.c_float * max(len(lrs), 1))(*lrs)
    before = lib.gs_kernel_launches()
    rc = lib.gs_adam_step_visible(bufs, bufs, bufs, bufs, n_flat,
                                  None if "starts" in null else a_s, None if "widths" in null else a_w,
                                  None if "lrs" in null else a_l, k if n_seg is None else n_seg, n_rows, visible, 0.9,
                                  0.99, 1e-8, step, None)
    assert lib.gs_kernel_launches() == before, "a refused or empty call must not launch"
    return rc, lib.gs_last_error().decode()


def test_adam_step_visible_refusals_need_no_gpu():
    lib = _lib()
    rc, msg = _call(lib, step=0)
    assert rc == INVALID and "bad arguments" in msg
    for k in (0, 9, -1):
        rc, msg = _call(lib, n_seg=k)
        assert rc == INVALID and "bad arguments" in msg, k
    for name in ("starts", "widths", "lrs"):
        rc, msg = _call(lib, null=(name,))
        assert rc == INVALID and "bad arguments" in msg, name
    assert _call(lib, n_rows=-1)[0] == INVALID
    assert _call(lib, n_flat=-4)[0] == INVALID
    rc, msg = _call(lib, n_flat=4001)
    assert rc == INVALID and "multiple of 4" in msg
    rc, msg = _call(lib, starts=(0, 302, 2000))                       # not a multiple of 4
    assert rc == INVALID and "ascending multiples of 4" in msg
    rc, msg = _call(lib, starts=(0, 2000, 304))                       # descending
    assert rc == INVALID and "ascending multiples of 4" in msg
    rc, msg = _call(lib, starts=(0, 296, 2000))                       # segment 1 starts inside segment 0 (300 floats)
    assert rc == INVALID and "overlap" in msg
    for w in (0, -3, (1 << 24) + 1):
        rc, msg = _call(lib, widths=(3, w, 4))
        assert rc == INVALID and "widths" in msg, w
    rc, msg = _call(lib, starts=(0, 304, 3700))                       # 3700 + 100 * 4 > 4000
    assert rc == INVALID and "beyond the flat buffer" in msg
    rc, msg = _call(lib, bufs=None)
    assert rc == INVALID and "null buffer" in msg
    rc, msg = _call(lib, visible=None)
    assert rc == INVALID and "null buffer" in msg


def test_adam_step_visible_with_no_rows_is_a_no_op():
    lib = _lib()
    assert _call(lib, n_rows=0)[0] == 0
    assert _call(lib, n_rows=0, bufs=None, visible=None, n_flat=0, starts=(0, 0, 0))[0] == 0
    assert _call(lib, n_rows=0, step=0)[0] == INVALID                 # still validated


def test_frame_visible_refuses_null_arguments():
    lib = _lib()
    before = lib.gs_kernel_launches()
    assert lib.gs_frame_visible(None, 0x2000, 10, 0, None) == INVALID
    assert "null" in lib.gs_last_error().decode()
    assert lib.gs_frame_visible(0x1000, None, 10, 0, None) == INVALID     # the mask is checked before the ctx is read
    assert "null" in lib.gs_last_error().decode()
    assert lib.gs_kernel_launches() == before
