"""gs_frame_scores is declared and exported, the ABI version is still 2, and it refuses before any launch what it can
refuse without a context (a null ctx or struct): GS_ERR_INVALID_ARG, gs_last_error set, the launch counter unchanged.
The refusals that need a context (no forward, another n, a surfel or packed-path forward) are in
test_scores_gpu.py."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "3d-gaussian-splatting_b200")
HEADER = os.path.join(ROOT, "include", "gs_b200.h")
INVALID = -1
B = 0x1000          # a fake device pointer


class Scores(ctypes.Structure):
    _fields_ = [("n", ctypes.c_int), ("weight_sum", ctypes.c_void_p), ("weight_max", ctypes.c_void_p)]


def _lib():
    lib = ctypes.CDLL(os.path.join(PKG, "libgs_b200.so"))
    lib.gs_last_error.restype = ctypes.c_char_p
    lib.gs_kernel_launches.restype = ctypes.c_ulonglong
    lib.gs_frame_scores.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    return lib


def test_entry_point_declared_and_abi_version_kept():
    text = open(HEADER).read()
    assert re.search(r"\bint gs_frame_scores\(gs_ctx\* ctx, const struct gs_frame_scores\* s, gs_stream_t stream\)",
                     text)
    assert re.search(r"struct gs_frame_scores \{\s*int n;[^}]*float\* weight_sum;[^}]*float\* weight_max;", text)
    lib = _lib()
    lib.gs_abi_version.restype = ctypes.c_int
    assert lib.gs_abi_version() == 2


def test_refusals_without_a_context_need_no_gpu():
    lib = _lib()
    s = Scores(10, B, B)
    for ctx, ps in ((None, ctypes.byref(s)), (None, None)):
        before = lib.gs_kernel_launches()
        assert lib.gs_frame_scores(ctx, ps, None) == INVALID
        assert "gs_frame_scores" in lib.gs_last_error().decode() and "null" in lib.gs_last_error().decode()
        assert lib.gs_kernel_launches() == before
