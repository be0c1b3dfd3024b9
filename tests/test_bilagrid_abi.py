"""gs_bilagrid_slice_fwd / _bwd / _workspace_bytes are declared and exported, the ABI version is still 2, and every
refusal happens before any launch: GS_ERR_INVALID_ARG, gs_last_error set, the launch counter unchanged.  No GPU is
needed: the pointers are never dereferenced."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "3d-gaussian-splatting_b200")
HEADER = os.path.join(ROOT, "include", "gs_b200.h")
INVALID = -1
P = 0x1000          # a fake device pointer
MAX_HW, MAX_L = 256, 16


def _lib():
    lib = ctypes.CDLL(os.path.join(PKG, "libgs_b200.so"))
    lib.gs_last_error.restype = ctypes.c_char_p
    lib.gs_kernel_launches.restype = ctypes.c_ulonglong
    vp, i = ctypes.c_void_p, ctypes.c_int
    lib.gs_bilagrid_workspace_bytes.restype = ctypes.c_size_t
    lib.gs_bilagrid_workspace_bytes.argtypes = [i] * 7
    lib.gs_bilagrid_slice_fwd.argtypes = [vp, vp, vp] + [i] * 7 + [vp, vp]
    lib.gs_bilagrid_slice_bwd.argtypes = [vp, vp, vp] + [i] * 7 + [vp, vp, vp, vp, ctypes.c_size_t, vp]
    return lib


def _ids(*v):
    return (ctypes.c_int * max(len(v), 1))(*v)


def test_entry_points_declared_and_abi_version_kept():
    text = open(HEADER).read()
    assert re.search(r"size_t gs_bilagrid_workspace_bytes\(int B, int H, int W, int V, int GH, int GW, int GL\);", text)
    assert re.search(r"int gs_bilagrid_slice_fwd\(const float\* image, const float\* grids, const int\* view_ids_host,",
                     text)
    assert re.search(r"int gs_bilagrid_slice_bwd\(const float\* image, const float\* grids, const int\* view_ids_host,",
                     text)
    assert f"#define GS_BILAGRID_MAX_HW {MAX_HW}" in text and f"#define GS_BILAGRID_MAX_L {MAX_L}" in text
    assert "grids.permute(0, 4, 3, 1, 2)" in text
    lib = _lib()
    lib.gs_abi_version.restype = ctypes.c_int
    assert lib.gs_abi_version() == 2
    assert lib.gs_bilagrid_workspace_bytes(2, 64, 64, 4, 16, 16, 8) > 0
    assert lib.gs_bilagrid_workspace_bytes(2, 64, 64, 4, 1, 16, 8) == 0


def _fwd_cases():
    ok = dict(image=P, grids=P, ids=_ids(0, 1), B=2, H=8, W=8, V=2, GH=4, GW=4, GL=4, out=P)
    yield "null image", dict(ok, image=None)
    yield "null grids", dict(ok, grids=None)
    yield "null ids", dict(ok, ids=None)
    yield "null out", dict(ok, out=None)
    for k in ("B", "H", "W", "V"):
        yield f"{k} = 0", dict(ok, **{k: 0})
        yield f"{k} < 0", dict(ok, **{k: -3})
    for k, hi in (("GH", MAX_HW), ("GW", MAX_HW), ("GL", MAX_L)):
        yield f"{k} = 1", dict(ok, **{k: 1})
        yield f"{k} above the bound", dict(ok, **{k: hi + 1})
    yield "view id = V", dict(ok, ids=_ids(0, 2))
    yield "view id < 0", dict(ok, ids=_ids(-1, 0))


def _call_fwd(lib, c):
    return lib.gs_bilagrid_slice_fwd(c["image"], c["grids"], c["ids"], c["B"], c["H"], c["W"], c["V"], c["GH"],
                                     c["GW"], c["GL"], c["out"], None)


def _call_bwd(lib, c, grad_out=P, gi=P, gg=P, ws=P, ws_bytes=None):
    if ws_bytes is None:
        ws_bytes = 1 << 40
    return lib.gs_bilagrid_slice_bwd(c["image"], c["grids"], c["ids"], c["B"], c["H"], c["W"], c["V"], c["GH"],
                                     c["GW"], c["GL"], grad_out, gi, gg, ws, ws_bytes, None)


@pytest.mark.parametrize("name,case", list(_fwd_cases()), ids=[n for n, _ in _fwd_cases()])
def test_refusals_before_any_launch(name, case):
    lib = _lib()
    for fn, call in (("gs_bilagrid_slice_fwd", _call_fwd), ("gs_bilagrid_slice_bwd", _call_bwd)):
        if fn.endswith("bwd") and name == "null out":
            continue
        before = lib.gs_kernel_launches()
        assert call(lib, case) == INVALID, (fn, name)
        assert fn in lib.gs_last_error().decode()
        assert lib.gs_kernel_launches() == before


def test_backward_refusals_before_any_launch():
    lib = _lib()
    c = dict(image=P, grids=P, ids=_ids(0, 1), B=2, H=8, W=8, V=2, GH=4, GW=4, GL=4)
    need = lib.gs_bilagrid_workspace_bytes(2, 8, 8, 2, 4, 4, 4)
    for kw, msg in ((dict(grad_out=None), "null"), (dict(ws=None), "null"), (dict(ws_bytes=need - 1), "workspace")):
        before = lib.gs_kernel_launches()
        assert _call_bwd(lib, c, **kw) == INVALID
        err = lib.gs_last_error().decode()
        assert "gs_bilagrid_slice_bwd" in err and msg in err
        assert lib.gs_kernel_launches() == before
    # nothing requested: no launch, no error
    before = lib.gs_kernel_launches()
    assert _call_bwd(lib, c, gi=None, gg=None, ws_bytes=need) == 0
    assert lib.gs_kernel_launches() == before
