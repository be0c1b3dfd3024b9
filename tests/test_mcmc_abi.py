"""gs_mcmc_relocate / gs_mcmc_add / gs_mcmc_noise are declared and exported, and refuse bad arguments before any
launch: GS_ERR_INVALID_ARG comes back, gs_last_error names the reason and the launch counter does not move.  The
pointers are fakes that a refused call never dereferences; no GPU is needed."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "3d-gaussian-splatting_b200")
HEADER = os.path.join(ROOT, "include", "gs_b200.h")
INVALID = -1
B = 0x1000          # a fake device pointer


def _lib():
    lib = ctypes.CDLL(os.path.join(PKG, "libgs_b200.so"))
    lib.gs_last_error.restype = ctypes.c_char_p
    lib.gs_kernel_launches.restype = ctypes.c_ulonglong
    P, I, F, LL, SZ = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_longlong, ctypes.c_size_t
    lib.gs_mcmc_workspace_bytes.restype = SZ
    lib.gs_mcmc_workspace_bytes.argtypes = [I]
    lib.gs_mcmc_relocate.argtypes = [P, P, P, P, P, P, I, I, I, I, F, P, P, P, LL, P, P, I, P, P, P, SZ, P]
    lib.gs_mcmc_add.argtypes = [P, P, P, P, P, P, I, I, I, I, F, I, P, P, P, P, P, P, P, P, SZ, P]
    lib.gs_mcmc_noise.argtypes = [P, P, P, P, I, I, F, ctypes.c_ulonglong, P, P]
    return lib


def test_entry_points_declared_and_abi_version_kept():
    text = open(HEADER).read()
    for fn in ("gs_mcmc_relocate", "gs_mcmc_add", "gs_mcmc_noise"):
        assert re.search(r"\bint " + fn + r"\(", text), fn
    assert re.search(r"\bsize_t gs_mcmc_workspace_bytes\(", text)
    lib = _lib()
    lib.gs_abi_version.restype = ctypes.c_int
    assert lib.gs_abi_version() == 2          # additive: no signature changed
    assert lib.gs_mcmc_workspace_bytes(-1) == 0
    assert lib.gs_mcmc_workspace_bytes(1000) > lib.gs_mcmc_workspace_bytes(10) > 0


def _relocate(lib, n=100, d=3, f=0, feat=None, act=0, min_opacity=0.005, null=(), moments=False, starts=(0, 300),
              widths=(3, 1), n_flat=400, ws=None, quat=B):
    ptr = {k: (None if k in null else B) for k in ("pos", "rgb", "opa", "quat", "scale", "u", "n_rel", "ws")}
    if "quat" not in null:
        ptr["quat"] = quat
    a_s = (ctypes.c_longlong * max(len(starts), 1))(*starts)
    a_w = (ctypes.c_int * max(len(widths), 1))(*widths)
    m = B if moments else None
    v = None if (moments == "m only") else m
    ws_bytes = lib.gs_mcmc_workspace_bytes(max(n, 0)) if ws is None else ws
    before = lib.gs_kernel_launches()
    rc = lib.gs_mcmc_relocate(ptr["pos"], ptr["rgb"], ptr["opa"], ptr["quat"], ptr["scale"], feat, f, n, d, act,
                              min_opacity, ptr["u"], m, v, n_flat, a_s, a_w, len(starts), None, ptr["n_rel"],
                              ptr["ws"], ws_bytes, None)
    assert lib.gs_kernel_launches() == before, "a refused call must not launch"
    return rc, lib.gs_last_error().decode()


def test_relocate_refusals_need_no_gpu():
    lib = _lib()
    for name in ("pos", "rgb", "opa", "quat", "scale", "u", "n_rel", "ws"):
        rc, msg = _relocate(lib, null=(name,))
        assert rc == INVALID and "bad arguments" in msg, name
    assert _relocate(lib, n=-1)[0] == INVALID
    for d in (0, 4, 9, 16):
        rc, msg = _relocate(lib, d=d)
        assert rc == INVALID and "d must be" in msg, d
    for f in (0, 4, 12, 64):
        rc, msg = _relocate(lib, feat=B, f=f)
        assert rc == INVALID and "d must be" in msg, f
    rc, msg = _relocate(lib, act=2)
    assert rc == INVALID and "activation" in msg
    for mo in (0.0, 1.0, -0.1, 1.5, float("nan")):
        rc, msg = _relocate(lib, min_opacity=mo)
        assert rc == INVALID and "min_opacity" in msg, mo
    rc, msg = _relocate(lib, moments="m only")
    assert rc == INVALID and "moment" in msg
    rc, msg = _relocate(lib, moments=True, starts=(0, 302))
    assert rc == INVALID and "ascending multiples of 4" in msg
    rc, msg = _relocate(lib, moments=True, starts=(0, 296))               # segment 1 starts inside segment 0
    assert rc == INVALID and "overlap" in msg
    rc, msg = _relocate(lib, moments=True, widths=(3, 0))
    assert rc == INVALID and "widths" in msg
    rc, msg = _relocate(lib, moments=True, n_flat=396)
    assert rc == INVALID and "beyond the flat buffer" in msg
    rc, msg = _relocate(lib, moments=True, n_flat=402)
    assert rc == INVALID and "segment table" in msg
    rc, msg = _relocate(lib, moments=True, starts=tuple(range(0, 3600, 400)), widths=(1,) * 9, n_flat=4000)
    assert rc == INVALID and "segment table" in msg                        # 9 segments
    rc, msg = _relocate(lib, ws=16)
    assert rc == INVALID and "workspace too small" in msg
    rc, msg = _relocate(lib, quat=B + 4)                                 # quat rows are read as float4
    assert rc == INVALID and "16-byte aligned" in msg


def test_relocate_with_no_gaussians_is_a_no_op():
    lib = _lib()
    assert _relocate(lib, n=0, null=("pos", "rgb", "opa", "quat", "scale", "u", "n_rel", "ws"))[0] == 0
    assert _relocate(lib, n=0, d=5)[0] == INVALID                         # still validated


def _add(lib, n=100, n_new=5, d=48, f=0, feat=None, out_feat=None, act=1, min_opacity=0.005, null=(), ws=None):
    ptr = {k: (None if k in null else B) for k in ("pos", "rgb", "opa", "quat", "scale", "u", "out", "ws")}
    o = ptr["out"]
    ws_bytes = lib.gs_mcmc_workspace_bytes(max(n, n_new, 0)) if ws is None else ws
    before = lib.gs_kernel_launches()
    rc = lib.gs_mcmc_add(ptr["pos"], ptr["rgb"], ptr["opa"], ptr["quat"], ptr["scale"], feat, f, n, d, act, min_opacity,
                         n_new, ptr["u"], o, o, o, o, o, out_feat, ptr["ws"], ws_bytes, None)
    assert lib.gs_kernel_launches() == before, "a refused call must not launch"
    return rc, lib.gs_last_error().decode()


def test_add_refusals_need_no_gpu():
    lib = _lib()
    for name in ("pos", "rgb", "opa", "quat", "scale", "u", "out", "ws"):
        rc, msg = _add(lib, null=(name,))
        assert rc == INVALID and "bad arguments" in msg, name
    assert _add(lib, n_new=-1)[0] == INVALID
    assert _add(lib, n=0, n_new=3)[0] == INVALID                          # nothing to copy from
    rc, msg = _add(lib, feat=B, f=8, out_feat=None)
    assert rc == INVALID and "bad arguments" in msg
    rc, msg = _add(lib, feat=B, f=10, out_feat=B)
    assert rc == INVALID and "d must be" in msg
    rc, msg = _add(lib, d=7)
    assert rc == INVALID and "d must be" in msg
    rc, msg = _add(lib, act=-1)
    assert rc == INVALID and "activation" in msg
    rc, msg = _add(lib, min_opacity=1.0)
    assert rc == INVALID and "min_opacity" in msg
    rc, msg = _add(lib, n=10, n_new=500, ws=lib.gs_mcmc_workspace_bytes(10))   # needs max(n, n_new)
    assert rc == INVALID and "workspace too small" in msg
    rc, msg = _add(lib, n=2 ** 31 - 10, n_new=20, ws=0)
    assert rc == INVALID and "fit an int" in msg
    before = lib.gs_kernel_launches()
    rc = lib.gs_mcmc_add(B, B, B, B, B, None, 0, 100, 3, 0, 0.005, 5, B, B, B, B, B + 8, B, None, B,
                         lib.gs_mcmc_workspace_bytes(100), None)
    assert rc == INVALID and "16-byte aligned" in lib.gs_last_error().decode()
    assert lib.gs_kernel_launches() == before


def test_noise_refusals_need_no_gpu():
    lib = _lib()
    before = lib.gs_kernel_launches()
    for i in range(4):
        ptrs = [B] * 4
        ptrs[i] = None
        assert lib.gs_mcmc_noise(*ptrs, 10, 0, 1.0, 7, None, None) == INVALID
        assert "bad arguments" in lib.gs_last_error().decode()
    assert lib.gs_mcmc_noise(B, B, B, B, -1, 0, 1.0, 7, None, None) == INVALID
    assert lib.gs_mcmc_noise(B, B, B, B, 10, 3, 1.0, 7, None, None) == INVALID
    assert "activation" in lib.gs_last_error().decode()
    for s in (float("nan"), float("inf")):
        assert lib.gs_mcmc_noise(B, B, B, B, 10, 1, s, 7, None, None) == INVALID
        assert "scaler" in lib.gs_last_error().decode()
    assert lib.gs_mcmc_noise(B, B + 4, B, B, 10, 1, 1.0, 7, None, None) == INVALID
    assert "16-byte aligned" in lib.gs_last_error().decode()
    assert lib.gs_mcmc_noise(None, None, None, None, 0, 0, 1.0, 7, None, None) == 0
    assert lib.gs_kernel_launches() == before
