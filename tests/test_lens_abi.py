"""gs_ctx_set_lens is declared and exported, gs_lens matches its ctypes mirror, and bad arguments are refused before
any launch: GS_ERR_INVALID_ARG comes back, gs_last_error names the reason and the launch counter does not move.  The
context is a fake that a refused call never dereferences; no GPU is needed.  Splatter refuses a bad camera_model and an
unsupported COLMAP camera before anything touches a device."""
import ctypes
import math
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "3d-gaussian-splatting_b200")
HEADER = os.path.join(ROOT, "include", "gs_b200.h")
INVALID = -1
B = 0x1000          # a fake context


class Lens(ctypes.Structure):
    _fields_ = [("model", ctypes.c_int), ("cx", ctypes.c_float), ("cy", ctypes.c_float), ("k", ctypes.c_float * 4)]


def _lib():
    lib = ctypes.CDLL(os.path.join(PKG, "libgs_b200.so"))
    lib.gs_last_error.restype = ctypes.c_char_p
    lib.gs_kernel_launches.restype = ctypes.c_ulonglong
    lib.gs_ctx_set_lens.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    return lib


def _lenses(n, **over):
    arr = (Lens * max(n, 1))()
    for ln in arr:
        ln.model, ln.cx, ln.cy = 1, 32.0, 24.0
    for name, value in over.items():
        if name.startswith("k"):
            arr[n - 1].k[int(name[1:])] = value
        else:
            setattr(arr[n - 1], name, value)
    return arr


def _set(lib, ctx=B, lenses="ok", n=2, **over):
    arr = _lenses(n, **over) if lenses == "ok" else None
    before = lib.gs_kernel_launches()
    rc = lib.gs_ctx_set_lens(ctx, arr, n)
    assert lib.gs_kernel_launches() == before, "a refused call must not launch"
    return rc, lib.gs_last_error().decode()


def test_entry_point_declared_and_abi_version_kept():
    text = open(HEADER).read()
    assert re.search(r"\bint gs_ctx_set_lens\(", text)
    for name, value in (("GS_LENS_PINHOLE", 0), ("GS_LENS_OPENCV", 1), ("GS_LENS_FISHEYE", 2)):
        assert re.search(r"#define " + name + r" " + str(value) + r"\b", text), name
    lib = _lib()
    lib.gs_abi_version.restype = ctypes.c_int
    assert lib.gs_abi_version() == 2          # additive: no signature changed


def test_gs_lens_layout_matches_the_header():
    text = open(HEADER).read()
    body = re.search(r"typedef struct gs_lens \{(.*?)\} gs_lens;", text, re.S).group(1)
    fields = re.findall(r"\b(int|float)\s+([\w, \[\]0-9]+);", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert fields == [("int", "model"), ("float", "cx, cy"), ("float", "k[4]")]
    assert ctypes.sizeof(Lens) == 28 and Lens.cx.offset == 4 and Lens.k.offset == 12


def test_set_lens_refusals():
    lib = _lib()
    rc, msg = _set(lib, ctx=None)
    assert rc == INVALID and "null ctx" in msg
    for n in (-1, 65):
        rc, msg = _set(lib, n=n)
        assert rc == INVALID and "GS_MAX_VIEWS" in msg, n
    rc, msg = _set(lib, lenses=None, n=1)
    assert rc == INVALID and "NULL lenses" in msg
    for model in (-1, 3, 7):
        rc, msg = _set(lib, model=model)
        assert rc == INVALID and "model" in msg, model
    for kw in (dict(cx=math.nan), dict(cy=math.inf), dict(k0=math.nan), dict(k3=-math.inf)):
        rc, msg = _set(lib, **kw)
        assert rc == INVALID and "finite" in msg, kw


def _views():
    return [dict(width=32, height=32, focal_x=30.0, focal_y=30.0, rot=[[1, 0, 0], [0, 1, 0], [0, 0, 1]], tran=[0, 0, 0])]


def _gaussians():
    import torch
    return dict(pos=torch.zeros(2, 3), rgb=torch.zeros(2, 3), opa=torch.zeros(2), quat=torch.tensor([[1.0, 0, 0, 0]] * 2),
                scale=torch.full((2, 3), 0.01))


@pytest.mark.parametrize("bad", ["opencv", "", None, "pinhole"])
def test_splatter_refuses_a_bad_camera_model(bad):
    import splatter
    with pytest.raises(ValueError, match="camera_model"):
        splatter.Splatter.from_tensors(_gaussians(), _views(), device="cpu", camera_model=bad)


@pytest.mark.parametrize("model", ["FULL_OPENCV", "FOV", "THIN_PRISM_FISHEYE"])
def test_splatter_refuses_an_unsupported_colmap_camera(tmp_path, model):
    import colmap_io
    import splatter
    npar = dict(colmap_io.CAMERA_MODELS.values())[model]
    params = np.array([40.0, 40.0, 32.0, 24.0] + [0.0] * (npar - 4))
    colmap_io.write_cameras_binary(str(tmp_path / "cameras.bin"), {1: colmap_io.Camera(1, model, 64, 48, params)})
    colmap_io.write_images_binary(str(tmp_path / "images.bin"), {})
    colmap_io.write_points3d_binary(str(tmp_path / "points3D.bin"),
                                    {1: colmap_io.Point3D(1, np.zeros(3), np.array([1, 2, 3]), 0.0)})
    with pytest.raises(ValueError, match=model):
        splatter.Splatter(str(tmp_path), str(tmp_path), device="cpu", camera_model="colmap")


def test_colmap_intrinsics_mapping():
    import splatter
    p = [100.0, 90.0, 33.0, 25.0, 0.1, 0.2, 0.3, 0.4]
    assert splatter.colmap_intrinsics("OPENCV", p, 2) == (50.0, 45.0, dict(model="OPENCV", cx=16.5, cy=12.5,
                                                                         k=[0.1, 0.2, 0.3, 0.4]))
    assert splatter.colmap_intrinsics("OPENCV_FISHEYE", p)[2]["model"] == "FISHEYE"
    assert splatter.colmap_intrinsics("SIMPLE_RADIAL", [80.0, 30.0, 20.0, -0.1]) == (
        80.0, 80.0, dict(model="OPENCV", cx=30.0, cy=20.0, k=[-0.1, 0.0, 0.0, 0.0]))
    assert splatter.colmap_intrinsics("RADIAL_FISHEYE", [80.0, 30.0, 20.0, 0.1, 0.2])[2] == dict(
        model="FISHEYE", cx=30.0, cy=20.0, k=[0.1, 0.2, 0.0, 0.0])
    assert splatter.colmap_intrinsics("SIMPLE_PINHOLE", [80.0, 31.0, 21.0])[2] == dict(
        model="PINHOLE", cx=31.0, cy=21.0, k=[0.0, 0.0, 0.0, 0.0])
