"""The batched camera-gradient backward's C entry point (gs_render_backward_batch_cam) is declared and exported, and
refuses a null context, a null grad_cams and a mixed set of parameter gradients with GS_ERR_INVALID_ARG before it reads
the context or touches CUDA."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "3d-gaussian-splatting_b200")
HEADER = os.path.join(ROOT, "include", "gs_b200.h")


def _invalid_arg():
    m = re.search(r"#define GS_ERR_INVALID_ARG\s+\(?(-?\d+)\)?", open(HEADER).read())
    assert m
    return int(m.group(1))


def test_batch_cam_entry_point_declared_and_exported():
    text = open(HEADER).read()
    assert re.search(r"\bint gs_render_backward_batch_cam\(", text)
    lib = ctypes.CDLL(os.path.join(PKG, "libgs_b200.so"))
    assert hasattr(lib, "gs_render_backward_batch_cam")


def test_batch_cam_argument_validation_needs_no_gpu():
    lib = ctypes.CDLL(os.path.join(PKG, "libgs_b200.so"))
    lib.gs_last_error.restype = ctypes.c_char_p
    P, I = ctypes.c_void_p, ctypes.c_int
    bwd = lib.gs_render_backward_batch_cam
    bwd.argtypes = [P] * 8 + [I] + [P] * 9
    bwd.restype = I
    invalid = _invalid_arg()
    fake_ctx = P(0x1000)   # never dereferenced: these checks come first
    tensors = [0x2000] * 7   # pos, rgb, opa, quat, scale, image, grad_image
    grads = [0x3000] * 5
    cams = 0x4000

    def call(ctx, g, grad_cams):
        rc = bwd(ctx, *tensors, 0, None, None, *g, grad_cams, None)
        return rc, lib.gs_last_error().decode()

    rc, msg = call(None, grads, cams)
    assert rc == invalid and "gs_render_backward_batch_cam" in msg and "null ctx" in msg
    rc, msg = call(fake_ctx, grads, None)
    assert rc == invalid and "grad_cams" in msg
    rc, msg = call(fake_ctx, [None] * 5, None)
    assert rc == invalid and "grad_cams" in msg
    for k in range(5):
        mixed = list(grads)
        mixed[k] = None
        rc, msg = call(fake_ctx, mixed, cams)
        assert rc == invalid and "all NULL or all non-NULL" in msg, k
        only = [None] * 5
        only[k] = 0x3000
        rc, msg = call(fake_ctx, only, cams)
        assert rc == invalid and "all NULL or all non-NULL" in msg, k
