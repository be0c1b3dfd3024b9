"""SURVEY.md §8 f-1: the reference's own train.py (oracle/_ref/train.py, the
byte-identical copy oracle/build_ref.py makes) runs UNCHANGED through 3d-gaussian-splatting_b200/dp_launch.py
on a synthetic COLMAP dataset:
  * on OUR splatter.py (fused frame path, fused SSIM through shims/torchmetrics, fused flat Adam);
  * on the REFERENCE's splatter.py + renderer.py with only the `gaussian` extension module being ours
    (the legacy per-stage C++ boundary, SURVEY.md §8b);
  * under torchrun with 2 ranks (view sharding + gradient exchange + summed densification statistics),
    when the box has 2 GPUs.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import synthetic as S

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAUNCH = os.path.join(ROOT, "3d-gaussian-splatting_b200", "dp_launch.py")
TRAIN_PY = os.path.join(ROOT, "oracle", "_ref", "train.py")


def make_colmap_dataset(root, cuda, n_teacher=4000, w=160, h=96, n_views=8, downsample=1):
    """<root>/sparse/0/{cameras,images,points3D}.bin + <root>/images_<downsample>/v*.png rendered from a
    teacher scene with our own renderer (the COLMAP intrinsics are those of the full-resolution camera)."""
    import cv2
    import colmap_io as C
    import splatter
    teacher = S.make_gaussians(n_teacher, w, h, 0)
    views = [S.make_view(w, h, k) for k in range(n_views)]
    vd = [dict(width=v.width, height=v.height, focal_x=v.fx, focal_y=v.fy, rot=v.rot, tran=v.tran) for v in views]
    sp_t = splatter.Splatter.from_tensors(teacher, vd, device=cuda)
    sparse, imgdir = os.path.join(root, "sparse", "0"), os.path.join(root, f"images_{downsample}")
    os.makedirs(sparse), os.makedirs(imgdir)
    cams = {1: C.Camera(1, "PINHOLE", w * downsample, h * downsample,
                        np.array([views[0].fx * downsample, views[0].fy * downsample, w * downsample / 2, h * downsample / 2]))}
    imgs = {}
    for k, v in enumerate(views):
        with torch.no_grad():
            im = (sp_t(k).clamp(0, 1) * 255).byte().cpu().numpy()
        cv2.imwrite(os.path.join(imgdir, f"v{k}.png"), im[..., ::-1])
        imgs[k + 1] = C.Image(k + 1, C.rotmat_to_qvec(v.rot.numpy()), v.tran.numpy(), 1, f"v{k}.png")
    pts = {i: C.Point3D(i, teacher["pos"][i].numpy(), (torch.sigmoid(teacher["rgb"][i]) * 255).byte().numpy(), 0.0)
           for i in range(0, n_teacher, 2)}
    C.write_cameras_binary(os.path.join(sparse, "cameras.bin"), cams)
    C.write_images_binary(os.path.join(sparse, "images.bin"), imgs)
    C.write_points3d_binary(os.path.join(sparse, "points3D.bin"), pts)
    return n_teacher // 2


def _run(cmd, cwd, timeout=600):
    env = dict(os.environ, PYTHONUNBUFFERED="1")
    r = subprocess.run(cmd, cwd=cwd, env=env, capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])
    return r


TRAIN_ARGS = ["--n_iters", "61", "--n_iters_warmup", "10", "--n_iters_test", "30", "--n_save_train_img", "30",
              "--render_downsample_start", "1", "--render_downsample", "1", "--scale_init_value", "0.5",
              "--opa_init_value", "0.3", "--lr", "0.003", "--ssim_weight", "0.1", "--n_history_track", "20",
              "--grad_accum_method", "mean", "--grad_accum_iters", "20", "--n_adaptive_control", "1000"]


def _check_outputs(exp, n_points):
    ckpt = torch.load(os.path.join(exp, "ckpt.pth"), map_location="cpu", weights_only=False)
    assert sorted(ckpt) == ["opa", "pos", "quat", "rgb", "scale"]                  # train.py:283-291
    assert ckpt["pos"].shape == (n_points, 3) and all(bool(torch.isfinite(v).all()) for v in ckpt.values())
    assert os.path.exists(os.path.join(exp, "imgs", "train_0.png")) and os.path.exists(os.path.join(exp, "imgs", "train_60.png"))
    assert any(f.startswith("iter_60_") for f in os.listdir(os.path.join(exp, "test_imgs")))
    return ckpt


@pytest.mark.parametrize("which", ["ours", "reference"])
def test_reference_train_py_runs_unchanged(gs, cuda, tmp_path, which):
    if not os.path.exists(TRAIN_PY):
        pytest.skip("oracle/_ref/train.py not present (oracle/build_ref.py copies it where /root/reference exists)")
    data = str(tmp_path / "data")
    n_points = make_colmap_dataset(data, cuda)
    exp = str(tmp_path / f"exp_{which}")
    r = _run([sys.executable, LAUNCH, "--train-py", TRAIN_PY, "--splatter", which, "--", "--data", data, "--exp", exp] + TRAIN_ARGS, str(tmp_path))
    ckpt = _check_outputs(exp, n_points)
    # the run really optimised: PSNR on the test split rose between iteration 0 and 60
    psnrs = [float(l.split(":")[1]) for l in r.stdout.splitlines() if l.startswith("TEST SPLIT PSNR")]
    assert len(psnrs) >= 3 and psnrs[-1] > psnrs[0] + 0.5, psnrs
    # a checkpoint written by train.py loads back through the reference's --ckpt path (splatter.py:417-424)
    import splatter
    v = S.make_view(160, 96, 0)
    sp = splatter.Splatter(ckpt, [dict(width=160, height=96, focal_x=v.fx, focal_y=v.fy, rot=v.rot, tran=v.tran)],
                           device=cuda, tile_culling_prob_thresh=0.05)
    assert bool(torch.isfinite(sp(0)).all())


def test_reference_train_py_data_parallel(gs, cuda, tmp_path):
    """2 (4, 8: GS_TEST_TRAIN_WORLD) ranks under torchrun: different views per rank, averaged gradient bucket,
    identical replicas (the multi-view training configuration at test size)."""
    world = int(os.environ.get("GS_TEST_TRAIN_WORLD", "2"))          # 2 (default), 4 or 8
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    if not os.path.exists(TRAIN_PY):
        pytest.skip("oracle/_ref/train.py not present")
    data = str(tmp_path / "data")
    n_points = make_colmap_dataset(data, cuda)
    exp = str(tmp_path / "exp_dp")
    port = 29500 + (os.getpid() % 500)
    # train.py only densifies after iteration 600 (train.py:88-90): run to 701 so that one prune / clone /
    # split round (with torch-sampled split positions) happens on both ranks before the final checkpoint
    args = list(TRAIN_ARGS)
    for name, val in (("--n_iters", "702"), ("--n_iters_test", "701"), ("--n_save_train_img", "701"),
                      ("--n_adaptive_control", "100")):
        args[args.index(name) + 1] = val
    _run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr",
          "127.0.0.1", "--master-port", str(port), LAUNCH, "--train-py", TRAIN_PY, "--", "--data", data, "--exp", exp, "--use_clone", "1",
          "--grad_thresh", "0.00001"] + args, str(tmp_path), timeout=900)
    c0 = torch.load(os.path.join(exp, "ckpt.pth"), map_location="cpu", weights_only=False)
    for r in range(1, world):
        c1 = torch.load(os.path.join(exp + f"_rank{r}", "ckpt.pth"), map_location="cpu", weights_only=False)
        for k in c0:
            assert c0[k].shape == c1[k].shape and torch.equal(c0[k], c1[k]), (r, k)   # replicas stayed bit-identical
    assert all(bool(torch.isfinite(v).all()) for v in c0.values())
