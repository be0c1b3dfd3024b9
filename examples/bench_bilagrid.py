"""Cost of the bilateral-grid slice (gs_bilagrid_slice_fwd / _bwd) at 1920x1080 with 16x16x8 grids, in one process:

  fwd_ms / bwd_ms            the kernels, B = 1 and B = 8 (backward: image and grid gradients), CUDA events over
                             --steps calls after warm-up, median of --rounds rounds
  torch_fwd_ms / torch_bwd_ms  the torch restatement (grid_sample + affine; its autograd backward) at the same shapes
  hbm_share_fwd / _bwd       algorithmic bytes (image in + out: 24 B/px forward; image, grad_out in, grad_image out:
                             36 B/px backward; the grid rows once) over kernel time, as a share of 3.35 TB/s (the
                             H100 SXM data-sheet figure, not a measurement)
  step_ms                    a C3 RGB training step (2.4 M Gaussians, 1920x1080: frame forward + backward, L1, fused
                             Adam) without and with --bilagrid's slice, TV term and grid Adam

Prints the card name and power limit read in the same run, then one JSON line.

  python examples/bench_bilagrid.py [--steps 50] [--rounds 5]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-gaussian-splatting_b200"))
sys.path.insert(0, os.path.join(ROOT, "examples"))

import bilagrid  # noqa: E402
import gaussian  # noqa: E402
import optim  # noqa: E402
import splatter  # noqa: E402
import synthetic as S  # noqa: E402
from bench_surfel import card, median  # noqa: E402

W, H, N, V = 1920, 1080, 2_400_000, 8
SHAPE = (16, 16, 8)
HBM = 3.35e12


def timed(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def torch_slice(image, grids, ids):
    """grid_sample + affine; z as the kernel computes it is not reproduced bit for bit here (timing only)"""
    b, h, w, _ = image.shape
    lum = 0.299 * image[..., 0] + 0.587 * image[..., 1] + 0.114 * image[..., 2]
    xs = ((torch.arange(w, device=image.device) + 0.5) / w).expand(b, h, w)
    ys = ((torch.arange(h, device=image.device) + 0.5) / h)[:, None].expand(b, h, w)
    coords = torch.stack([xs, ys, lum.clamp(0, 1)], dim=-1)[:, None] * 2 - 1
    A = torch.nn.functional.grid_sample(grids.permute(0, 4, 3, 1, 2)[ids], coords, mode="bilinear",
                                        padding_mode="border", align_corners=True)[:, :, 0].permute(0, 2, 3, 1)
    M = A.reshape(b, h, w, 3, 4)
    return (M[..., :3] * image[..., None, :]).sum(-1) + M[..., 3]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    name, limit = card()
    dev = torch.device("cuda", 0)
    res = {"card": name, "power_limit": limit, "width": W, "height": H, "grid": list(SHAPE), "steps": args.steps}
    gen = torch.Generator().manual_seed(0)
    grids = (bilagrid.identity_grids(V, SHAPE, dev) + 0.05 * torch.randn(V, *SHAPE, 12, generator=gen).to(dev))
    row_bytes = SHAPE[0] * SHAPE[1] * SHAPE[2] * 12 * 4
    for b in (1, 8):
        ids = list(range(b))
        img = torch.rand(b, H, W, 3, generator=gen).to(dev)
        go = torch.randn(b, H, W, 3, generator=gen).to(dev)
        px = b * H * W

        def fwd():
            gaussian.bilagrid_slice(img, grids, ids)

        def bwd():
            gaussian.bilagrid_slice_backward(img, grids, ids, go, True, True)

        gt = grids.clone().requires_grad_(True)
        it = img.clone().requires_grad_(True)
        idt = torch.tensor(ids, device=dev)

        def tfwd():
            with torch.no_grad():
                torch_slice(img, grids, idt)

        def tbwd():
            gt.grad = None
            it.grad = None
            torch_slice(it, gt, idt).backward(go)

        for f in (fwd, bwd, tfwd, tbwd):                              # warm-up every shape
            timed(f, 3)
        r = {}
        for key, f, steps in (("fwd_ms", fwd, args.steps), ("bwd_ms", bwd, args.steps),
                              ("torch_fwd_ms", tfwd, max(args.steps // 5, 3)),
                              ("torch_bwd_ms", tbwd, max(args.steps // 5, 3))):
            r[key] = median([timed(f, steps) for _ in range(args.rounds)])
        fwd_bytes = 24 * px + b * row_bytes
        bwd_bytes = 36 * px + b * row_bytes * 2                     # grid rows read, gradient rows written
        r["bytes_fwd"], r["bytes_bwd"] = fwd_bytes, bwd_bytes
        r["hbm_share_fwd"] = fwd_bytes / HBM / (r["fwd_ms"] * 1e-3)
        r["hbm_share_bwd"] = bwd_bytes / HBM / (r["bwd_ms"] * 1e-3)
        r["roof_fwd_us"], r["roof_bwd_us"] = fwd_bytes / HBM * 1e6, bwd_bytes / HBM * 1e6
        res[f"B{b}"] = r
        del img, go, gt, it
        torch.cuda.empty_cache()

    # a C3 RGB training step, without and with the grids
    g = S.make_gaussians(N, W, H, 0)
    vs = [S.make_view(W, H, k) for k in range(V)]
    views = [dict(width=v.width, height=v.height, focal_x=v.fx, focal_y=v.fy, rot=v.rot, tran=v.tran) for v in vs]
    gts = [torch.rand(H, W, 3, generator=gen).to(dev) for _ in range(V)]
    for use in (False, True):
        sp = splatter.Splatter.from_tensors(g, views, device=dev, near=vs[0].near)
        gp = sp.gaussian_3ds
        opt = optim.FlatAdam([{"params": gp.opa, "lr": 0.03}, {"params": gp.rgb, "lr": 0.03},
                              {"params": gp.pos, "lr": 0.003}, {"params": gp.scale, "lr": 0.003},
                              {"params": gp.quat, "lr": 0.003}], betas=(0.9, 0.99))
        bg = bilagrid.BilateralGrids(V, SHAPE, device=dev) if use else None
        bopt = torch.optim.Adam(bg.parameters(), lr=2e-3, eps=1e-15) if use else None
        k = [0]

        def step():
            v = k[0] % V
            k[0] += 1
            opt.zero_grad(set_to_none=True)
            img = sp(v)
            if use:
                bopt.zero_grad(set_to_none=True)
                img = bg(img, v)
            loss = (img - gts[v]).abs().mean()
            if use:
                loss = loss + 10.0 * bg.tv_loss([v])
            loss.backward()
            opt.step()
            if use:
                bopt.step()

        timed(step, 5)
        res["step_ms_bilagrid" if use else "step_ms"] = median([timed(step, max(args.steps // 5, 5))
                                                                for _ in range(args.rounds)])
        del sp, opt, bg, bopt
        torch.cuda.empty_cache()
    print(f"card: {name}, power limit {limit}")
    for b in (1, 8):
        r = res[f"B{b}"]
        print(f"B={b}: slice fwd {r['fwd_ms'] * 1e3:.1f} us ({r['hbm_share_fwd'] * 100:.0f} % of the HBM roof "
              f"{r['roof_fwd_us']:.1f} us), bwd {r['bwd_ms'] * 1e3:.1f} us ({r['hbm_share_bwd'] * 100:.0f} % of "
              f"{r['roof_bwd_us']:.1f} us); torch fwd {r['torch_fwd_ms'] * 1e3:.1f} us, bwd {r['torch_bwd_ms'] * 1e3:.1f} us")
    print(f"C3 RGB training step: {res['step_ms']:.3f} ms, with --bilagrid {res['step_ms_bilagrid']:.3f} ms")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
