"""Cost of Mip-Splatting's 3-D filter on the C3 scene (2.4 M Gaussians).

1. The sampling-rate filter (gaussian.filter3d_compute, two kernels) with 50 and 300 views, against a torch
   restatement of Mip-Splatting's per-camera loop (the same rule: N-sized torch ops per view, max / min at the end).
2. Forward + backward of one frame (render_frame_final) with the 2-D antialias filter alone and with the 3-D filter
   too, for RGB and per-Gaussian SH of degree 3, at 1920x1080 and at twice its focal length (the zoom-in case), the
   variants alternated in one process.

Prints the card name and power limit read in the same run, then one JSON line.

  python examples/bench_filter3d.py [--steps 20] [--rounds 5]
"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-gaussian-splatting_b200"))

import gaussian  # noqa: E402
import renderer  # noqa: E402
import synthetic as S  # noqa: E402

NAMES = ("pos", "rgb", "opa", "quat", "scale")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (s.strip() for s in out.split(","))
    except Exception:  # noqa: BLE001 - report what torch knows
        name, limit = torch.cuda.get_device_name(0), "unknown"
    return name, limit


def median(ts):
    return sorted(ts)[len(ts) // 2]


def views_of(k, w=1920, h=1080):
    out = []
    for i in range(k):
        v = S.make_view(w, h, i % 8)
        s = 0.6 + 0.8 * ((i * 0.618) % 1.0)
        out.append(S.View(w, h, v.fx, v.fy, v.rot, v.tran * s, v.near))
    return out


def torch_loop(pos, views, margin=0.15, variance=0.2):
    """Mip-Splatting's compute_3D_filter restated with the rule of gs_filter3d_compute (max fx / z over the views that
    see a Gaussian, the smallest seen rate for the others)."""
    nu = torch.zeros(pos.shape[0], device=pos.device)
    for v in views:
        R = torch.as_tensor(v.rot, device=pos.device, dtype=torch.float32)
        t = torch.as_tensor(v.tran, device=pos.device, dtype=torch.float32)
        pc = pos @ R.T + t
        x, y, z = pc.unbind(1)
        u = v.fx * x / z + v.width / 2
        w = v.fy * y / z + v.height / 2
        seen = (z > v.near) & (u >= -margin * v.width) & (u <= (1 + margin) * v.width) & \
               (w >= -margin * v.height) & (w <= (1 + margin) * v.height)
        nu = torch.maximum(nu, torch.where(seen, v.fx / z, torch.zeros_like(z)))
    seen = nu > 0
    nu = torch.where(seen, nu, nu[seen].min())
    return math.sqrt(variance) / nu


def timed(fn, steps, rounds):
    ts = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) / steps)
    return ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    name, limit = card()
    dev = torch.device("cuda", 0)
    n = 2_400_000
    res = {"card": name, "power_limit": limit, "steps": args.steps, "rounds": args.rounds}

    # 1. the sampling-rate filter
    pos = S.make_gaussians(n, 1920, 1080, 0)["pos"].to(dev)
    rctx = gaussian.RenderContext()
    for k in (50, 300):
        vs = views_of(k)
        size = torch.tensor([[v.width, v.height] for v in vs])
        focal = torch.tensor([[v.fx, v.fy] for v in vs], dtype=torch.float32)
        rot = torch.stack([torch.as_tensor(v.rot, dtype=torch.float32) for v in vs])
        tran = torch.stack([torch.as_tensor(v.tran, dtype=torch.float32) for v in vs])
        out = torch.empty(n, device=dev)

        def kernel():
            gaussian.filter3d_compute(rctx, pos, size, focal, rot, tran, 0.3, 0.15, 0.2, out)

        kernel()
        ref = torch_loop(pos, vs)
        torch.cuda.synchronize()
        rel = float(((out - ref).abs() / ref.abs()).max())
        tk = timed(kernel, args.steps, args.rounds)
        tt = timed(lambda: torch_loop(pos, vs), max(1, args.steps // 10), args.rounds)
        res[f"filter3d_{k}views"] = {"kernel_ms_median": round(median(tk), 4), "torch_loop_ms_median": round(median(tt), 3),
                                     "speedup": round(median(tt) / median(tk), 1), "max_rel_diff_vs_torch_fp32": rel}

    # 2. frames: antialias alone vs antialias + 3-D filter
    variants = {}
    for colour, dim in (("rgb", 3), ("sh3", 48)):
        g = S.make_gaussians(n, 1920, 1080, 0, sh_dim=dim)
        params = {k: t.to(dev).requires_grad_(True) for k, t in g.items()}
        v0 = S.make_view(1920, 1080, 0)
        f3 = torch.empty(n, device=dev)
        ctx0 = gaussian.RenderContext()
        gaussian.filter3d_compute(ctx0, params["pos"].detach(), torch.tensor([[1920, 1080]]),
                                  torch.tensor([[v0.fx, v0.fy]], dtype=torch.float32),
                                  torch.as_tensor(v0.rot, dtype=torch.float32)[None],
                                  torch.as_tensor(v0.tran, dtype=torch.float32)[None], v0.near, 0.15, 0.2, f3)
        for zoom in (1, 2):
            go = ((torch.rand(1080, 1920, 3, generator=torch.Generator().manual_seed(1)) * 2 - 1) / (1080 * 1920)).to(dev)
            cam = (1920, 1080, v0.fx * zoom, v0.fy * zoom, v0.rot, v0.tran, v0.near, 0.05, "abs")
            for with3d in (False, True):
                rc = gaussian.RenderContext()
                rc.set_sh_eval(renderer.SH_EVAL["gaussian"])
                rc.set_filter2d(renderer.FILTER2D["antialias"], 0.1)
                if with3d:
                    rc.set_filter3d(f3)
                variants[f"{colour}_zoom{zoom}_{'aa+3d' if with3d else 'aa'}"] = (rc, params, cam, go)

    def frame(label):
        rc, params, cam, go = variants[label]
        for p in params.values():
            p.grad = None
        img, _ = renderer.render_frame_final(rc, *(params[k] for k in NAMES), *cam)
        img.backward(go)

    for label in variants:
        for _ in range(3):
            frame(label)
    torch.cuda.synchronize()
    times = {k: [] for k in variants}
    for _ in range(args.rounds):
        for label in variants:
            times[label] += timed(lambda: frame(label), args.steps, 1)
    for label in variants:
        st = variants[label][0].stats()
        res[label] = {"frame_ms_median": round(median(times[label]), 4),
                      "frame_ms_all": [round(t, 4) for t in times[label]], "n_instances": st["n_instances"]}
    for colour in ("rgb", "sh3"):
        for zoom in (1, 2):
            res[f"{colour}_zoom{zoom}_3d_over_aa"] = round(res[f"{colour}_zoom{zoom}_aa+3d"]["frame_ms_median"] /
                                                          res[f"{colour}_zoom{zoom}_aa"]["frame_ms_median"], 4)
    print(f"card: {name}, power limit {limit}")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
