"""Cost of camera pose gradients (renderer.render_frame_cam, gs_render_backward_cam) on the C3 frame (2.4 M Gaussians,
1080p).

Times forward + backward of one frame for four variants, for RGB and for per-Gaussian SH of degree 3, all alternated in
one process so that they share the card's state:
  frame     render_frame_final, image gradient (the plain frame, for reference)
  aux       render_frame_aux over a background, image + depth gradients, parameter gradients
  aux_cam   render_frame_cam, the same plus dL/drot and dL/dtran (one more kernel, one 48-byte host read)
  cam_only  render_frame_cam with the scene frozen: camera gradients only (tracking)
Afterwards it reads the per-stage device times of each variant (CUDA events, a separate pass): blend backward and
projection backward (which covers the camera-gradient kernels).  Prints the card name and power limit read in the
same run, then one JSON line.

  python examples/bench_pose_grad.py [--steps 20] [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-gaussian-splatting_b200"))

import renderer  # noqa: E402
import synthetic as S  # noqa: E402
import gaussian  # noqa: E402

NAMES = ("pos", "rgb", "opa", "quat", "scale")
# gs_frame_stage_ms indices
STAGES = {"blend_bwd": 6, "project_bwd": 7}
BG = (0.2, 0.5, 0.9)


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    name, limit = card()
    dev = torch.device("cuda", 0)
    n, w, h = 2_400_000, 1920, 1080
    v = S.make_view(w, h, 0)
    intr = (w, h, v.fx, v.fy)
    rot, tran = v.rot.to(dev).requires_grad_(True), v.tran.to(dev).requires_grad_(True)
    gen = torch.Generator().manual_seed(1)
    go = ((torch.rand(h, w, 3, generator=gen) * 2 - 1) / (h * w)).to(dev)
    gd = ((torch.rand(h, w, generator=gen) * 2 - 1) / (h * w) * 1e-2).to(dev)

    scenes = {}
    for colour, d, mode in (("rgb", 3, "pixel"), ("sh48_gaussian", 48, "gaussian")):
        # the generator draws colours last: both colours have the same geometry
        scenes[colour] = (S.make_gaussians(n, w, h, 0, sh_dim=d), mode)
    variants = {}
    for colour, (g, mode) in scenes.items():
        for kind in ("frame", "aux", "aux_cam", "cam_only"):
            params = {k: t.to(dev).requires_grad_(kind != "cam_only") for k, t in g.items()}
            rctx = gaussian.RenderContext()
            rctx.set_sh_eval(renderer.SH_EVAL[mode])
            variants[f"{colour}_{kind}"] = (rctx, params, kind)

    def frame(label):
        rctx, params, kind = variants[label]
        for p in list(params.values()) + [rot, tran]:
            p.grad = None
        ps = [params[k] for k in NAMES]
        if kind == "frame":
            img, _ = renderer.render_frame_final(rctx, *ps, *intr, v.rot, v.tran, v.near, 0.05, "abs")
            img.backward(go)
            return
        fn = renderer.render_frame_aux if kind == "aux" else renderer.render_frame_cam
        r, t = (v.rot, v.tran) if kind == "aux" else (rot, tran)
        img, dep, _, _ = fn(rctx, *ps, *intr, r, t, v.near, 0.05, "abs", background=BG)
        torch.autograd.backward([img, dep], [go, gd])

    for label in variants:                 # warm-up: module loads, workspace growth
        for _ in range(3):
            frame(label)
    torch.cuda.synchronize()
    times = {k: [] for k in variants}
    for _ in range(args.rounds):
        for label in variants:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                frame(label)
            e1.record()
            torch.cuda.synchronize()
            times[label].append(e0.elapsed_time(e1) / args.steps)

    stages = {k: {s: [] for s in STAGES} for k in variants}
    for rctx, _, _ in variants.values():
        rctx.set_timing(True)
    for _ in range(args.rounds):
        for label, (rctx, _, _) in variants.items():
            frame(label)
            ms = rctx.stage_ms()
            for s, i in STAGES.items():
                stages[label][s].append(ms[i])

    res = {"card": name, "power_limit": limit, "workload": "C3 forward+backward", "steps": args.steps,
           "rounds": args.rounds}
    for label in variants:
        r = {"frame_ms_median": round(median(times[label]), 4), "frame_ms_all": [round(t, 4) for t in times[label]]}
        for s in STAGES:
            r[f"{s}_ms_median"] = round(median(stages[label][s]), 4)
        res[label] = r
    for colour in scenes:
        base = res[f"{colour}_aux"]["frame_ms_median"]
        for kind in ("aux_cam", "cam_only"):
            res[f"{colour}_{kind}_minus_aux_ms"] = round(res[f"{colour}_{kind}"]["frame_ms_median"] - base, 4)
    print(f"card: {name}, power limit {limit}")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
