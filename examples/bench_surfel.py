"""Cost of 2D Gaussian surfels (gs_render_forward_surfel) against 3D Gaussians on the C3 scene (2.4 M Gaussians,
1920x1080): forward + backward of one frame for RGB and per-Gaussian SH of degree 3,

  gaussian       render_frame_final                        surfel       render_frame_surfel(maps=False)
  gaussian_maps  render_frame_aux (depth, alpha gradients)  surfel_maps  render_frame_surfel (all five map gradients)

the variants alternated in one process.  Per variant: the frame time, the eight stage times (a pass of their own) and
M / M_eff.  The same parameter tensors serve both primitives (the surfel uses the first two scale axes).

Prints the card name and power limit read in the same run, then one JSON line.

  python examples/bench_surfel.py [--steps 20] [--rounds 5]
"""
import argparse
import json
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
W, H = 1920, 1080
STAGES = ("project", "scan", "emit", "tile_sort", "pack", "blend_fwd", "blend_bwd", "project_bwd")


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
    n = 2_400_000
    res = {"card": name, "power_limit": limit, "steps": args.steps, "rounds": args.rounds}
    v0 = S.make_view(W, H, 0)
    cam = (W, H, v0.fx, v0.fy, v0.rot, v0.tran, v0.near, 0.05, "abs")
    gen = torch.Generator().manual_seed(1)
    go = ((torch.rand(H, W, 3, generator=gen) * 2 - 1) / (H * W)).to(dev)
    gm = {k: ((torch.rand(H, W, *((3,) if k == "normal" else ()), generator=gen) * 2 - 1) / (H * W)).to(dev)
          for k in renderer.SURFEL_MAPS}
    variants = {}
    for colour, dim in (("rgb", 3), ("sh3", 48)):
        g = S.make_gaussians(n, W, H, 0, sh_dim=dim)
        params = {k: t.to(dev).requires_grad_(True) for k, t in g.items()}
        for kind in ("gaussian", "gaussian_maps", "surfel", "surfel_maps"):
            rc = gaussian.RenderContext()
            rc.set_sh_eval(renderer.SH_EVAL["gaussian"])
            variants[f"{colour}_{kind}"] = (rc, params, kind)

    def frame(label):
        rc, params, kind = variants[label]
        for p in params.values():
            p.grad = None
        P = [params[k] for k in NAMES]
        if kind == "gaussian":
            img, _ = renderer.render_frame_final(rc, *P, *cam)
            img.backward(go)
        elif kind == "gaussian_maps":
            img, depth, alpha, _ = renderer.render_frame_aux(rc, *P, *cam, background=[0.1, 0.1, 0.1], final=True)
            torch.autograd.backward([img, depth, alpha], [go, gm["depth"], gm["alpha"]])
        else:
            maps = kind == "surfel_maps"
            img, mp, _ = renderer.render_frame_surfel(rc, *P, *cam, background=[0.1, 0.1, 0.1], final=True, maps=maps)
            outs, grads = [img], [go]
            for k in mp:
                outs.append(mp[k])
                grads.append(gm[k])
            torch.autograd.backward(outs, grads)

    for label in variants:
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
    for label in variants:
        rc = variants[label][0]
        rc.set_timing(True)                      # stage times from frames of their own
        stages = []
        for _ in range(args.rounds):
            frame(label)
            stages.append(rc.stage_ms())
        rc.set_timing(False)
        st = rc.stats()
        res[label] = {"frame_ms_median": round(median(times[label]), 4),
                      "frame_ms_all": [round(t, 4) for t in times[label]],
                      "stage_ms_median": {s: round(median([x[i] for x in stages]), 4) for i, s in enumerate(STAGES)},
                      "M": st["n_instances"], "M_eff": st["n_instances_eff"]}
    print(f"card: {name}, power limit {limit}")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
