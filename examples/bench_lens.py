"""Cost of camera lenses on the fused frame path (gs_ctx_set_lens) on the C3 scene (2.4 M Gaussians, 1920x1080).

Forward + backward of one frame (render_frame_final) for RGB and per-Gaussian SH of degree 3, with no lens, an
off-centre pinhole (principal point only), OPENCV with mild k1 / k2 and FISHEYE with COLMAP-like coefficients, the
variants alternated in one process.  Per variant: the frame time, the projection forward and backward stages
(stage_ms[0] and stage_ms[7], the only stages a lens touches), and M / M_eff, since a distortion changes what is
binned.

Prints the card name and power limit read in the same run, then one JSON line.

  python examples/bench_lens.py [--steps 20] [--rounds 5]
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
LENSES = {
    "none": None,
    "pinhole_offset": (gaussian.LENS_PINHOLE, [W / 2 + 7.5, H / 2 - 4.25, 0.0, 0.0, 0.0, 0.0]),
    "opencv": (gaussian.LENS_OPENCV, [W / 2 + 3.0, H / 2 + 2.0, -0.08, 0.02, 0.0005, -0.0003]),
    "fisheye": (gaussian.LENS_FISHEYE, [W / 2 - 2.0, H / 2 + 1.0, 0.03, -0.006, 0.001, -0.0002]),
}


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
    go = ((torch.rand(H, W, 3, generator=torch.Generator().manual_seed(1)) * 2 - 1) / (H * W)).to(dev)
    variants = {}
    for colour, dim in (("rgb", 3), ("sh3", 48)):
        g = S.make_gaussians(n, W, H, 0, sh_dim=dim)
        params = {k: t.to(dev).requires_grad_(True) for k, t in g.items()}
        for lens, spec in LENSES.items():
            rc = gaussian.RenderContext()
            rc.set_sh_eval(renderer.SH_EVAL["gaussian"])
            if spec is not None:
                rc.set_lens([spec[0]], torch.tensor([spec[1]], dtype=torch.float32))
            variants[f"{colour}_{lens}"] = (rc, params)

    def frame(label):
        rc, params = variants[label]
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
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                frame(label)
            e1.record()
            torch.cuda.synchronize()
            times[label].append(e0.elapsed_time(e1) / args.steps)
    for label in variants:
        rc = variants[label][0]
        # the stage times from frames of their own, timed by the context's events (a separate pass: the events add
        # host work to the timed loop above)
        rc.set_timing(True)
        fwd, bwd = [], []
        for _ in range(args.rounds):
            frame(label)
            sm = rc.stage_ms()
            fwd.append(sm[0])
            bwd.append(sm[7])
        rc.set_timing(False)
        st = rc.stats()
        res[label] = {"frame_ms_median": round(median(times[label]), 4),
                      "frame_ms_all": [round(t, 4) for t in times[label]],
                      "project_fwd_ms_median": round(median(fwd), 4), "project_bwd_ms_median": round(median(bwd), 4),
                      "M": st["n_instances"], "M_eff": st["n_instances_eff"]}
    print(f"card: {name}, power limit {limit}")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
