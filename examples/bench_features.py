"""Cost of the feature maps (renderer.render_frame_feat) on the C3 scene (2.4 M Gaussians) at 1920x1080.

Times forward + backward of one frame for RGB colour and per-Gaussian SH of degree 3, each as the aux frame without
features (render_frame_aux) and with F = 8, 16 and 32 features, the backward taking an image gradient and (with
features) a feature-map gradient.  The variants are alternated in one process so that they share the card's state;
medians of `rounds` rounds of `steps` frames.  Afterwards it reads the per-stage device times of each variant (CUDA
events, a separate pass): blend_fwd / blend_bwd are the blend kernels, project_bwd the projection backward plus the
feature segment sum.  Prints the card name and power limit read in the same run, then one JSON line.

  python examples/bench_features.py [--steps 20] [--rounds 5]
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
WIDTHS = (0, 8, 16, 32)   # 0: the aux frame without features
COLOURS = {"rgb": (3, "pixel"), "sh48": (48, "gaussian")}
# gs_frame_stage_ms indices
STAGES = {"project_fwd": 0, "sort_scan": 1, "emit": 2, "tile_sort": 3, "ranges": 4, "blend_fwd": 5, "blend_bwd": 6,
          "project_bwd": 7}


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
    w, h = 1920, 1080
    v = S.make_view(w, h, 0)
    go = ((torch.rand(h, w, 3, generator=torch.Generator().manual_seed(1)) * 2 - 1) / (h * w)).to(dev)
    gen = torch.Generator().manual_seed(2)
    gfeat = {f: ((torch.rand(h, w, f, generator=gen) * 2 - 1) / (h * w)).to(dev) for f in WIDTHS if f}
    feats = {f: (torch.rand(n, f, generator=gen) * 2 - 1).to(dev).requires_grad_(True) for f in WIDTHS if f}
    variants, scenes = {}, {}
    for colour, (sh_dim, sh_eval) in COLOURS.items():
        scenes[colour] = {k: t.to(dev).requires_grad_(True)
                          for k, t in S.make_gaussians(n, w, h, 0, sh_dim).items()}
        for f in WIDTHS:
            rctx = gaussian.RenderContext()
            rctx.set_sh_eval(renderer.SH_EVAL[sh_eval])
            variants[f"{colour}_{'aux' if f == 0 else f'f{f}'}"] = (rctx, colour, f,
                                                                    (w, h, v.fx, v.fy, v.rot, v.tran, v.near, 0.05,
                                                                     "abs"))

    def frame(label):
        rctx, colour, f, cam = variants[label]
        params = scenes[colour]
        for p in list(params.values()) + list(feats.values()):
            p.grad = None
        if f == 0:
            img, _, _, _ = renderer.render_frame_aux(rctx, *(params[k] for k in NAMES), *cam, background=(1, 1, 1))
            img.backward(go)
        else:
            img, fm, _, _, _ = renderer.render_frame_feat(rctx, *(params[k] for k in NAMES), feats[f], *cam,
                                                          background=(1, 1, 1))
            torch.autograd.backward([img, fm], [go, gfeat[f]])

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
    for rctx, _, _, _ in variants.values():
        rctx.set_timing(True)
    for _ in range(args.rounds):
        for label, (rctx, _, _, _) in variants.items():
            frame(label)
            ms = rctx.stage_ms()
            for s, i in STAGES.items():
                stages[label][s].append(ms[i])

    res = {"card": name, "power_limit": limit,
           "workload": "C3 scene 1920x1080, forward+backward, image + feature gradient", "steps": args.steps,
           "rounds": args.rounds}
    for label in variants:
        r = {"frame_ms_median": round(median(times[label]), 4), "frame_ms_all": [round(t, 4) for t in times[label]]}
        for s in STAGES:
            r[f"{s}_ms_median"] = round(median(stages[label][s]), 4)
        st = variants[label][0].stats()
        r["n_instances"], r["n_instances_eff"] = st["n_instances"], st["n_instances_eff"]
        res[label] = r
    for colour in COLOURS:
        for f in WIDTHS[1:]:
            res[f"{colour}_f{f}_over_aux"] = round(res[f"{colour}_f{f}"]["frame_ms_median"] /
                                                  res[f"{colour}_aux"]["frame_ms_median"], 4)
    print(f"card: {name}, power limit {limit}")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
