"""Roofline of the frame's memory-bound stages on the C3 scene (2.4 M Gaussians, 1920x1080, RGB, forward + backward).

Builds the scene the way bench.py does (same generator, seed, view 0 and upstream gradient, through Splatter) and, in
one process:
  * times a ~1 GB device-to-device copy with CUDA events: the HBM bandwidth this card reaches (bytes read + written);
  * times the frame (median of --rounds rounds of --steps frames);
  * reads the per-stage device times (RenderContext.stage_ms, CUDA events recorded by the library) after every frame of
    a second pass of --rounds x --steps frames and takes the medians;
  * sets each memory-bound stage's bytes (formulas below, from the frame's N, M and M_eff) against its time and against
    the measured copy bandwidth.
With --trace DIR it instead runs one profiled frame (torch.profiler, CUDA activities) and prints every kernel, copy and
memset of the frame in stream order with its duration and the gap before it; the chrome trace is written to DIR.
The card's name, power limit and maximum SM clock are read in the same run and printed with the numbers.

  python examples/bench_frontend.py [--steps 20] [--rounds 5] [--trace DIR]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-gaussian-splatting_b200"))

import splatter  # noqa: E402
import synthetic as S  # noqa: E402

N, W, H = 2_400_000, 1920, 1080
STAGES = ("project", "depth_sort+scan+readback", "emit_keys", "tile_sort", "tile_ranges", "blend_fwd", "blend_bwd",
          "project_bwd")


def stage_bytes(n, m, m_eff):
    """Bytes each memory-bound stage has to move at the frame's N Gaussians, M tile instances and M_eff consumed
    instances (DESIGN.md §3).  The project row counts a whole 64-byte record per Gaussian (an upper bound: only binned
    Gaussians write one)."""
    return {
        # pos, rgb, opa, quat, scale read; record, count, depth key, culling mask written
        "project": (12 + 12 + 4 + 16 + 12) * n + (64 + 4 + 4 + 8) * n,
        # scan of the counts in id order, 32-bit stable depth sort (keys + ids), count gather + scan in depth order
        "depth_sort+scan+readback": 90 * n,
        # u16 tile key + u32 Gaussian id per instance written; perm, offsets and one 32-byte sector of the tile
        # rectangle gathered per Gaussian
        "emit_keys": 6 * m + 32 * n,
        # two onesweep passes, each reading and writing the (u16, u32) pairs
        "tile_sort": 6 * m * 2 * 2,
        # consumed 48-byte gradient rows, one row tag per instance, parameters + offsets + counts read; five gradient
        # arrays written
        "project_bwd": 48 * m_eff + 4 * m + 56 * n + 56 * n,
    }


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit, clk = (s.strip() for s in out.split(","))
    except Exception:  # noqa: BLE001 - report what torch knows
        name, limit, clk = torch.cuda.get_device_name(0), "unknown", "unknown"
    return name, limit, clk


def median(ts):
    return sorted(ts)[len(ts) // 2]


def copy_gbs(dev, nbytes=1 << 30, iters=20):
    """Device-to-device copy of nbytes: (read + written bytes) / time, median of iters timed copies."""
    src = torch.empty(nbytes // 4, dtype=torch.float32, device=dev).uniform_()
    dst = torch.empty_like(src)
    for _ in range(3):
        dst.copy_(src)
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        dst.copy_(src)
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ms = median(ts)
    del src, dst
    torch.cuda.empty_cache()
    return 2 * nbytes / (ms * 1e-3) / 1e9, ms


class Scene:
    """bench.py's C3 scene: seed 0, RGB, opacities in [0.05, 0.9], view 0, its fixed upstream gradient."""

    def __init__(self, dev):
        g = S.make_gaussians(N, W, H, 0, sh_dim=3, opa_range=(0.05, 0.9))
        views = [S.make_view(W, H, k) for k in range(8)]
        vd = [dict(width=v.width, height=v.height, focal_x=v.fx, focal_y=v.fy, rot=v.rot, tran=v.tran) for v in views]
        self.sp = splatter.Splatter.from_tensors(g, vd, device=dev, use_sh_coeff=False)
        self.params = list(self.sp.gaussian_3ds.parameters())
        self.go = S.make_grad_output(H, W, 0).to(dev)

    def step(self):
        for p in self.params:
            p.grad = None
        img = self.sp(0)
        img.backward(self.go)


def trace(sc, out_dir):
    from torch.profiler import ProfilerActivity, profile
    os.makedirs(out_dir, exist_ok=True)
    for _ in range(5):
        sc.step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        sc.step()
        torch.cuda.synchronize()
    path = os.path.join(out_dir, "frontend_frame.pt.trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        ev = json.load(f)["traceEvents"]
    gpu = sorted((e for e in ev if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")),
                 key=lambda e: e["ts"])
    print(f"{'start_us':>9} {'gap_us':>7} {'dur_us':>8}  name")
    t0 = gpu[0]["ts"] if gpu else 0.0
    end = t0
    for e in gpu:
        print(f"{e['ts'] - t0:9.1f} {e['ts'] - end:7.1f} {e['dur']:8.1f}  {e['name'][:150]}")
        end = max(end, e["ts"] + e["dur"])
    busy = sum(e["dur"] for e in gpu)
    print(f"frame span {end - t0:.1f} us, GPU busy {busy:.1f} us, idle {end - t0 - busy:.1f} us")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--trace", default=None, metavar="DIR", help="profile one frame instead; trace written to DIR")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    name, limit, clk = card()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print(f"card: {name}, power limit {limit}, max SM clock {clk}")
    gbs, copy_ms = copy_gbs(dev)
    sc = Scene(dev)
    if args.trace:
        trace(sc, args.trace)
        return

    for _ in range(5):                       # module loads, workspace growth
        sc.step()
    torch.cuda.synchronize()
    frame = []
    for _ in range(args.rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            sc.step()
        e1.record()
        torch.cuda.synchronize()
        frame.append(e0.elapsed_time(e1) / args.steps)

    sc.sp._rctx.set_timing(True)
    per_stage = {s: [] for s in STAGES}
    for _ in range(args.rounds * args.steps):
        sc.step()
        for s, v in zip(STAGES, sc.sp._rctx.stage_ms()):
            per_stage[s].append(v)
    sc.sp._rctx.set_timing(False)
    st = sc.sp.frame_stats()
    m, m_eff = int(st["n_instances"]), int(st.get("n_instances_eff_bwd", st["n_instances_eff"]))
    nb = stage_bytes(N, m, m_eff)

    res = {"card": name, "power_limit": limit, "max_sm_clock": clk,
           "workload": "C3: 2.4 M Gaussians, 1920x1080, RGB, forward+backward (bench.py's scene, view 0)",
           "copy": {"bytes": 1 << 30, "ms": round(copy_ms, 4), "GBps": round(gbs, 1)},
           "frame_ms_median": round(median(frame), 4), "frame_ms_all": [round(t, 4) for t in frame],
           "N": N, "M": m, "M_eff": m_eff, "stages": {}}
    print(f"copy bandwidth {gbs:.0f} GB/s (1 GiB D2D, read + write); frame {median(frame):.4f} ms "
          f"(rounds {', '.join(f'{t:.4f}' for t in frame)}); N {N}, M {m}, M_eff {m_eff}")
    print(f"{'stage':<26} {'ms':>7} {'MB':>7} {'GB/s':>7} {'of copy':>8} {'floor ms':>9}")
    for s in STAGES:
        ms = median(per_stage[s])
        row = {"ms": round(ms, 4)}
        if s in nb:
            b = nb[s]
            achieved = b / (ms * 1e-3) / 1e9
            row.update({"MB": round(b / 1e6, 1), "GBps": round(achieved, 1), "share_of_copy": round(achieved / gbs, 3),
                        "floor_ms": round(b / (gbs * 1e9) * 1e3, 4)})
            print(f"{s:<26} {ms:7.4f} {b / 1e6:7.1f} {achieved:7.0f} {achieved / gbs:8.1%} {row['floor_ms']:9.4f}")
        else:
            print(f"{s:<26} {ms:7.4f}")
        res["stages"][s] = row
    print(json.dumps(res))


if __name__ == "__main__":
    main()
