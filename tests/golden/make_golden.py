"""Generates tests/golden/*.npz by running the REFERENCE's own CUDA build (oracle/_ref,
built by oracle/build_ref.py from the unmodified sources) on a GPU.

Run on a GPU:   python tests/golden/make_golden.py <output dir>
then copy the files into tests/golden/ and commit them.  Nothing of ours (kernels or
oracle arithmetic) produces the stored outputs; the oracle only prepares the sorted
per-instance INPUTS of the `draw` case, which are stored alongside.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
for p in ("3d-gaussian-splatting_b200", "oracle", "tests"):
    sys.path.insert(0, os.path.join(ROOT, p))

import golden_cases as GC  # noqa: E402
import ref_pipeline  # noqa: E402


def main(out_dir):
    os.makedirs(out_dir, exist_ok=True)
    dev = torch.device("cuda", 0)
    gref, rref = ref_pipeline.load_reference()
    assert gref is not None, "oracle/_ref is missing: run oracle/build_ref.py where /root/reference exists"
    cpu = lambda t: t.detach().cpu().numpy()

    # ---- project.npz : global_culling forward + backward -------------------------------
    pos, nq, ns, cam, go_pos, go_cov = GC.project_inputs()
    p = pos.to(dev).requires_grad_(True)
    q = nq.to(dev).requires_grad_(True)
    s = ns.to(dev).requires_grad_(True)
    rp, rc, m = rref.global_culling(p, q, s, cam.rot.to(dev), cam.tran.to(dev), cam.near, cam.half_w, cam.half_h)
    ((rp * go_pos.to(dev)).sum() + (rc * go_cov.to(dev)).sum()).backward()
    np.savez_compressed(os.path.join(out_dir, "project.npz"), res_pos=cpu(rp), res_cov=cpu(rc), mask=cpu(m),
                        grad_pos=cpu(p.grad), grad_quat=cpu(q.grad), grad_scale=cpu(s.grad))

    # ---- tiles.npz : calc_tile_list method 2 --------------------------------------------
    pos2, cov2, cam = GC.tiles_inputs()
    T = cam.ntx * cam.nty
    n = pos2.shape[0]
    cnt = torch.zeros(T, dtype=torch.int32, device=dev)
    lst = torch.full((T, n), -1, dtype=torch.int32, device=dev)
    cobj = gref.Gaussian3ds()
    cobj.pos, cobj.cov = pos2.to(dev), cov2.to(dev)
    cobj.rgb, cobj.opa = torch.zeros(n, 3, device=dev), torch.zeros(n, device=dev)
    tiles = gref.Tiles()
    tiles.top = tiles.bottom = tiles.left = tiles.right = torch.zeros(T, device=dev)
    gref.calc_tile_list(cobj, tiles, cnt, lst, 0.05, 2, cam.tile_lx, cam.tile_ly, cam.ntx, cam.nty, cam.leftmost,
                        cam.topmost)
    cnt_c, lst_c = cnt.cpu(), lst.cpu()
    flat = [sorted(lst_c[t, :int(cnt_c[t])].tolist()) for t in range(T)]
    np.savez_compressed(os.path.join(out_dir, "tiles.npz"), counts=cnt_c.numpy(),
                        flat_ids=np.array([i for f in flat for i in f], dtype=np.int32))

    # ---- draw_rgb.npz : draw + draw_backward on sorted per-instance inputs ----------------
    inst, cam, grad_img = GC.draw_inputs()
    t = {k: inst[k].to(dev).float().contiguous().requires_grad_(True) for k in ("pos", "rgb", "opa", "cov")}
    dummy = torch.zeros(3, device=dev)
    img = rref.draw(t["pos"], t["rgb"], t["opa"], t["cov"], inst["accum"].to(dev), cam.Hp, cam.Wp, cam.fx, cam.fy,
                    False, False, False, True, dummy, dummy, dummy, dummy)
    img.backward(grad_img.to(dev))
    counts = inst["accum"][1:] - inst["accum"][:-1]
    assert int(counts.max()) <= 500, "outside the reference backward's safe regime"
    np.savez_compressed(os.path.join(out_dir, "draw_rgb.npz"), image=cpu(img),
                        in_pos=cpu(inst["pos"]), in_rgb=cpu(inst["rgb"]), in_opa=cpu(inst["opa"]),
                        in_cov=cpu(inst["cov"]), in_accum=cpu(inst["accum"]),
                        grad_pos=cpu(t["pos"].grad), grad_rgb=cpu(t["rgb"].grad), grad_opa=cpu(t["opa"].grad),
                        grad_cov=cpu(t["cov"].grad))

    # ---- draw_sh.npz : draw + draw_backward with per-pixel SH-27 colour ---------------------------
    inst, cam, grad_img, rays = GC.draw_sh_inputs()
    counts = inst["accum"][1:] - inst["accum"][:-1]
    assert int(counts.max()) <= 160, "outside the reference SH backward's safe regime"
    t = {k: inst[k].to(dev).float().contiguous().requires_grad_(True) for k in ("pos", "rgb", "opa", "cov")}
    r = [x.to(dev).float().contiguous() for x in rays]
    img = rref.draw(t["pos"], t["rgb"], t["opa"], t["cov"], inst["accum"].to(dev), cam.Hp, cam.Wp, cam.fx, cam.fy,
                    False, False, True, True, r[0], r[1], r[2], r[3])
    img.backward(grad_img.to(dev))
    np.savez_compressed(os.path.join(out_dir, "draw_sh.npz"), image=cpu(img),
                        in_pos=cpu(inst["pos"]), in_rgb=cpu(inst["rgb"]), in_opa=cpu(inst["opa"]),
                        in_cov=cpu(inst["cov"]), in_accum=cpu(inst["accum"]),
                        grad_pos=cpu(t["pos"].grad), grad_rgb=cpu(t["rgb"].grad), grad_opa=cpu(t["opa"].grad),
                        grad_cov=cpu(t["cov"].grad))

    # ---- frame_c1.npz : the reference's whole per-frame pipeline ---------------------------
    g, v, cam, go = GC.frame_inputs()
    c = GC.CASES["frame_c1.npz"]
    bad, mx, maxp = GC.reference_key_collisions(g, cam)
    assert bad == 0 and mx <= maxp, (bad, mx, maxp)
    frame = ref_pipeline.LegacyFrame(gref, rref, c["w"], c["h"], v.fx, v.fy, v.rot.to(dev), v.tran.to(dev))
    pr = {k: x.to(dev).clone().requires_grad_(True) for k, x in g.items()}
    img = frame(pr["pos"], pr["rgb"], pr["opa"], pr["quat"], pr["scale"])
    img.backward(go.to(dev))
    # inside the reference's own limits: dense-list capacity MAXP = Nc//20 (splatter.py:569) and the
    # backward's 500-instance chunk (SURVEY.md hazards 1, 4)
    assert frame.aux["max_tile"] <= min(500, frame.aux["MAXP"]), frame.aux["max_tile"]
    np.savez_compressed(os.path.join(out_dir, "frame_c1.npz"), n=c["n"], w=c["w"], h=c["h"], image=cpu(img),
                        **{"grad_" + k: cpu(pr[k].grad) for k in pr})
    print("golden fixtures written to", out_dir, sorted(os.listdir(out_dir)))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "golden_out"))
