"""The GPU rebuild (b200pt_update_instance_transforms with B200PT_REBUILD_GPU) against the refit and the host rebuild, on the GPU.

Per scene (as profiles/instance_refit.py: Cornell flat, glass default and big mode, Viking, BreakfastRoom with its BVH4):
  - update time of refit, host rebuild (the set_scene tree) and GPU rebuild, alternated in one session: host clock around the call followed by
    a device synchronise, median of --reps calls after two warm-up calls; the first refit after a GPU rebuild (its lbvh_refit_prepare runs on
    the host again) against a steady refit; the host rebuild with B200PT_BVH_SAH=0 (the LBVH build and its host depth walk, no tree pass);
    the builder alone on the scene's references (b200pt_bvh2_ploc_build_query, boxes copied in and the trees copied out);
  - tree quality of the GPU tree, the host level-3 tree and the LBVH (B200PT_BVH_SAH=0 on a fresh handle): nodes and triangles per camera ray
    (b200pt_trace_stats, 192 x 108 camera rays) and Mpaths/s of a fixed render, the three trees alternated, --runs runs each;
  - the animation sweep of instance_refit.py with a third column: a GPU rebuild at every angle.
Prints the card's name, power limit and max SM clock read in the same run.  Writes nothing but --out (JSON), if given.
usage: python profiles/gpu_rebuild.py [--reps 10] [--frames 16] [--size 1920x1080] [--steps 7] [--runs 3] [--scenes breakfast] [--out FILE]"""
import argparse, json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "profiles"))
import numpy as np
import util
from instance_refit import SCENES, gpu_info, turned, camera_rays, timed, render_rate


def refs_in_morton_order(fixture):
    import bvh_lab
    sc = bvh_lab.load_fixture(os.path.join(ROOT, "tests", "golden", f"{fixture}.npz"))
    rb, _ = bvh_lab.split_refs(bvh_lab.world_triangles(sc))
    return rb[np.argsort(bvh_lab.morton_keys(rb), kind="stable")].reshape(-1, 6).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10); ap.add_argument("--frames", type=int, default=16); ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--size", default="1920x1080"); ap.add_argument("--steps", type=int, default=7); ap.add_argument("--out")
    ap.add_argument("--scenes", default="", help="comma-separated substrings of the scene labels (default: all)")
    a = ap.parse_args()
    W, H = (int(v) for v in a.size.split("x"))
    import torch
    if not torch.cuda.is_available(): sys.exit("gpu_rebuild.py measures on the GPU: no CUDA device")
    card = gpu_info()
    print("card (name, power limit, max SM clock):", card)
    res = {"card": card, "size": [W, H], "frames": a.frames, "depth": 8, "scenes": {}}
    pick = [s for s in a.scenes.split(",") if s]
    for label, fixture, env, inst in SCENES:
        if pick and not any(p in label for p in pick): continue
        for k in ("B200PT_SMEM_BIG", "B200PT_BVH_SAH"): os.environ.pop(k, None)
        os.environ.update(env)
        sc = util.scene_dict(fixture)
        T = util.product_tracer(fixture, W, H, MaxDepth=8)
        xf0 = T.get_instance_transforms(); xf1 = turned(sc, inst, 30.0)
        flip = [0]
        def upd(rebuild, h=T):
            flip[0] ^= 1; h.update_instance_transforms(xf1 if flip[0] else xf0, rebuild=rebuild)
        r = {}
        for _ in range(2):                                                  # alternated: each mode timed twice, the lower median kept
            for key, mode in (("refit_ms", False), ("host_rebuild_ms", True), ("gpu_rebuild_ms", "gpu")):
                r[key] = min(r.get(key, 1e30), timed(lambda: upd(mode), T, a.reps) * 1e3)
        ts = []
        for _ in range(a.reps):                                             # first refit after a GPU rebuild
            upd("gpu"); T.synchronize()
            t0 = time.perf_counter(); upd(False); T.synchronize(); ts.append(time.perf_counter() - t0)
        r["first_refit_after_gpu_rebuild_ms"] = float(np.median(ts)) * 1e3
        os.environ["B200PT_BVH_SAH"] = "0"
        r["host_rebuild_lbvh_only_ms"] = timed(lambda: upd(True), T, a.reps) * 1e3
        os.environ.pop("B200PT_BVH_SAH")
        rb = refs_in_morton_order(fixture)
        r["references"] = len(rb)
        r["builder_alone_ms"] = timed(lambda: T.bvh2_ploc_build_query(rb), T, a.reps) * 1e3
        print(f"\n{label}: {len(rb)} references | " + " | ".join(f"{k} {v:.2f}" for k, v in r.items() if k.endswith("_ms")))
        # tree quality: host level 3 (T back at 0 degrees, rebuilt as set_scene builds), LBVH (fresh handle, B200PT_BVH_SAH=0), GPU tree
        T.update_instance_transforms(xf0, rebuild=True)
        os.environ["B200PT_BVH_SAH"] = "0"; L = util.product_tracer(fixture, W, H, MaxDepth=8); os.environ.pop("B200PT_BVH_SAH")
        G = util.product_tracer(fixture, W, H, MaxDepth=8); G.update_instance_transforms(xf0, rebuild="gpu")
        o, d = camera_rays(T)
        trees = {"host_level3": T, "lbvh": L, "gpu": G}
        q = {k: {"mpaths_s": []} for k in trees}
        for k, h in trees.items():
            st = h.trace_stats(o, d, 0.0, 1e30).astype(np.float64)
            q[k]["nodes"] = float(st[:, 0].mean()); q[k]["tris"] = float(st[:, 1].mean())
        for _ in range(a.runs):
            for k, h in trees.items(): q[k]["mpaths_s"].append(render_rate(h, a.frames))
        for k in trees:
            print(f"  {k:12s} nodes/ray {q[k]['nodes']:6.1f}  tris/ray {q[k]['tris']:6.1f}  Mpaths/s " + " ".join(f"{v:.0f}" for v in q[k]["mpaths_s"]))
        r["quality"] = q
        L.close()
        # animation sweep: refit of the 0-degree tree (R), host rebuild (T), GPU rebuild (G) at every angle
        R = util.product_tracer(fixture, W, H, MaxDepth=8)
        print(f"  {'deg':>5} | {'refit Mp/s':>10} {'nodes':>6} | {'host Mp/s':>9} {'nodes':>6} | {'gpu Mp/s':>8} {'nodes':>6}")
        sweep = []
        for deg in np.linspace(0.0, 90.0, a.steps):
            xf = turned(sc, inst, float(deg))
            R.update_instance_transforms(xf, rebuild=False); T.update_instance_transforms(xf, rebuild=True); G.update_instance_transforms(xf, rebuild="gpu")
            row = {"deg": float(deg)}
            for key, h in (("refit", R), ("host_rebuild", T), ("gpu_rebuild", G)):
                st = h.trace_stats(o, d, 0.0, 1e30).astype(np.float64)
                row[key] = {"mpaths_s": render_rate(h, a.frames), "nodes": float(st[:, 0].mean()), "tris": float(st[:, 1].mean())}
            sweep.append(row)
            print(f"  {deg:5.1f} | {row['refit']['mpaths_s']:10.0f} {row['refit']['nodes']:6.1f} | {row['host_rebuild']['mpaths_s']:9.0f} "
                  f"{row['host_rebuild']['nodes']:6.1f} | {row['gpu_rebuild']['mpaths_s']:8.0f} {row['gpu_rebuild']['nodes']:6.1f}")
        r["sweep"] = sweep
        res["scenes"][label] = r
        T.close(); R.close(); G.close()
        for k in env: os.environ.pop(k, None)
    if a.out:
        with open(a.out, "w") as f: json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
