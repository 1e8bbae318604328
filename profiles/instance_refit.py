"""Instance transform updates on the GPU: what an update costs, and what a refit tree costs the render afterwards.

Per scene (Cornell flat; Cornell glass, default and B200PT_SMEM_BIG=1; Viking; BreakfastRoom with its BVH4):
  - update time of b200pt_update_instance_transforms with refit and with rebuild, and of b200pt_set_scene_arrays: host clock around the call
    followed by a device synchronise, median of --reps calls after two warm-up calls;
  - an animation sweep: one instance turned 0-90 degrees about a vertical axis through its centre.  At every step one handle refits the tree
    it built for 0 degrees and another rebuilds it; for each, Mpaths/s of a fixed render (--size, depth 8, --frames frames) and the mean BVH
    nodes visited and triangles tested per camera ray (b200pt_trace_stats, a 192 x 108 grid of camera rays).
Prints the card's name, power limit and max SM clock read in the same run, then the tables.  Writes nothing but --out (JSON), if given.
usage: python profiles/instance_refit.py [--reps 10] [--frames 16] [--size 1920x1080] [--steps 7] [--out FILE]"""
import argparse, json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import util

SCENES = [   # label, fixture, env, instance turned in the sweep
    ("cornell (flat)", "cornell_box", {}, 5),
    ("glass", "cornell_box_glass", {}, 6),
    ("glass big", "cornell_box_glass", {"B200PT_SMEM_BIG": "1"}, 6),
    ("viking", "viking_room", {}, 0),
    ("breakfast (bvh4)", "breakfast_room", {}, 9),
]


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                                                 # the numbers below still stand; say why the card is unnamed
        return f"nvidia-smi unavailable ({e})"


def turned(sc, i, deg):
    xf = np.stack([np.asarray(x, np.float32).reshape(16) for x, _, _ in sc["instances"]])
    M = xf[i].reshape(4, 4).T.astype(np.float64)
    xfm, m, _ = sc["instances"][i]
    p = sc["meshes"][m][0]["pos"].astype(np.float64) @ M[:3, :3].T + M[:3, 3]
    c = 0.5 * (p.min(0) + p.max(0))
    a = np.radians(deg); R = np.eye(4); R[0, 0] = R[2, 2] = np.cos(a); R[0, 2] = np.sin(a); R[2, 0] = -np.sin(a)
    T0 = np.eye(4); T0[:3, 3] = -c; T1 = np.eye(4); T1[:3, 3] = c
    xf[i] = (T1 @ R @ T0 @ M).T.reshape(-1).astype(np.float32)
    return xf


def camera_rays(T, nx=192, ny=108):
    vi, pi = T.get_camera()
    VI = vi.reshape(4, 4).T.astype(np.float64); PI = pi.reshape(4, 4).T.astype(np.float64)
    x, y = np.meshgrid((np.arange(nx) + 0.5) / nx * 2 - 1, (np.arange(ny) + 0.5) / ny * 2 - 1)
    tgt = np.stack([x.ravel(), y.ravel(), np.ones(x.size), np.ones(x.size)], 1) @ PI.T
    d = tgt[:, :3] / np.linalg.norm(tgt[:, :3], axis=1, keepdims=True) @ VI[:3, :3].T
    o = np.repeat(VI[None, :3, 3], len(d), 0)
    return o.astype(np.float32), d.astype(np.float32)


def timed(fn, T, reps):
    for _ in range(2): fn(); T.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter(); fn(); T.synchronize(); ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def render_rate(T, frames):
    T.reset(); T.path_trace(frames, util.BASE_SEED); T.synchronize()         # warm-up: this tree's launch shapes and the full-size waves
    T.reset(); p0 = T.counters()["paths"]
    t0 = time.perf_counter(); T.path_trace(frames, util.BASE_SEED); T.synchronize(); dt = time.perf_counter() - t0
    return (T.counters()["paths"] - p0) / dt / 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10); ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--size", default="1920x1080"); ap.add_argument("--steps", type=int, default=7); ap.add_argument("--out")
    a = ap.parse_args()
    W, H = (int(v) for v in a.size.split("x"))
    import torch
    if not torch.cuda.is_available(): sys.exit("instance_refit.py measures on the GPU: no CUDA device")
    card = gpu_info()
    print("card (name, power limit, max SM clock):", card)
    res = {"card": card, "size": [W, H], "frames": a.frames, "depth": 8, "scenes": {}}
    for label, fixture, env, inst in SCENES:
        for k in ("B200PT_SMEM_BIG",): os.environ.pop(k, None)
        os.environ.update(env)
        sc = util.scene_dict(fixture)
        T = util.product_tracer(fixture, W, H, MaxDepth=8)
        xf0 = T.get_instance_transforms(); xf1 = turned(sc, inst, 30.0)
        flip = [0]
        def upd(rebuild):
            flip[0] ^= 1; T.update_instance_transforms(xf1 if flip[0] else xf0, rebuild=rebuild)
        t_refit = timed(lambda: upd(False), T, a.reps)
        t_rebuild = timed(lambda: upd(True), T, a.reps)
        t_set = timed(lambda: T.set_scene(sc), T, a.reps)
        T.resize(W, H)                                                      # set_scene sets the image to 1080 rows
        print(f"\n{label}: {T.scene_stats()['triangles']} triangles | update refit {t_refit * 1e3:.2f} ms | rebuild {t_rebuild * 1e3:.1f} ms | set_scene_arrays {t_set * 1e3:.1f} ms")
        R = util.product_tracer(fixture, W, H, MaxDepth=8)                  # refit handle (tree of 0 degrees); T rebuilds
        o, d = camera_rays(T)
        print(f"  {'deg':>5} | {'refit Mp/s':>10} {'nodes':>7} {'tris':>6} | {'rebuild Mp/s':>12} {'nodes':>7} {'tris':>6}")
        sweep = []
        for deg in np.linspace(0.0, 90.0, a.steps):
            xf = turned(sc, inst, float(deg))
            R.update_instance_transforms(xf, rebuild=False); T.update_instance_transforms(xf, rebuild=True)
            row = {"deg": float(deg)}
            for key, h in (("refit", R), ("rebuild", T)):
                st = h.trace_stats(o, d, 0.0, 1e30).astype(np.float64)
                row[key] = {"mpaths_s": render_rate(h, a.frames), "nodes": float(st[:, 0].mean()), "tris": float(st[:, 1].mean())}
            sweep.append(row)
            print(f"  {deg:5.1f} | {row['refit']['mpaths_s']:10.0f} {row['refit']['nodes']:7.1f} {row['refit']['tris']:6.1f} | "
                  f"{row['rebuild']['mpaths_s']:12.0f} {row['rebuild']['nodes']:7.1f} {row['rebuild']['tris']:6.1f}")
        res["scenes"][label] = {"update_refit_ms": t_refit * 1e3, "update_rebuild_ms": t_rebuild * 1e3, "set_scene_ms": t_set * 1e3, "sweep": sweep}
        T.close(); R.close()
        for k in env: os.environ.pop(k, None)
    if a.out:
        with open(a.out, "w") as f: json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
