"""Mesh vertex updates (b200pt_update_mesh_vertices) on the GPU: update time and what a refit tree costs as the deformation grows.

  - update time per scene (glass sphere, Viking, BreakfastRoom's largest mesh, all of BreakfastRoom's meshes at once): host vs device input
    (a CUDA tensor) x refit / GPU rebuild / host rebuild.  Host clock around the call followed by a device synchronise, median of --reps calls
    after two warm-up calls; every call alternates between the original and the wobbled vertices, so every call changes the mesh;
  - the device-to-host copy of the host mirror: a pageable device-to-host copy of the same bytes (torch .cpu(), as the engine copies into its
    std::vector), against the device-input refit time;
  - wobble-amplitude sweep on BreakfastRoom's largest mesh: nodes per camera ray (b200pt_trace_stats, 192 x 108 camera rays) and Mpaths/s of a
    fixed render, for a refit of the undeformed tree and for a GPU rebuild at every amplitude.
Prints the card's name, power limit and max SM clock read in the same run.  Writes nothing but --out (JSON), if given.
usage: python profiles/mesh_deform.py [--reps 10] [--frames 16] [--size 1920x1080] [--out FILE]"""
import argparse, json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "profiles"))
import numpy as np
import util
from instance_refit import gpu_info, camera_rays, timed, render_rate

MODES = (("refit", False), ("gpu_rebuild", "gpu"), ("host_rebuild", True))


def vertex_normals(pos, idx):
    """area-weighted vertex normals; a vertex whose triangles have no area gets (0, 0, 1)"""
    p = pos.astype(np.float64); t = np.asarray(idx, np.int64).reshape(-1, 3)
    fn = np.cross(p[t[:, 1]] - p[t[:, 0]], p[t[:, 2]] - p[t[:, 0]])
    n = np.zeros_like(p)
    for k in range(3): np.add.at(n, t[:, k], fn)
    ln = np.linalg.norm(n, axis=1, keepdims=True)
    return np.where(ln > 0, n / np.maximum(ln, 1e-300), np.array([0.0, 0.0, 1.0]))


def wobbled(v, idx, amp):
    """radial wobble of relative amplitude amp about the mesh's centroid, normals recomputed"""
    p = v["pos"].astype(np.float64); c = p.mean(0); r = p - c
    d = r / np.maximum(np.linalg.norm(r, axis=1, keepdims=True), 1e-30)
    out = v.copy()
    out["pos"] = (c + r * (1.0 + amp * np.sin(5.0 * d[:, 0]) * np.cos(3.0 * d[:, 1]))[:, None]).astype(np.float32)
    if amp: out["nrm"] = vertex_normals(out["pos"], idx).astype(np.float32)
    return out


def rows(v):
    return np.ascontiguousarray(v).view(np.float32).reshape(-1, 8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10); ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--size", default="1920x1080"); ap.add_argument("--out")
    a = ap.parse_args()
    W, H = (int(v) for v in a.size.split("x"))
    import torch
    if not torch.cuda.is_available(): sys.exit("mesh_deform.py measures on the GPU: no CUDA device")
    card = gpu_info()
    print("card (name, power limit, max SM clock):", card)
    res = {"card": card, "size": [W, H], "frames": a.frames, "depth": 8, "update_ms": {}, "mirror_copy": {}, "sweep": []}
    br = util.scene_dict("breakfast_room")
    big = int(np.argmax([len(v) for v, _ in br["meshes"]]))
    cases = [("glass_sphere", "cornell_box_glass", [6]), ("viking", "viking_room", [0]), (f"breakfast_mesh{big}", "breakfast_room", [big]),
             ("breakfast_all", "breakfast_room", [m for m, (v, _) in enumerate(br["meshes"]) if len(v)])]
    for label, fixture, meshes in cases:
        sc = util.scene_dict(fixture)
        T = util.product_tracer(fixture, W, H, MaxDepth=8)
        orig = {m: rows(sc["meshes"][m][0]) for m in meshes}
        wob = {m: rows(wobbled(sc["meshes"][m][0], sc["meshes"][m][1], 0.1)) for m in meshes}
        dev = {k: {m: torch.from_numpy(x.copy()).cuda(0) for m, x in s.items()} for k, s in (("orig", orig), ("wob", wob))}
        nv = sum(len(x) for x in orig.values())
        r = {"vertices": nv}
        for _ in range(2):                                                  # alternated: each combination timed twice, the lower median kept
            for inp in ("host", "device"):
                for key, mode in MODES:
                    flip = [0]
                    def upd():
                        flip[0] ^= 1
                        if inp == "host": T.update_mesh_vertices(wob if flip[0] else orig, rebuild=mode)
                        else: T.update_mesh_vertices(dev["wob"] if flip[0] else dev["orig"], rebuild=mode)
                    k = f"{inp}_{key}_ms"
                    r[k] = min(r.get(k, 1e30), timed(upd, T, a.reps) * 1e3)
        res["update_ms"][label] = r
        print(f"{label}: {nv} vertices | " + " | ".join(f"{k} {v:.3f}" for k, v in r.items() if k.endswith("_ms")))
        # the mirror: a pageable device-to-host copy of the same bytes
        flat = torch.cat([t.reshape(-1) for t in dev["wob"].values()])
        for _ in range(2): flat.cpu()
        torch.cuda.synchronize(); ts = []
        for _ in range(a.reps):
            t0 = time.perf_counter(); flat.cpu(); torch.cuda.synchronize(); ts.append(time.perf_counter() - t0)
        cp = float(np.median(ts)) * 1e3
        res["mirror_copy"][label] = {"bytes": nv * 32, "d2h_ms": cp, "share_of_device_refit": cp / r["device_refit_ms"]}
        print(f"  mirror copy ({nv * 32} B, pageable D2H) {cp:.3f} ms = {100 * cp / r['device_refit_ms']:.1f} % of the device-input refit")
        T.close()
    # amplitude sweep: refit of the undeformed tree (R) against a GPU rebuild (G) at every amplitude
    R = util.product_tracer("breakfast_room", W, H, MaxDepth=8); G = util.product_tracer("breakfast_room", W, H, MaxDepth=8)
    o, d = camera_rays(R)
    v0, idx = br["meshes"][big]
    print(f"  {'amp':>5} | {'refit Mp/s':>10} {'nodes':>6} | {'gpu Mp/s':>8} {'nodes':>6}")
    for amp in (0.0, 0.05, 0.1, 0.2, 0.4):
        v = wobbled(v0, idx, amp)
        R.update_mesh_vertices({big: v}); G.update_mesh_vertices({big: v}, rebuild="gpu")
        row = {"amp": amp}
        for key, h in (("refit", R), ("gpu_rebuild", G)):
            st = h.trace_stats(o, d, 0.0, 1e30).astype(np.float64)
            row[key] = {"mpaths_s": render_rate(h, a.frames), "nodes": float(st[:, 0].mean()), "tris": float(st[:, 1].mean())}
        res["sweep"].append(row)
        print(f"  {amp:5.2f} | {row['refit']['mpaths_s']:10.0f} {row['refit']['nodes']:6.1f} | {row['gpu_rebuild']['mpaths_s']:8.0f} {row['gpu_rebuild']['nodes']:6.1f}")
    R.close(); G.close()
    if a.out:
        with open(a.out, "w") as f: json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
