"""glTF pose (b200pt_pose) on the GPU: cost per call, the pose kernels and the commit's mirror copy, for synthetic skinned and morphed grids.

  - shapes: 64k, 1M and 4M vertices, 4 or 8 influences (JOINTS_0 [+ JOINTS_1]), 0 or 8 active morph targets (POSITION + NORMAL deltas);
  - pose time: host clock around pose() followed by a device synchronise, median of --reps calls after two warm-ups; every call poses
    another time, so every call changes the mesh; refit and GPU rebuild at every size, host rebuild at 64k;
  - kernels: k_pose_vertices (+ k_pose_normals) from torch.profiler in a run of their own, with achieved GB/s against the bytes model
    (per vertex: 32 B rest + 8 B per influence + 24 B per active target, 32 B written);
  - the device-to-host mirror copy of the commit, from the same profile;
  - the user-side alternative: skinning and morphing in torch on the GPU, then update_mesh_vertices from the CUDA tensor.
Prints the card's name, power limit and max SM clock read in the same run; fails without a GPU.  Writes glTF files to a temporary directory
and nothing else but --out (JSON), if given.
The host evaluation is not timed on its own.
usage: python profiles/gltf_animation.py [--reps 10] [--sizes 65536,1048576,4194304] [--out FILE]"""
import argparse, json, os, sys, tempfile, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "profiles"))
import numpy as np
import torch
from instance_refit import gpu_info
from test_gltf_animation import Gltf, quat

JOINTS = 32


def grid_scene(path, nv, infl, targets):
    side = int(round(np.sqrt(nv))); n = side * side
    u, v = np.meshgrid(np.linspace(0, 1, side, dtype=np.float32), np.linspace(0, 1, side, dtype=np.float32))
    P = np.stack([u.ravel() * 4 - 2, v.ravel() * 4, np.zeros(n, np.float32)], 1).astype(np.float32)
    N = np.tile(np.array([0, 0, 1], np.float32), (n, 1)); U = np.stack([u.ravel(), v.ravel()], 1).astype(np.float32)
    q = (np.arange(side - 1)[:, None] * side + np.arange(side - 1)[None, :]).ravel().astype(np.uint32)
    I = np.stack([q, q + 1, q + side, q + 1, q + side + 1, q + side], 1).ravel()
    rng = np.random.default_rng(1)
    base = np.clip((P[:, 1] / 4 * (JOINTS - 1)).astype(np.int64), 0, JOINTS - 1)
    J = (base[:, None] + np.arange(infl)[None, :]) % JOINTS
    Wt = rng.random((n, infl)).astype(np.float32); Wt /= Wt.sum(1, keepdims=True)
    G = Gltf(); F32 = 5126
    at = {"POSITION": G.acc(P, F32, "VEC3"), "NORMAL": G.acc(N, F32, "VEC3"), "TEXCOORD_0": G.acc(U, F32, "VEC2")}
    for s in range(infl // 4):
        at[f"JOINTS_{s}"] = G.acc(J[:, 4 * s:4 * s + 4].astype(np.uint16), 5123, "VEC4", 1)
        at[f"WEIGHTS_{s}"] = G.acc(Wt[:, 4 * s:4 * s + 4], F32, "VEC4", 1)
    prim = {"attributes": at, "indices": G.acc(I, 5125, "SCALAR")}
    if targets:
        prim["targets"] = [{"POSITION": G.acc((rng.normal(0, 0.01, (n, 3))).astype(np.float32), F32, "VEC3", 1),
                            "NORMAL": G.acc((rng.normal(0, 0.01, (n, 3))).astype(np.float32), F32, "VEC3", 1)} for _ in range(targets)]
    nodes = [{"mesh": 0, "skin": 0}] + [{"translation": [0, 4.0 / JOINTS if k else 0, 0], "children": [k + 2] if k + 1 < JOINTS else []} for k in range(JOINTS)]
    kt = np.array([0, 1, 2], np.float32)
    smp = [{"input": G.acc(kt, F32, "SCALAR", 1), "output": G.acc(np.array([quat((1, 0, 0), 0), quat((1, 0, 0), 4), quat((0, 1, 0), -3)], np.float32), F32, "VEC4", 1)}]
    chans = [{"sampler": 0, "target": {"node": 1 + k, "path": "rotation"}} for k in range(JOINTS)]
    if targets:
        smp.append({"input": G.acc(kt, F32, "SCALAR", 1), "output": G.acc(np.tile(np.array([[0.2], [0.9], [0.5]], np.float32), (1, targets)).ravel(), F32, "SCALAR", 1)})
        chans.append({"sampler": 1, "target": {"node": 0, "path": "weights"}})
    g = {"asset": {"version": "2.0"}, "scenes": [{"nodes": [0, 1]}], "nodes": nodes, "skins": [{"joints": list(range(1, JOINTS + 1))}],
         "meshes": [{"primitives": [prim], **({"weights": [0.5] * targets} if targets else {})}], "materials": [{}],
         "animations": [{"samplers": smp, "channels": chans}], "accessors": G.accs, "bufferViews": G.views,
         "buffers": [{"uri": "geo.bin", "byteLength": len(G.blob[0])}, {"uri": "anim.bin", "byteLength": len(G.blob[1])}]}
    d = os.path.dirname(path)
    open(os.path.join(d, "geo.bin"), "wb").write(G.blob[0]); open(os.path.join(d, "anim.bin"), "wb").write(G.blob[1])
    open(path, "w").write(json.dumps(g))
    return dict(n=n, P=P, N=N, U=U, J=J, W=Wt)


def torch_pose(T, S, pal, dpos, w):
    """the user-side alternative: skin + morph with torch on the GPU, then update_mesh_vertices from the tensor"""
    p = S["P"] + (dpos * w[:, None, None]).sum(0) if dpos is not None else S["P"]
    M = (pal[S["J"]] * S["W"][..., None, None]).sum(1)                            # (n, 3, 4)
    pos = torch.einsum("nij,nj->ni", M[:, :, :3], p) + M[:, :, 3]
    nrm = torch.nn.functional.normalize(torch.einsum("nij,nj->ni", M[:, :, :3], S["N"]), dim=1)
    T.update_mesh_vertices({0: torch.cat([pos, nrm, S["U"]], 1).contiguous()})


def main():
    ap = argparse.ArgumentParser(); ap.add_argument("--reps", type=int, default=10); ap.add_argument("--out")
    ap.add_argument("--sizes", default="65536,1048576,4194304")
    a = ap.parse_args()
    if not torch.cuda.is_available(): sys.exit("gltf_animation.py needs a CUDA device")
    import vpt_b200 as pt
    info = gpu_info(); print("GPU:", info)
    rows = []
    for nv in [int(x) for x in a.sizes.split(",")]:
        for infl, targets in ((4, 0), (8, 0), (4, 8), (8, 8)):
            with tempfile.TemporaryDirectory() as d:
                path = os.path.join(d, "g.gltf"); S = grid_scene(path, nv, infl, targets)
                T = pt.PathTracer(0); T.set_scene_file(path); T.resize(64, 64)
                row = dict(vertices=S["n"], influences=infl, targets=targets)
                modes = [("refit", False), ("gpu_rebuild", "gpu")] + ([("host_rebuild", True)] if nv <= 65536 else [])
                for name, rb in modes:
                    ts = []
                    for k in range(a.reps + 2):
                        t0 = time.perf_counter(); T.pose(0, 0.1 + 0.17 * k, rebuild=rb); T.synchronize(); ts.append(time.perf_counter() - t0)
                    row[f"pose_{name}_ms"] = 1e3 * float(np.median(ts[2:]))
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    for k in range(a.reps): T.pose(0, 0.3 + 0.11 * k); T.synchronize()
                kern = dtoh = 0.0
                for e in prof.events():
                    dur = getattr(e, "device_time", 0) or 0
                    if "k_pose_" in e.name: kern += dur
                    elif "DtoH" in e.name or "Memcpy DtoH" in e.name: dtoh += dur
                kern_ms, dtoh_ms = kern / 1e3 / a.reps, dtoh / 1e3 / a.reps
                nbytes = S["n"] * (32 + 8 * infl + 24 * targets + 32)
                row.update(kernels_ms=kern_ms, kernels_GBps=nbytes / max(kern_ms, 1e-9) / 1e6, bytes_model=nbytes, mirror_dtoh_ms=dtoh_ms)
                # the user-side alternative, same shapes
                dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
                TS = dict(P=dev(S["P"]), N=dev(S["N"]), U=dev(S["U"]), J=dev(S["J"].astype(np.int64)), W=dev(S["W"]))
                pal = torch.eye(3, 4, device="cuda").repeat(JOINTS, 1, 1) + 0.01 * torch.randn(JOINTS, 3, 4, device="cuda")
                dpos = torch.randn(targets, S["n"], 3, device="cuda") * 0.01 if targets else None
                wv = torch.full((targets,), 0.5, device="cuda") if targets else None
                ts = []
                for k in range(a.reps + 2):
                    t0 = time.perf_counter(); torch_pose(T, TS, pal, dpos, wv); T.synchronize(); ts.append(time.perf_counter() - t0)
                row["torch_then_update_refit_ms"] = 1e3 * float(np.median(ts[2:]))
                T.close(); del TS, pal, dpos; torch.cuda.empty_cache()
                print(json.dumps(row)); rows.append(row)
    if a.out: json.dump(dict(gpu=info, rows=rows), open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
