"""Small end-to-end workload for compute-sanitizer (memcheck / racecheck / initcheck): every kernel family once, tiny sizes.
usage: compute-sanitizer --tool memcheck python profiles/sanitize_small.py"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import util

FOG = dict(CornerMin=(-4.0, -4.0, -10.0), CornerMax=(4.5, 3.0, -1.0), Density=0.35, Color=(0.8, 0.7, 0.6), Anisotropy=0.4, Alpha=1.5, DropletSize=14.0)
def run(name, W, H, frames, depth, **kw):
    T = util.product_tracer(name, W, H, MaxDepth=depth, **kw)
    T.path_trace(frames, util.BASE_SEED)
    img = T.get_hdr(); assert np.isfinite(img).all()
    T.post_process(); T.get_ldr()
    T.post_process_rows(8, min(H, 24)); T.get_ldr_rows(8, min(H, 24))
    print(name, kw.get("Volumes") is not None, os.environ.get("B200PT_FUSE"), os.environ.get("B200PT_TRAV"), "ok", float(img[..., :3].mean()))

run("cornell_box", 64, 36, 2, 6)                                   # BVH in shared memory (TMA), flat traversal, uniform class, k_camera, k_shade_hit<., ., true> + k_extend
os.environ["B200PT_FLAT_MAX"] = "0"; run("cornell_box", 48, 32, 1, 4); del os.environ["B200PT_FLAT_MAX"]      # BVH2 stack traversal in shared memory (k_camera too)
os.environ["B200PT_CAMERA"] = "0"; run("cornell_box", 48, 32, 2, 6); del os.environ["B200PT_CAMERA"]          # k_raygen + k_extend<., true, .>
os.environ["B200PT_SMEM_BIG"] = "1"; run("cornell_box_glass", 48, 48, 2, 8); del os.environ["B200PT_SMEM_BIG"]  # big mode: 512-thread k_camera, k_extend, fused k_shade_hit
run("cornell_box", 48, 32, 1, 5, Volumes=[FOG])                     # k_volume_decide / k_shade_volume
run("cornell_box", 48, 32, 2, 5, EnableAtmosphere=1, SkyRotationAltitude=-30.0)                       # atmosphere: sun NEE, delta tracking, transmittance walks
run("cornell_box", 40, 30, 1, 5, EnableAtmosphere=1, SkyRotationAltitude=-20.0, Volumes=[FOG])        # atmosphere + homogeneous volume
def _het():
    from oracle import orc
    z, y, x = np.mgrid[0:20, 0:34, 0:36].astype(np.float32)
    d = np.exp(-(((x - 18) / 9) ** 2 + ((y - 17) / 9) ** 2 + ((z - 10) / 6) ** 2)).astype(np.float32) * 2.0
    return dict(Position=(0.2, -0.2, -5.5), Scale=(3.0, 3.0, 3.0), Density=4.0, Grid=orc.prepare_density_grid(d, index_min=(-18, -17, -10), temperature=d * 100.0))
run("cornell_box", 40, 30, 1, 5, Volumes=[FOG, _het()])                                              # grid volume: delta tracking, ratio-tracked NEE transmittance in k_connect<.., true>
run("cornell_box", 40, 30, 1, 5, EnableAtmosphere=1, SkyRotationAltitude=-20.0, Volumes=[_het()])    # ... under the atmosphere
def _adaptive(name, **kw):                                          # adaptive sampling: k_camera<., true> / k_raygen<true>, k_resolve_adaptive, k_adaptive_update + _compact
    T = util.product_tracer(name, 40, 30, MaxDepth=5, **kw)
    T.set_adaptive(Enable=1, Threshold=0.3, MinSamples=4, Interval=4)
    T.path_trace(12, util.BASE_SEED)
    assert np.isfinite(T.get_hdr()).all() and 0 <= T.active_pixels() <= 40 * 30
    print(name, "adaptive", T.active_pixels(), "ok")
_adaptive("cornell_box"); _adaptive("cornell_box", Volumes=[FOG])
def _denoise(name, **kw):                                           # per-pixel statistics, k_features<SMEM>, k_record_variance, the a-trous filter, its post chain
    T = util.product_tracer(name, 40, 30, MaxDepth=5, **kw)
    T.set_track_variance(True)
    T.path_trace(4, util.BASE_SEED)
    T.denoise(FeatureSamples=2); d = T.get_denoised(); assert np.isfinite(d).all()
    a, nd, v = T.denoise_inputs(FeatureSamples=2); T.denoise_image(T.get_hdr(), a, nd, v, Iterations=2)
    T.post_process_denoised(); T.get_ldr()
    print(name, "denoise ok")
_denoise("cornell_box"); _denoise("cornell_box_glass")
run("cornell_box_glass", 48, 48, 2, 8)                              # dynamic-fetch BVH2 kernels, class queues (glass / diffuse)
os.environ["B200PT_WIDE"] = "1"; run("viking_room", 48, 48, 1, 4); del os.environ["B200PT_WIDE"]              # BVH4 + textures
def _queries(name):                                                 # b200pt_trace_query: every shape the scene has, every query kind, with and without stats
    import vpt_b200 as pt
    T = util.product_tracer(name, 16, 16)
    rng = np.random.default_rng(1)
    o = (rng.random((300, 3)) * 6 - 3).astype(np.float32); d = rng.normal(size=(300, 3)).astype(np.float32)
    for shape in pt.PathTracer.TRAV_SHAPES:
        for kind in ("closest", "any", "target"):
            for stats in (True, False):
                try: T.trace_query(shape, kind, o, d, 1e-4, 1e6, target=np.arange(300) % 7, fma=kind != "closest", stats=stats)
                except pt.B200ptError: pass                             # shape absent in this scene (flat walk, BVH4, shared memory)
    print(name, "trace_query ok")
_queries("cornell_box"); _queries("viking_room")
def _shade(name):                                                   # b200pt_shade_query: every class instantiation and the general one, with an extra L
    S = util.oracle_scene(name); T = util.product_tracer(name, 16, 16)
    rng = np.random.default_rng(2)
    o = (rng.normal(size=(300, 3)) * 0.3).astype(np.float32); d = rng.normal(size=(300, 3)); d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    t, prim, inst, uv = S.trace_closest(o, d, 1e-3, 1e5); h = t > 0
    for general in (False, True):
        r = T.shade_query(inst[h], prim[h], uv[h], d[h], o[h], 0.5, np.arange(h.sum()), L=-d[h], force_general=general)
        assert r.shape == (h.sum(), 97)
    print(name, "shade_query ok")
    for kw in (dict(), dict(ShowEnvMapDirectly=0), dict(EnableSkyMIS=0, FurnaceTestMode=1)):   # b200pt_miss_query: every branch of miss_emission
        T = util.product_tracer(name, 16, 16, SkyRotationAzimuth=70.0, SkyRotationAltitude=20.0, **kw)
        r = T.miss_query(d, np.arange(300) % 2, 0.5)
        assert r.shape == (300, 4) and np.isfinite(r).all()
    print(name, "miss_query ok")
_shade("cornell_box"); _shade("cornell_box_glass")
def _bounce():                                                      # b200pt_bounce_query: one fused bounce of 33 paths (a partial second warp)
    import test_bounce_queries as B
    R = B.make_records(B.case_scene("classes"), 33, 4, 5)
    T = util.product_tracer("cornell_box", 8, 8, scene=B.case_scene("classes"), MaxDepth=5)
    out, m = T.bounce_query(R, store=True, carry=True)
    assert out.shape == (33, B.BQ_OUT["STRIDE"]) and int(out[:, B.BQ_OUT["ALIVE"]].sum()) == m
    print("bounce_query ok")
_bounce()
def _update(name, inst, env=None):                                  # instance updates: k_refit_slots / k_refit_level (/ k_refit_wide), and the rebuild path
    for k, v in (env or {}).items(): os.environ[k] = v
    T = util.product_tracer(name, 40, 30, MaxDepth=5)
    T.path_trace(1, util.BASE_SEED)
    xf = T.get_instance_transforms(); xf[inst, 12:15] += (0.3, -0.2, 0.1)
    for rebuild in (False, True, "gpu", False):                         # refit, host rebuild, GPU rebuild (ploc.cu), refit of the GPU tree
        T.update_instance_transforms(xf, rebuild=rebuild); T.path_trace(1, util.BASE_SEED)
        assert np.isfinite(T.get_hdr()).all()
    for k in (env or {}): del os.environ[k]
    print(name, "instance updates ok")
_update("cornell_box", 5); _update("cornell_box_glass", 6); _update("viking_room", 0, {"B200PT_WIDE": "1"})
def _deform(name, mesh):                                            # mesh vertex updates: host input (refit), device input (k_flag_nonfinite, refit + k_refresh_shade)
    import torch
    T = util.product_tracer(name, 40, 30, MaxDepth=5)
    T.path_trace(1, util.BASE_SEED)
    v = T.get_mesh_vertices(mesh).view(np.float32).reshape(-1, 8).copy(); v[:, 0:3] *= 1.1
    T.update_mesh_vertices({mesh: v}); T.path_trace(1, util.BASE_SEED)
    v[:, 0:3] *= 0.9
    T.update_mesh_vertices({mesh: torch.from_numpy(v).cuda(0)}); T.path_trace(1, util.BASE_SEED)
    assert np.isfinite(T.get_hdr()).all()
    print(name, "mesh updates ok")
_deform("cornell_box_glass", 6)
def _post_block():                                                  # fresh handle, unaligned row block, 2-level chain: k_bloom_down_first + k_bloom_final on rows
    import vpt_b200 as pt
    T = pt.PathTracer(0); T.set_scene(util.scene_dict("cornell_box")); T.resize(65, 37)
    T.set_bloom(2.0, 1.0, 2, 5.0)
    rng = np.random.default_rng(4); hdr = np.ones((37, 65, 4), np.float32); hdr[..., :3] = rng.random((37, 65, 3)) * 5
    T.set_hdr(hdr); T.post_process_rows(9, 20); T.get_ldr_rows(9, 20)
    print("post row block ok")
_post_block()
def _pose():                                                        # glTF pose: k_pose_vertices (palette in shared memory), k_pose_normals, refit
    import tempfile, test_gltf_animation as ga
    import vpt_b200 as pt
    with tempfile.TemporaryDirectory() as d:
        import pathlib
        g, blobs, _ = ga.build_scene(); path = ga.write(pathlib.Path(d), g, blobs)
        T = pt.PathTracer(0); T.set_scene_file(path); ga._configure(T); T.resize(40, 30)
        T.path_trace(1, util.BASE_SEED); T.pose(1, 1.3); T.path_trace(1, util.BASE_SEED); T.pose(0, 0.7, rebuild="gpu")
        assert np.isfinite(T.get_hdr()).all()
    print("pose ok")
_pose()
print("sanitize_small done")
