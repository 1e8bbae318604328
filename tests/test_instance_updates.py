"""Instance transform updates (b200pt_update_instance_transforms, the counterpart of TLAS::Update): refit in place or rebuild.

The exact check: closest hits do not depend on the tree (test_traversal_queries.py), every slot record is recomputed with the arithmetic of a
fresh build, and the emissive records come from the same host code, so after an update the image equals, bit for bit, the image of a fresh
handle loaded with the moved scene.  The counters of the work done (paths, rays, hits) must agree too; the launch count may not, since a
fresh handle may choose another traversal shape.
"""
import ctypes as C

import numpy as np
import pytest

import util
import test_traversal_queries as tt

W, H, F, DEPTH = 96, 54, 4, 6
SEED = util.BASE_SEED
WORK = ("paths", "extend_rays", "shade_invocations", "surface_hits", "misses", "shadow_rays")


# ---------------------------------------------------------------- motions (world-space 4x4, applied on the left of an instance's o2w)
def rot(axis, deg):
    a = np.radians(deg); c, s = np.cos(a), np.sin(a)
    i, j = [k for k in range(3) if k != axis]
    m = np.eye(4); m[i, i] = c; m[i, j] = -s; m[j, i] = s; m[j, j] = c
    return m


def trans(t):
    m = np.eye(4); m[:3, 3] = t
    return m


def scale(s):
    return np.diag([s[0], s[1], s[2], 1.0])


def about(m, c):
    """m applied about the point c"""
    return trans(c) @ m @ trans(-np.asarray(c, np.float64))


def o2w(xf):
    return np.asarray(xf, np.float64).reshape(4, 4).T                       # column-major -> row-major


def centre(sc, i):
    xf, m, _ = sc["instances"][i]
    p = sc["meshes"][m][0]["pos"].astype(np.float64)
    w = p @ o2w(xf)[:3, :3].T + o2w(xf)[:3, 3]
    return 0.5 * (w.min(0) + w.max(0))


def moved(sc, motions):
    """copy of the scene dict with instance i's transform replaced by motions[i] @ o2w (float32, column-major as stored)"""
    out = dict(sc); inst = list(sc["instances"])
    for i, m in motions.items():
        xf, mesh, mat = inst[i]
        inst[i] = ((np.asarray(m, np.float64) @ o2w(xf)).T.reshape(-1).astype(np.float32), mesh, mat)
    out["instances"] = inst
    return out


def transforms(sc):
    return np.stack([np.asarray(xf, np.float32).reshape(16) for xf, _, _ in sc["instances"]])


def _cornell_light_mirror(sc):
    return {5: about(rot(1, 30), centre(sc, 5)) @ trans((0.7, -0.2, 0.4)), 0: about(scale((-1, 1, 1)), centre(sc, 0))}


CASES = {   # name: (fixture, extra env, motions)
    "cornell_light_mirror": ("cornell_box", {}, _cornell_light_mirror),
    "glass_sphere": ("cornell_box_glass", {}, lambda sc: {6: about(scale((1.3, 0.7, 1.1)), centre(sc, 6)) @ trans((1.1, 0.4, -0.8))}),
    "glass_sphere_big": ("cornell_box_glass", {"B200PT_SMEM_BIG": "1"}, lambda sc: {6: about(scale((1.3, 0.7, 1.1)), centre(sc, 6)) @ trans((1.1, 0.4, -0.8))}),
    "viking_turn_shear": ("viking_room", {}, lambda sc: {0: about(rot(1, 45) @ np.array([[1, 0.3, 0, 0], [0, 1, 0, 0], [0.2, 0, 1, 0], [0, 0, 0, 1.0]]), centre(sc, 0))}),
    "breakfast_legs": ("breakfast_room", {}, lambda sc: {9: about(rot(1, 30), centre(sc, 9)), 10: trans((0.3, 0.05, -0.2))}),
    "zero_scale": ("cornell_box_glass", {}, lambda sc: {6: about(scale((0, 0, 0)), centre(sc, 6))}),
    "far_1e4": ("cornell_box_glass", {}, lambda sc: {6: trans((1e4, 0, 0))}),
}


@pytest.fixture(scope="module")
def pt():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import vpt_b200
    return vpt_b200


def _env(monkeypatch, env):
    for k in ("B200PT_FLAT_MAX", "B200PT_SMEM_BIG", "B200PT_BVH_SAH", "B200PT_WIDE_STACK", "B200PT_TRAV", "B200PT_WIDE"): monkeypatch.delenv(k, raising=False)
    for k, v in env.items(): monkeypatch.setenv(k, v)


def _tracer(name, scene=None, variance=True, **kw):
    T = util.product_tracer(name, W, H, scene=scene, MaxDepth=DEPTH, **kw)
    if variance: T.set_track_variance(True)
    return T


def _case(name):
    fixture, env, motion = CASES[name]
    sc = util.scene_dict(fixture)
    return fixture, env, sc, moved(sc, motion(sc))


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _hits_on(sc, insts, n=6):
    """a few shading queries per moved instance: rays from outside the triangle's plane onto its centroid"""
    rng = np.random.default_rng(4)
    inst, prim, uv, org, d = [], [], [], [], []
    for i in insts:
        xf, m, _ = sc["instances"][i]
        v, idx = sc["meshes"][m]
        P = v["pos"][np.asarray(idx, np.int64)].reshape(-1, 3, 3).astype(np.float64) @ o2w(xf)[:3, :3].T + o2w(xf)[:3, 3]
        for p in rng.integers(0, len(P), n):
            c = P[p].mean(0); nrm = np.cross(P[p][1] - P[p][0], P[p][2] - P[p][0]); nrm /= max(np.linalg.norm(nrm), 1e-30)
            o = c + 0.5 * nrm
            inst.append(i); prim.append(p); uv.append((0.3, 0.3)); org.append(o); d.append((c - o) / np.linalg.norm(c - o))
    n = len(inst)
    return dict(inst=np.array(inst, np.uint32), prim=np.array(prim, np.uint32), uv=np.array(uv, np.float32), org=np.array(org, np.float32),
                dir=np.array(d, np.float32), pdf=np.full(n, 0.7, np.float32), rng=rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32))


def _shade(T, R):
    return T.shade_query(R["inst"], R["prim"], R["uv"], R["dir"], R["org"], R["pdf"], R["rng"], -R["dir"])


# ---------------------------------------------------------------- CPU: the C-ABI checks its arguments before it needs a GPU
def test_null_handle_or_null_transforms_is_wrong_arguments():
    import vpt_b200 as P
    L = P.lib()
    xf = np.eye(4, dtype=np.float32).reshape(1, 16); n = C.c_uint32()
    assert L.b200pt_update_instance_transforms(None, P.binding._p(xf), 1, 0) == P.binding.ERR_WRONG_ARGUMENTS
    assert L.b200pt_update_instance_transforms(None, None, 1, 1) == P.binding.ERR_WRONG_ARGUMENTS
    assert L.b200pt_get_instance_transforms(None, P.binding._p(xf), 1) == P.binding.ERR_WRONG_ARGUMENTS
    assert L.b200pt_get_instance_transforms(None, None, 1) == P.binding.ERR_WRONG_ARGUMENTS
    assert L.b200pt_instance_count(None, C.byref(n)) == P.binding.ERR_WRONG_ARGUMENTS
    assert L.b200pt_instance_count(None, None) == P.binding.ERR_WRONG_ARGUMENTS
    assert {"b200pt_instance_count", "b200pt_get_instance_transforms", "b200pt_update_instance_transforms"} <= set(P.declared_symbols())


def test_motions_move_what_they_should():
    """the fixtures' instance indices name the objects the cases mean (light, wall, sphere, chair legs)"""
    for name in CASES:
        fixture, _, sc, mv = _case(name)
        changed = [i for i in range(len(sc["instances"])) if not np.array_equal(transforms(sc)[i], transforms(mv)[i])]
        assert changed == sorted(CASES[name][2](sc)), name
    sc = util.scene_dict("cornell_box")
    assert sc["materials"]["EmissiveColor"][sc["instances"][5][2]].max() > 0                   # instance 5 is the light
    det = lambda s: np.linalg.det(o2w(s["instances"][0][0])[:3, :3])
    assert det(sc) * det(_case("cornell_light_mirror")[3]) < 0                                # the wall is mirrored: its orientation flips
    assert len(util.scene_dict("breakfast_room")["meshes"][9][1]) // 3 == 86880                  # the sliver chair legs


# ---------------------------------------------------------------- GPU: a refit equals a fresh scene
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_refit_equals_fresh_scene(pt, name, monkeypatch):
    fixture, env, sc, mv = _case(name)
    _env(monkeypatch, env)
    A = _tracer(fixture)
    A.path_trace(F, SEED)                                   # in flight while the update runs: the update orders itself after these waves
    A.update_instance_transforms(transforms(mv))
    assert A.samples_accumulated() == 0
    assert np.array_equal(A.get_instance_transforms(), transforms(mv))
    A.path_trace(F, SEED)
    B = _tracer(fixture, scene=mv)
    B.path_trace(F, SEED)
    C0 = _tracer(fixture)                                   # the work of A's first call alone
    C0.path_trace(F, SEED)
    a, b = A.get_hdr(), B.get_hdr()
    assert np.array_equal(_bits(a), _bits(b)), (name, int((_bits(a) != _bits(b)).any(-1).sum()))
    ca, cb, c0 = A.counters(), B.counters(), C0.counters()
    assert {k: ca[k] for k in WORK} == {k: cb[k] + c0[k] for k in WORK}
    for x, y in zip(A.denoise_inputs(FeatureSamples=2), B.denoise_inputs(FeatureSamples=2)):
        assert np.array_equal(_bits(x), _bits(y)), name
    motions = CASES[name][2](sc)
    R = _hits_on(mv, sorted(motions))
    assert np.array_equal(_bits(_shade(A, R)), _bits(_shade(B, R))), name


# ---------------------------------------------------------------- GPU: ray by ray against the float64 brute force of the moved triangles
def _quarter_turn(axis, k):
    """exact rotation by k * 90 degrees (a signed permutation: no rounding)"""
    m = np.eye(4); i, j = [a for a in range(3) if a != axis]
    c, s = [(1, 0), (0, 1), (-1, 0), (0, -1)][k % 4]
    m[i, i] = c; m[i, j] = -s; m[j, i] = s; m[j, j] = c
    return m


def _synthetic_motion(name, sc):
    # The boxes of `instances` stay axis-aligned (quarter turns): turned by arbitrary angles, their faces lie within the float64 margins of the
    # exactly axis-aligned rays of the "axis" set so often that one such ray is judged wrong -- for a fresh handle of that scene just as for the
    # refit one, which answers identically.
    n = len(sc["instances"])
    if name == "instances":
        return {i: _quarter_turn(i % 3, i + 1) @ trans((0.3 * i, -0.2, 0.1 * i)) for i in range(n)}
    if name == "instances_mirrored":
        return {i: scale(((-1) ** i, 1, (-1) ** (i // 2))) @ trans((0.1, 0.2 * i, -0.3)) for i in range(n)}
    return {0: rot(2, 35) @ trans((0.2, -0.1, 0.3)) @ scale((1.0, 1.4, 0.8))}


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["instances", "instances_mirrored", "deep", "one_centroid"])
def test_refit_ray_by_ray(pt, name, monkeypatch):
    _env(monkeypatch, {})
    sc = tt.scene_dict("instances" if name == "instances_mirrored" else name)
    mv = moved(sc, _synthetic_motion(name, sc))
    T = pt.PathTracer(0); T.set_scene(sc)
    T.update_instance_transforms(transforms(mv))
    ref = tt.Ref(mv)
    sets = tt.ray_sets(ref, 31, n=300)
    shapes = [s for s in tt.SHAPES if tt._has(T, s, *sets["random"])]
    assert {"shared", "global", "dyn2"} <= set(shapes), shapes
    if name == "deep": assert {"dyn4", "dyn4_spill"} <= set(shapes), shapes
    tt.run_case(T, ref, f"refit/{name}", shapes, sets)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["far_1e4", "zero_scale"])
def test_refit_far_and_vanished_instances_ray_by_ray(pt, name, monkeypatch):
    """far_1e4 moves the scene's largest |coordinate| from ~12 to 1e4: the absolute box pad (2e-6 x that) must grow with it, or rays from far
    out slip past boxes they cross (a refit that keeps the pad of the old bounds fails the edge and far rays here).  zero_scale leaves 960
    degenerate triangles, which no ray may hit.  Every answer must equal a fresh handle's bit for bit, and be right against the float64
    brute force.  On the far16 rays (origins up to 1.6e5 units out) run_case's extra probe -- the same hit again at tmax = t + 1 ulp -- is
    left out: a fresh handle of this scene misses 2 of 400 hits there as well, a property of the traversal that far out, not of the refit."""
    fixture, env, sc, mv = _case(name)
    _env(monkeypatch, env)
    A = pt.PathTracer(0); A.set_scene(sc)
    A.update_instance_transforms(transforms(mv))
    B = pt.PathTracer(0); B.set_scene(mv)
    ref = tt.Ref(mv)
    sets = tt.ray_sets(ref, 41, n=400)
    shapes = [s for s in tt.SHAPES if tt._has(A, s, *sets["random"]) and s != "fixed_origin"]
    assert {"global", "dyn2"} <= set(shapes), shapes
    for set_name, (o, d) in sets.items():
        tmin = np.full(len(o), tt.TMIN[set_name], np.float32); tmax = np.full(len(o), 1e6, np.float32)
        for shape in shapes:
            for fma in (False, True):
                for kind, keys in (("closest", ("t", "prim", "inst", "uv")), ("any", ("occluded",))):
                    ra = A.trace_query(shape, kind, o, d, tmin, tmax, fma=fma); rb = B.trace_query(shape, kind, o, d, tmin, tmax, fma=fma)
                    assert all(np.array_equal(np.asarray(ra[k]).view(np.uint8), np.asarray(rb[k]).view(np.uint8)) for k in keys), (set_name, shape, fma, kind)
    far = sets.pop("far16")
    tt.run_case(A, ref, f"refit/{name}", shapes, sets)
    o, d = far
    tmin = np.full(len(o), tt.TMIN["far16"], np.float32); tmax = np.full(len(o), 1e6, np.float32)
    cls = ref.classify(o, d, tmin, tmax)
    for shape in shapes:
        r = tt.query(A, shape, "closest", o, d, tmin, tmax, fma=True)
        assert not tt.check_closest(ref, cls, ref.gid(r["prim"], r["inst"]), r["t"], r["uv"])[0] and not r["stats"][:, 2].any(), shape
        r = tt.query(A, shape, "any", o, d, tmin, tmax, fma=True)
        assert not tt.check_any(cls, r["occluded"])[0] and not r["stats"][:, 2].any(), shape


@pytest.mark.gpu
def test_refit_breakfast_room_bvh4_ray_by_ray(pt, monkeypatch):
    _env(monkeypatch, {})
    _, _, sc, mv = _case("breakfast_legs")
    T = pt.PathTracer(0); T.set_scene(sc)
    T.update_instance_transforms(transforms(mv))
    ref = tt.Ref(mv)
    rng = np.random.default_rng(5)
    sets = {"random": tt.rays_random(ref, 400, rng), "edges": tt.rays_edges(ref, 150, rng), "surface_nee": tt.rays_from_surface(ref, 150, rng),
            "far16": tt.rays_from_surface(ref, 100, rng, far=16.0)}
    tt.run_case(T, ref, "refit/breakfast_room", ["dyn4", "dyn4_spill"], sets, max_ambiguous=5e-3)


# ---------------------------------------------------------------- GPU: round trip, rebuild
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["glass_sphere", "breakfast_legs"])
def test_round_trip_restores_the_never_moved_image(pt, name, monkeypatch):
    fixture, env, sc, mv = _case(name)
    _env(monkeypatch, env)
    A = _tracer(fixture, variance=False)
    A.update_instance_transforms(transforms(mv)); A.path_trace(1, SEED)
    A.update_instance_transforms(transforms(sc)); A.path_trace(F, SEED)
    B = _tracer(fixture, variance=False); B.path_trace(F, SEED)
    assert np.array_equal(_bits(A.get_hdr()), _bits(B.get_hdr()))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cornell_light_mirror", "glass_sphere", "breakfast_legs"])
def test_rebuild_equals_fresh_scene(pt, name, monkeypatch):
    fixture, env, sc, mv = _case(name)
    _env(monkeypatch, env)
    A = _tracer(fixture, variance=False)
    A.path_trace(1, SEED)
    A.update_instance_transforms(transforms(mv), rebuild=True)
    B = _tracer(fixture, scene=mv, variance=False)
    assert A.scene_stats() == B.scene_stats()
    ref = tt.Ref(mv)
    o, d = tt.rays_random(ref, 2000, np.random.default_rng(9))
    assert np.array_equal(A.trace_stats(o, d, 1e-4, 1e6), B.trace_stats(o, d, 1e-4, 1e6))
    A.path_trace(F, SEED); B.path_trace(F, SEED)
    assert np.array_equal(_bits(A.get_hdr()), _bits(B.get_hdr()))


# ---------------------------------------------------------------- GPU: the contract
@pytest.mark.gpu
def test_rejected_calls_change_nothing(pt, monkeypatch):
    _env(monkeypatch, {})
    fixture, _, sc, mv = _case("glass_sphere")
    E = pt.PathTracer(0)
    with pytest.raises(pt.B200ptError) as e: E.update_instance_transforms(transforms(sc))
    assert e.value.code == pt.binding.ERR_NO_SCENE
    with pytest.raises(pt.B200ptError) as e: E.instance_count()
    assert e.value.code == pt.binding.ERR_NO_SCENE
    A = _tracer(fixture, variance=False)
    assert A.instance_count() == len(sc["instances"])
    A.path_trace(2, SEED)
    bad = [transforms(mv)[:-1], np.concatenate([transforms(mv), transforms(mv)[:1]])]
    for v in (np.nan, np.inf, -np.inf):
        x = transforms(mv).copy(); x[6, 13] = v; bad.append(x)
    x = transforms(mv).copy(); x[3, 15] = np.nan; bad.append(x)                 # row 3 is not used, but a non-finite entry is still refused
    for x in bad:
        for rebuild in (False, True):
            with pytest.raises(pt.B200ptError) as e: A.update_instance_transforms(x, rebuild=rebuild)
            assert e.value.code == pt.binding.ERR_WRONG_ARGUMENTS
    assert np.array_equal(A.get_instance_transforms(), transforms(sc))
    A.path_trace(2, SEED + 1)
    B = _tracer(fixture, variance=False)
    B.path_trace(2, SEED); B.path_trace(2, SEED + 1)
    assert np.array_equal(_bits(A.get_hdr()), _bits(B.get_hdr()))
    assert A.samples_accumulated() == B.samples_accumulated() == 4


@pytest.mark.gpu
def test_adaptive_sampling_after_an_update(pt, monkeypatch):
    fixture, env, sc, mv = _case("glass_sphere")
    _env(monkeypatch, env)
    kw = dict(Enable=1, Threshold=0.05, MinSamples=4, Interval=2)
    A = _tracer(fixture, variance=False); A.set_adaptive(**kw)
    A.path_trace(8, SEED)
    A.update_instance_transforms(transforms(mv))
    A.path_trace(16, SEED)
    B = _tracer(fixture, scene=mv, variance=False); B.set_adaptive(**kw)
    B.path_trace(16, SEED)
    assert np.array_equal(_bits(A.get_hdr()), _bits(B.get_hdr()))
    assert A.active_pixels() == B.active_pixels()


@pytest.mark.gpu
def test_two_ranks_each_updated_give_the_one_rank_image(pt, monkeypatch):
    fixture, env, sc, mv = _case("cornell_light_mirror")
    _env(monkeypatch, env)
    one = _tracer(fixture, scene=mv, variance=False); one.path_trace(F, SEED)
    full = one.get_hdr()
    got = np.zeros_like(full)
    for r in range(2):
        T = _tracer(fixture, variance=False); T.set_partition(r, 2, 16); T.resize(W, H)
        T.path_trace(1, SEED)
        T.update_instance_transforms(transforms(mv))
        T.path_trace(F, SEED)
        got[pt.partition_rows(H, r, 2, 16)] = T.get_hdr()
    assert np.array_equal(_bits(got), _bits(full))


@pytest.mark.gpu
def test_checkpoint_after_an_update_continues_bit_for_bit(pt, monkeypatch, tmp_path):
    fixture, env, sc, mv = _case("glass_sphere")
    _env(monkeypatch, env)
    A = _tracer(fixture, variance=False)
    A.update_instance_transforms(transforms(mv))
    A.path_trace(F, SEED)
    A.save_checkpoint(tmp_path / "a.ckpt")
    A.path_trace(F, SEED)
    B = _tracer(fixture, variance=False)
    B.update_instance_transforms(transforms(mv))
    B.load_checkpoint(tmp_path / "a.ckpt")
    B.path_trace(F, SEED)
    assert np.array_equal(_bits(A.get_hdr()), _bits(B.get_hdr()))
