"""Mesh vertex updates (b200pt_update_mesh_vertices): skinning, cloth, morph targets without a scene load; refit, GPU rebuild or host rebuild.

The exact check is the one of test_instance_updates.py: closest hits do not depend on the tree, and after an update every slot record,
shading record and emissive record comes from the arithmetic of a fresh build, so the image equals, bit for bit, the image of a fresh handle
loaded with the deformed scene.  The work counters agree too (the launch count excepted).  Normals of deformed meshes are recomputed here.
"""
import ctypes as C

import numpy as np
import pytest

import util
import test_traversal_queries as tt
import test_instance_updates as ti

W, H, F, DEPTH = ti.W, ti.H, ti.F, ti.DEPTH
SEED = util.BASE_SEED
REBUILDS = {"refit": False, "gpu": "gpu", "host": True}


# ---------------------------------------------------------------- deformations (object space, float64, stored as float32)
def vertex_normals(pos, idx):
    """area-weighted vertex normals; a vertex whose triangles have no area keeps (0, 0, 1)"""
    p = pos.astype(np.float64); t = np.asarray(idx, np.int64).reshape(-1, 3)
    fn = np.cross(p[t[:, 1]] - p[t[:, 0]], p[t[:, 2]] - p[t[:, 0]])
    n = np.zeros_like(p)
    for k in range(3): np.add.at(n, t[:, k], fn)
    ln = np.linalg.norm(n, axis=1, keepdims=True)
    return np.where(ln > 0, n / np.maximum(ln, 1e-300), np.array([0.0, 0.0, 1.0]))


def deformed(v, idx, pos=None, uv_shift=None, normals=True):
    out = v.copy()
    if pos is not None:
        out["pos"] = pos.astype(np.float32)
        if normals: out["nrm"] = vertex_normals(out["pos"], idx).astype(np.float32)
    if uv_shift is not None: out["uv"] = (v["uv"].astype(np.float64) + uv_shift).astype(np.float32)
    return out


def _light_corner(v, idx):
    # the quad turns non-planar and its area changes; object -y is world +y here, away from the ceiling into the box, so the light stays visible
    p = v["pos"].astype(np.float64).copy(); p[0] += (0.2, -0.15, -0.1)
    return deformed(v, idx, p, normals=False)


LIGHT_MOTION = {5: ti.trans((0.3, 0.1, 0.2))}                                 # world +y: further below the ceiling, into the box


def _below_ceiling(sc):
    """every vertex of the Cornell light (instance 5) lies inside the box, below the ceiling (instance 3), which covers its x / z extent"""
    def world(i):
        xf, m, _ = sc["instances"][i]
        return sc["meshes"][m][0]["pos"].astype(np.float64) @ ti.o2w(xf)[:3, :3].T + ti.o2w(xf)[:3, 3]
    light, ceil = world(5), world(3)
    covered = (ceil.min(0)[[0, 2]] <= light.min(0)[[0, 2]]).all() and (light.max(0)[[0, 2]] <= ceil.max(0)[[0, 2]]).all()
    return covered and light[:, 1].min() > ceil[:, 1].max()


def _wobble(v, idx):
    p = v["pos"].astype(np.float64); c = p.mean(0); r = p - c
    d = r / np.maximum(np.linalg.norm(r, axis=1, keepdims=True), 1e-30)
    return deformed(v, idx, c + r * (1.0 + 0.15 * np.sin(5.0 * d[:, 0]) * np.cos(3.0 * d[:, 1]))[:, None])


def _twist(v, idx):
    p = v["pos"].astype(np.float64); y = (p[:, 1] - p[:, 1].min()) / np.ptp(p[:, 1])
    a = 0.6 * y; c, s = np.cos(a), np.sin(a)
    q = p.copy(); q[:, 0] = c * p[:, 0] - s * p[:, 2]; q[:, 2] = s * p[:, 0] + c * p[:, 2]
    return deformed(v, idx, q, uv_shift=(0.13, -0.07))


def _bend(v, idx):
    p = v["pos"].astype(np.float64).copy(); z = (p[:, 2] - p[:, 2].min()) / np.ptp(p[:, 2])
    p[:, 1] += 0.4 * z ** 2
    return deformed(v, idx, p)


def _collapse(v, idx):
    p = v["pos"].astype(np.float64)
    return deformed(v, idx, np.repeat(p.mean(0, keepdims=True), len(p), 0), normals=False)


def _far(v, idx):
    return deformed(v, idx, v["pos"].astype(np.float64) + (1e4, 0.0, 0.0), normals=False)


def _with_second_sphere(sc):
    out = dict(sc); inst = list(sc["instances"])
    xf, m, mat = inst[6]
    inst.append(((ti.trans((-1.2, 0.3, 0.9)) @ ti.o2w(xf)).T.reshape(-1).astype(np.float32), m, mat))
    out["instances"] = inst
    return out


CASES = {   # name: (fixture, extra env, instance whose mesh is deformed, deformation, scene edit before loading)
    "cornell_light": ("cornell_box", {}, 5, _light_corner, None),
    "glass_sphere": ("cornell_box_glass", {}, 6, _wobble, None),
    "glass_sphere_big": ("cornell_box_glass", {"B200PT_SMEM_BIG": "1"}, 6, _wobble, None),
    "viking_twist": ("viking_room", {}, 0, _twist, None),
    "breakfast_legs": ("breakfast_room", {}, 9, _bend, None),
    "shared_mesh": ("cornell_box_glass", {}, 6, _wobble, _with_second_sphere),
    "collapsed": ("cornell_box_glass", {}, 6, _collapse, None),
    "far_1e4": ("cornell_box_glass", {}, 6, _far, None),
}


def with_meshes(sc, new):
    """copy of the scene dict with mesh m's vertices replaced by new[m]"""
    out = dict(sc); ms = list(sc["meshes"])
    for m, v in new.items(): ms[m] = (v, ms[m][1])
    out["meshes"] = ms
    return out


def _case(name):
    fixture, env, inst, deform, edit = CASES[name]
    sc = util.scene_dict(fixture)
    if edit: sc = edit(sc)
    m = sc["instances"][inst][1]
    v, idx = sc["meshes"][m]
    new = {m: deform(v, idx)}
    return fixture, env, sc, with_meshes(sc, new), new


def _insts_of(sc, meshes):
    return [i for i, (_, m, _) in enumerate(sc["instances"]) if m in meshes]


def _as_rows(v):
    return np.ascontiguousarray(v).view(np.float32).reshape(-1, 8)


@pytest.fixture(scope="module")
def pt():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import vpt_b200
    return vpt_b200


_bits = ti._bits
_env = ti._env


def _tracer(name, scene, variance=True):
    return ti._tracer(name, scene=scene, variance=variance)


# ---------------------------------------------------------------- CPU
def test_null_handle_or_null_arguments_is_wrong_arguments():
    import vpt_b200 as P
    L = P.lib(); E = P.binding.ERR_WRONG_ARGUMENTS
    v = np.zeros((4, 8), np.float32); n = C.c_uint32()
    ups = (P.binding.MeshUpdate * 1)(P.binding.MeshUpdate(0, 4, v.ctypes.data))
    assert L.b200pt_update_mesh_vertices(None, C.addressof(ups), 1, 0, 0) == E
    assert L.b200pt_update_mesh_vertices(None, None, 1, 0, 0) == E
    assert L.b200pt_get_mesh_vertices(None, 0, P.binding._p(v), 4) == E
    assert L.b200pt_get_mesh_vertices(None, 0, None, 4) == E
    assert L.b200pt_mesh_vertex_count(None, 0, C.byref(n)) == E
    assert L.b200pt_mesh_vertex_count(None, 0, None) == E
    assert L.b200pt_mesh_count(None, C.byref(n)) == E
    assert L.b200pt_mesh_count(None, None) == E
    assert {"b200pt_mesh_count", "b200pt_mesh_vertex_count", "b200pt_get_mesh_vertices", "b200pt_update_mesh_vertices"} <= set(P.declared_symbols())
    assert C.sizeof(P.binding.MeshUpdate) == 16 and P.binding.VERTEX_DTYPE.itemsize == 32


def test_deformations_change_what_they_should():
    for name in CASES:
        _, _, sc, mv, new = _case(name)
        (m, v), = new.items()
        old = sc["meshes"][m][0]
        assert np.isfinite(_as_rows(v)).all() and not np.array_equal(_as_rows(v), _as_rows(old)), name
        assert all(np.array_equal(a[1], b[1]) for a, b in zip(sc["meshes"], mv["meshes"])), name          # topology stays
    sc = util.scene_dict("cornell_box")
    assert sc["materials"]["EmissiveColor"][sc["instances"][5][2]].max() > 0                            # instance 5 is the light
    v = _case("cornell_light")[4][5]; P = v["pos"].astype(np.float64)[np.asarray(sc["meshes"][5][1], np.int64)].reshape(-1, 3, 3)
    nrm = np.cross(P[:, 1] - P[:, 0], P[:, 2] - P[:, 0])
    assert abs(np.dot(nrm[0], nrm[1])) < 0.999 * np.linalg.norm(nrm[0]) * np.linalg.norm(nrm[1])      # non-planar
    mv = _case("cornell_light")[3]
    assert _below_ceiling(sc) and _below_ceiling(mv) and _below_ceiling(ti.moved(mv, LIGHT_MOTION))           # the light stays visible
    assert len(_insts_of(_case("shared_mesh")[2], {6})) == 2


# ---------------------------------------------------------------- GPU: an update equals a fresh scene
@pytest.mark.gpu
@pytest.mark.parametrize("rebuild", list(REBUILDS))
@pytest.mark.parametrize("name", list(CASES))
def test_update_equals_fresh_scene(pt, name, rebuild, monkeypatch):
    fixture, env, sc, mv, new = _case(name)
    _env(monkeypatch, env)
    A = _tracer(fixture, sc)
    A.path_trace(F, SEED)                                   # in flight while the update runs: the update orders itself after these waves
    A.update_mesh_vertices(new, rebuild=REBUILDS[rebuild])
    assert A.samples_accumulated() == 0
    for m, v in new.items(): assert np.array_equal(_as_rows(A.get_mesh_vertices(m)), _as_rows(v))
    A.path_trace(F, SEED)
    B = _tracer(fixture, mv)
    B.path_trace(F, SEED)
    C0 = _tracer(fixture, sc)                               # the work of A's first call alone
    C0.path_trace(F, SEED)
    a, b = A.get_hdr(), B.get_hdr()
    assert np.array_equal(_bits(a), _bits(b)), (name, rebuild, int((_bits(a) != _bits(b)).any(-1).sum()))
    ca, cb, c0 = A.counters(), B.counters(), C0.counters()
    assert {k: ca[k] for k in ti.WORK} == {k: cb[k] + c0[k] for k in ti.WORK}
    for x, y in zip(A.denoise_inputs(FeatureSamples=2), B.denoise_inputs(FeatureSamples=2)):
        assert np.array_equal(_bits(x), _bits(y)), name
    if name != "collapsed":                                 # a collapsed triangle has no plane to aim a query ray at
        R = ti._hits_on(mv, _insts_of(mv, set(new)))
        assert np.array_equal(_bits(ti._shade(A, R)), _bits(ti._shade(B, R))), name


# ---------------------------------------------------------------- GPU: ray by ray against the float64 brute force of the deformed triangles
@pytest.mark.gpu
@pytest.mark.parametrize("rebuild", list(REBUILDS))
@pytest.mark.parametrize("name", list(CASES))
def test_update_ray_by_ray(pt, name, rebuild, monkeypatch):
    fixture, env, sc, mv, new = _case(name)
    _env(monkeypatch, env)
    A = pt.PathTracer(0); A.set_scene(sc)
    A.update_mesh_vertices(new, rebuild=REBUILDS[rebuild])
    ref = tt.Ref(mv)
    if fixture == "breakfast_room":                         # as test_instance_updates: the BVH4 walks, the sliver legs' wider margins
        rng = np.random.default_rng(5)
        sets = {"random": tt.rays_random(ref, 400, rng), "edges": tt.rays_edges(ref, 150, rng), "surface_nee": tt.rays_from_surface(ref, 150, rng),
                "far16": tt.rays_from_surface(ref, 100, rng, far=16.0)}
        tt.run_case(A, ref, f"{rebuild}/{name}", ["dyn4", "dyn4_spill"], sets, max_ambiguous=5e-3)
        return
    B = pt.PathTracer(0); B.set_scene(mv)
    sets = tt.ray_sets(ref, 43, n=300)
    shapes = [s for s in tt.SHAPES if tt._has(A, s, *sets["random"])]
    # every traversal answer equals a fresh handle's, bit for bit
    for set_name, (o, d) in sets.items():
        tmin = np.full(len(o), tt.TMIN[set_name], np.float32); tmax = np.full(len(o), 1e6, np.float32)
        for shape in shapes:
            if shape == "fixed_origin": continue
            for fma in ((False, True) if shape != "flat" else (False,)):
                for kind, keys in (("closest", ("t", "prim", "inst", "uv")), ("any", ("occluded",))):
                    ra = A.trace_query(shape, kind, o, d, tmin, tmax, fma=fma); rb = B.trace_query(shape, kind, o, d, tmin, tmax, fma=fma)
                    assert all(np.array_equal(np.asarray(ra[k]).view(np.uint8), np.asarray(rb[k]).view(np.uint8)) for k in keys), (set_name, shape, fma, kind)
    # far16 without run_case's extra probes (test_instance_updates: a fresh handle misses a few far hits there too)
    o, d = sets.pop("far16")
    tt.run_case(A, ref, f"{rebuild}/{name}", shapes, sets)
    tmin = np.full(len(o), tt.TMIN["far16"], np.float32); tmax = np.full(len(o), 1e6, np.float32)
    cls = ref.classify(o, d, tmin, tmax)
    for shape in shapes:
        if shape in ("fixed_origin", "flat"): continue
        r = tt.query(A, shape, "closest", o, d, tmin, tmax, fma=True)
        assert not tt.check_closest(ref, cls, ref.gid(r["prim"], r["inst"]), r["t"], r["uv"])[0] and not r["stats"][:, 2].any(), shape
        r = tt.query(A, shape, "any", o, d, tmin, tmax, fma=True)
        assert not tt.check_any(cls, r["occluded"])[0] and not r["stats"][:, 2].any(), shape


# ---------------------------------------------------------------- GPU: device input, the host mirror, sequences
def _tensor(v):
    import torch
    return torch.from_numpy(_as_rows(v).copy()).cuda(0)


@pytest.mark.gpu
@pytest.mark.parametrize("rebuild", list(REBUILDS))
def test_device_input_equals_host_input(pt, rebuild, monkeypatch):
    fixture, env, sc, mv, new = _case("viking_twist")
    _env(monkeypatch, env)
    A = _tracer(fixture, sc, variance=False); A.path_trace(1, SEED)
    A.update_mesh_vertices(new, rebuild=REBUILDS[rebuild]); A.path_trace(F, SEED)
    D = _tracer(fixture, sc, variance=False); D.path_trace(1, SEED)
    D.update_mesh_vertices({m: _tensor(v) for m, v in new.items()}, rebuild=REBUILDS[rebuild]); D.path_trace(F, SEED)
    for m in new: assert np.array_equal(_as_rows(A.get_mesh_vertices(m)), _as_rows(D.get_mesh_vertices(m)))
    assert np.array_equal(_bits(A.get_hdr()), _bits(D.get_hdr()))


@pytest.mark.gpu
def test_device_input_keeps_the_host_mirror_for_a_later_instance_update(pt, monkeypatch):
    """the emissive records of an instance update come from the host copy of the meshes: a device-input update must have written it"""
    fixture, env, sc, mv, new = _case("cornell_light")
    _env(monkeypatch, env)
    motion = LIGHT_MOTION
    A = _tracer(fixture, sc, variance=False); A.path_trace(1, SEED)
    A.update_mesh_vertices({m: _tensor(v) for m, v in new.items()})
    A.update_instance_transforms(ti.transforms(ti.moved(mv, motion)))
    A.path_trace(F, SEED)
    B = _tracer(fixture, ti.moved(mv, motion), variance=False); B.path_trace(F, SEED)
    assert np.array_equal(_bits(A.get_hdr()), _bits(B.get_hdr()))


@pytest.mark.gpu
@pytest.mark.parametrize("rebuild", list(REBUILDS))
def test_deform_move_deform_equals_fresh_scene(pt, rebuild, monkeypatch):
    fixture, env, sc, mv, new = _case("shared_mesh")
    _env(monkeypatch, env)
    (m, v1), = new.items()
    v2 = _twist(sc["meshes"][m][0], sc["meshes"][m][1])
    motion = {6: ti.about(ti.rot(1, 30), ti.centre(sc, 6)), 7: ti.trans((0.2, -0.3, 0.1))}
    A = _tracer(fixture, sc, variance=False); A.path_trace(1, SEED)
    A.update_mesh_vertices({m: v1}, rebuild=REBUILDS[rebuild]); A.path_trace(1, SEED)
    A.update_instance_transforms(ti.transforms(ti.moved(sc, motion)), rebuild=REBUILDS[rebuild]); A.path_trace(1, SEED)
    A.update_mesh_vertices({m: _tensor(v2)}, rebuild=REBUILDS[rebuild]); A.path_trace(F, SEED)
    fin = with_meshes(ti.moved(sc, motion), {m: v2})
    B = _tracer(fixture, fin, variance=False); B.path_trace(F, SEED)
    assert np.array_equal(_bits(A.get_hdr()), _bits(B.get_hdr()))
    R = ti._hits_on(fin, [6, 7])
    assert np.array_equal(_bits(ti._shade(A, R)), _bits(ti._shade(B, R)))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["glass_sphere", "breakfast_legs"])
def test_round_trip_restores_the_original_image(pt, name, monkeypatch):
    fixture, env, sc, mv, new = _case(name)
    _env(monkeypatch, env)
    A = _tracer(fixture, sc, variance=False)
    A.update_mesh_vertices(new); A.path_trace(1, SEED)
    A.update_mesh_vertices({m: sc["meshes"][m][0] for m in new}); A.path_trace(F, SEED)
    B = _tracer(fixture, sc, variance=False); B.path_trace(F, SEED)
    assert np.array_equal(_bits(A.get_hdr()), _bits(B.get_hdr()))


@pytest.mark.gpu
def test_several_meshes_in_one_batch(pt, monkeypatch):
    """every mesh of BreakfastRoom at once: one tree update for the batch"""
    _env(monkeypatch, {})
    sc = util.scene_dict("breakfast_room")
    new = {m: _wobble(v, idx) for m, (v, idx) in enumerate(sc["meshes"]) if len(v) >= 3}
    mv = with_meshes(sc, new)
    A = _tracer("breakfast_room", sc, variance=False); A.path_trace(1, SEED)
    A.update_mesh_vertices(new, rebuild="gpu"); A.path_trace(2, SEED)
    B = _tracer("breakfast_room", mv, variance=False); B.path_trace(2, SEED)
    assert np.array_equal(_bits(A.get_hdr()), _bits(B.get_hdr()))


# ---------------------------------------------------------------- GPU: the contract
@pytest.mark.gpu
def test_rejected_calls_change_nothing(pt, monkeypatch):
    import torch
    _env(monkeypatch, {})
    fixture, _, sc, mv, new = _case("glass_sphere")
    (m, v), = new.items()
    E = pt.PathTracer(0)
    for call in (lambda: E.update_mesh_vertices(new), E.mesh_count, lambda: E.get_mesh_vertices(0)):
        with pytest.raises(pt.B200ptError) as e: call()
        assert e.value.code == pt.binding.ERR_NO_SCENE
    A = _tracer(fixture, sc, variance=False)
    assert A.mesh_count() == len(sc["meshes"])
    A.path_trace(2, SEED)
    c_before = A.counters()
    nan = _as_rows(v).copy(); nan[7, 1] = np.nan
    inf = _as_rows(v).copy(); inf[3, 6] = -np.inf                          # a UV component
    bad0 = _as_rows(sc["meshes"][0][0]).copy(); bad0[-1, 0] = np.inf        # the second update of a batch whose first is valid
    bad = [{m: _as_rows(v)[:-1]}, {m: np.concatenate([_as_rows(v), _as_rows(v)[:1]])}, {m: nan}, {m: inf},
           {len(sc["meshes"]): _as_rows(v)}, {-1: _as_rows(v)}, {m: _as_rows(v), 0: bad0},
           {m: torch.from_numpy(nan).cuda(0)}, {m: torch.from_numpy(inf).cuda(0)},
           {m: torch.from_numpy(_as_rows(v).copy()).cuda(0), 0: torch.from_numpy(bad0).cuda(0)}]
    for x in bad:
        for rebuild in REBUILDS.values():
            with pytest.raises(pt.B200ptError) as e: A.update_mesh_vertices(x, rebuild=rebuild)
            assert e.value.code == pt.binding.ERR_WRONG_ARGUMENTS, x.keys()
    # a repeated mesh, a null vertex pointer and an empty batch go through the C ABI directly
    L = pt.lib(); rows = _as_rows(v)
    ups = (pt.binding.MeshUpdate * 2)(pt.binding.MeshUpdate(m, len(rows), rows.ctypes.data), pt.binding.MeshUpdate(m, len(rows), rows.ctypes.data))
    for dev in (0, 1):
        assert L.b200pt_update_mesh_vertices(A.h, C.addressof(ups), 2, dev, 0) == pt.binding.ERR_WRONG_ARGUMENTS
    ups[0].vertices = None
    assert L.b200pt_update_mesh_vertices(A.h, C.addressof(ups), 1, 0, 0) == pt.binding.ERR_WRONG_ARGUMENTS
    assert L.b200pt_update_mesh_vertices(A.h, C.addressof(ups), 0, 0, 0) == pt.binding.ERR_WRONG_ARGUMENTS
    assert L.b200pt_get_mesh_vertices(A.h, m, P_(rows), len(rows) - 1) == pt.binding.ERR_WRONG_ARGUMENTS
    with pytest.raises(ValueError): A.update_mesh_vertices(new, rebuild=3)
    with pytest.raises(ValueError): A.update_mesh_vertices({m: _as_rows(v)[:, :6]})
    assert A.counters() == c_before
    for k, (vk, _) in enumerate(sc["meshes"]): assert np.array_equal(_as_rows(A.get_mesh_vertices(k)), _as_rows(vk))
    A.path_trace(2, SEED + 1)
    B = _tracer(fixture, sc, variance=False)
    B.path_trace(2, SEED); B.path_trace(2, SEED + 1)
    assert np.array_equal(_bits(A.get_hdr()), _bits(B.get_hdr()))
    assert A.samples_accumulated() == B.samples_accumulated() == 4


def P_(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.mark.gpu
def test_adaptive_sampling_after_an_update(pt, monkeypatch):
    fixture, env, sc, mv, new = _case("glass_sphere")
    _env(monkeypatch, env)
    kw = dict(Enable=1, Threshold=0.05, MinSamples=4, Interval=2)
    A = _tracer(fixture, sc, variance=False); A.set_adaptive(**kw)
    A.path_trace(8, SEED)
    A.update_mesh_vertices(new)
    assert A.samples_accumulated() == 0
    A.path_trace(16, SEED)
    B = _tracer(fixture, mv, variance=False); B.set_adaptive(**kw)
    B.path_trace(16, SEED)
    assert np.array_equal(_bits(A.get_hdr()), _bits(B.get_hdr()))
    assert A.active_pixels() == B.active_pixels()
