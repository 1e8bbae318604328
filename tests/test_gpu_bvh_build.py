"""The GPU tree builder: PLOC clustering over the LBVH's Morton-ordered references, SAH leaf formation, depth-first layout, slot permutation and
the BVH4 collapse on the device (csrc/ploc.cu), used by b200pt_update_instance_transforms(rebuild == B200PT_REBUILD_GPU).

CPU: the host restatement (b200pt_bvh2_ploc_build) builds a well-formed tree on adversarial reference sets, rejects what the SAH build
rejects, and stays close to the SAH build's cost on the fixtures.  GPU: the device builder equals the restatement bit for bit and its BVH4
equals the host collapse byte for byte; after a GPU rebuild the image equals a fresh handle's, and every traversal shape answers every
query kind right against the float64 brute force.
"""
import os
import sys

import numpy as np
import pytest

import util
import test_traversal_queries as tt
import test_instance_updates as iu

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "profiles"))
import bvh_lab  # noqa: E402  (numpy mirror of the LBVH's references and Morton order; instance_refit: camera rays)

LEAF_MAX = 4
# SAH cost of the PLOC tree over that of the host binned-SAH build (b200pt_bvh2_sah_build) on the fixtures' references: 0.78 .. 0.9994 measured
# (DESIGN.md section 13, R = 16); the bar allows 5 % above the SAH build
QUALITY_BAR = 1.05


def morton_sorted(rb):
    """reference boxes [n, 6] in the Morton order of bvh_lab's mirror of k_morton (stable sort, as the radix sort)"""
    rb = np.ascontiguousarray(rb, np.float32).reshape(-1, 6)
    return rb[np.argsort(bvh_lab.morton_keys(rb.reshape(-1, 2, 3)), kind="stable")]


def fixture_refs(name):
    """the fixture's references (bvh_lab's mirror of split clipping) in Morton order, and their keys"""
    sc = bvh_lab.load_fixture(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", f"{name}.npz"))
    rb, _ = bvh_lab.split_refs(bvh_lab.world_triangles(sc))
    keys = bvh_lab.morton_keys(rb)
    order = np.argsort(keys, kind="stable")
    return rb[order].reshape(-1, 6).astype(np.float32), keys[order]


def _tris_boxes(tris):
    tris = np.asarray(tris, np.float32)
    return np.concatenate([tris.min(1), tris.max(1)], 1)


def ref_set(name, n=3000):
    rng = np.random.default_rng(ADVERSARIAL.index(name) + 1)
    c = rng.random((n, 3)).astype(np.float32)
    if name == "random":
        e = (0.01 * rng.random((n, 1))).astype(np.float32)
    elif name == "coplanar":
        c[:, 0] = 0.5; e = (0.01 * rng.random((n, 1))).astype(np.float32)
    elif name == "identical":
        c[:] = 0.25; e = np.full((n, 1), 0.01, np.float32)
    elif name == "overlapping":
        e = (0.5 * rng.random((n, 1))).astype(np.float32)
    elif name == "deep":
        return morton_sorted(_tris_boxes(tt.deep_tris()))
    else:
        raise KeyError(name)
    return morton_sorted(np.concatenate([c - e, c + e], 1))


ADVERSARIAL = ["random", "coplanar", "identical", "deep", "overlapping"]


def check_tree(rb, nodes, perm, depth):
    """perm is a permutation; leaves hold 1..4 contiguous slots; nodes = leaves - 1, depth-first with root 0 (left first); depth is the real
    depth; every child box is the padded union of its subtree's reference boxes (bvh_pad_child with the pad of the union of all references,
    its fp32 FMAs evaluated in float64: within one ulp, and never smaller than the union)"""
    n = len(rb)
    assert np.array_equal(np.sort(perm), np.arange(n))
    pabs = np.float64(np.float32(2e-6 * np.float64(np.abs(rb).max()) + 1e-30))
    slots = rb[perm]
    state = dict(next=0, max_d=0, leaves=0)

    def walk(i, d, first):                                              # returns the references below node i
        assert i == state["next"], (i, state["next"])                   # pre-order numbering: root 0, left subtree, then right subtree
        state["next"] += 1; state["max_d"] = max(state["max_d"], d)
        N = nodes[i]; f = first
        for side in (0, 1):
            c = int(N["c1" if side else "c0"])
            if c < 0:
                r = ~c; s, k = r >> 2, (r & 3) + 1
                assert s == f and 1 <= k <= LEAF_MAX
                state["leaves"] += 1; cnt = k
            else:
                cnt = walk(c, d + 1, f)
            lo = slots[f:f + cnt, :3].min(0).astype(np.float64); hi = slots[f:f + cnt, 3:].max(0).astype(np.float64)
            p = (np.float64(np.float32(4e-7)) * np.maximum(np.abs(lo), np.abs(hi)) + pabs).astype(np.float32).astype(np.float64)
            want_lo, want_hi = (lo - p).astype(np.float32), (hi + p).astype(np.float32)
            tol_lo, tol_hi = np.spacing(np.maximum(np.abs(want_lo), p).astype(np.float32)), np.spacing(np.maximum(np.abs(want_hi), p).astype(np.float32))
            got_lo, got_hi = N["lo1" if side else "lo0"], N["hi1" if side else "hi0"]
            assert np.all(np.abs(got_lo - want_lo) <= tol_lo) and np.all(got_lo <= lo), (i, side)
            assert np.all(np.abs(got_hi - want_hi) <= tol_hi) and np.all(got_hi >= hi), (i, side)
            f += cnt
        return f - first

    sys.setrecursionlimit(max(sys.getrecursionlimit(), 10000))
    assert walk(0, 1, 0) == n
    assert state["next"] == len(nodes) == state["leaves"] - 1
    assert state["max_d"] == depth


# ---------------------------------------------------------------- CPU: the host restatement
@pytest.mark.parametrize("name", ADVERSARIAL)
def test_restatement_builds_a_well_formed_tree(name):
    from vpt_b200 import binding as B
    rb = ref_set(name)
    nodes, perm, depth, cost = B.bvh2_ploc_build(rb)
    check_tree(rb, nodes, perm, depth)
    assert cost > 0


@pytest.mark.parametrize("n", [5, 6, 17, 64, 65])
def test_restatement_small_sets(n):
    from vpt_b200 import binding as B
    rb = ref_set("random")[:n]
    nodes, perm, depth, _ = B.bvh2_ploc_build(rb)
    check_tree(rb, nodes, perm, depth)


def test_restatement_rejects_what_the_sah_build_rejects():
    from vpt_b200 import binding as B
    rb = ref_set("random")[:40]
    for n in (1, 2, 4):
        assert len(B.bvh2_ploc_build(rb[:n])[0]) == 0 and len(B.bvh2_sah_build(rb[:n])[0]) == 0
    for v, where in ((np.nan, (3, 1)), (np.nan, (7, 5)), (None, 11)):
        x = rb.copy()
        if v is None: x[where, :3], x[where, 3:] = rb[where, 3:], rb[where, :3] - 0.01     # inverted box
        else: x[where] = v
        assert len(B.bvh2_ploc_build(x)[0]) == 0 and len(B.bvh2_sah_build(x)[0]) == 0
    L = B.lib()
    assert L.b200pt_bvh2_ploc_build(None, 10, None, None, None, None, None) == B.ERR_WRONG_ARGUMENTS
    assert L.b200pt_bvh2_ploc_build_query(None, B._p(rb), len(rb), B._p(rb), B._p(rb), None, None, B._p(rb), None, None) == B.ERR_WRONG_ARGUMENTS
    assert {"b200pt_bvh2_ploc_build", "b200pt_bvh2_ploc_build_query"} <= set(B.declared_symbols())


@pytest.mark.parametrize("name", ["cornell_box", "cornell_box_glass", "viking_room", "breakfast_room"])
def test_restatement_quality_on_the_fixtures(name):
    from vpt_b200 import binding as B
    rb, keys = fixture_refs(name)
    nodes, perm, depth, cost = B.bvh2_ploc_build(rb)
    _, _, _, sah = B.bvh2_sah_build(rb)
    lbvh_cost = B.bvh2_sah_rebuild(bvh_lab.build_lbvh(rb.reshape(-1, 2, 3), keys))[2][0]
    print(f"{name}: PLOC {cost:.3f}  SAH {sah:.3f}  LBVH mirror {lbvh_cost:.3f}  depth {depth}")
    assert cost < lbvh_cost
    assert cost <= QUALITY_BAR * sah, (cost, sah)
    if name != "breakfast_room": check_tree(rb, nodes, perm, depth)


def test_python_rebuild_argument():
    """Python's rebuild values map to the C API's: False / 0 refit, True / 1 host rebuild, "gpu" / 2 (B200PT_REBUILD_GPU) GPU rebuild"""
    import vpt_b200 as pt
    sent = []

    class FakeLib:                                                      # no device needed: records the mode the call passes
        def b200pt_update_instance_transforms(self, h, xf, n, mode): sent.append(mode); return 0

    T = pt.PathTracer.__new__(pt.PathTracer)
    T.L, T.h = FakeLib(), None
    xf = np.eye(4, dtype=np.float32).reshape(1, 16)
    for arg, mode in ((False, 0), (0, 0), (True, 1), (1, 1), ("gpu", 2), (2, 2), (pt.PathTracer.REBUILD_GPU, 2), (np.int32(2), 2)):
        T.update_instance_transforms(xf, rebuild=arg)
        assert sent.pop() == mode, arg
    for bad in ("host", 3, -1, 1.0, None):
        with pytest.raises(ValueError):
            T.update_instance_transforms(xf, rebuild=bad)
    assert not sent
    T.L = None


def test_ties_go_to_the_lower_index():
    """six identical boxes: every distance ties, so each cluster pairs with the lowest position in its window -- positions 0 and 1 merge,
    then the merged cluster absorbs 2, 3, 4, 5 in turn.  The node of 0..3 is the topmost that qualifies as a leaf.  (Ties to the higher
    index would merge 4 and 5 first and make the leaf of 2..5.)"""
    from vpt_b200 import binding as B
    rb = np.tile(np.array([[0.0, 0.0, 0.0, 1.0, 1.0, 1.0]], np.float32), (6, 1))
    nodes, perm, depth, _ = B.bvh2_ploc_build(rb)
    leaf = lambda first, count: ~((first << 2) | (count - 1))
    assert len(nodes) == 2 and depth == 2 and np.array_equal(perm, np.arange(6))
    assert (int(nodes[0]["c0"]), int(nodes[0]["c1"])) == (1, leaf(5, 1))
    assert (int(nodes[1]["c0"]), int(nodes[1]["c1"])) == (leaf(0, 4), leaf(4, 1))


# ---------------------------------------------------------------- GPU: the device builder against the restatement
@pytest.fixture(scope="module")
def pt():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import vpt_b200
    return vpt_b200


HOOK_SETS = ["n5", "n6", "n17", "n1024", "n1025", "n65536", "n65537", "n150000"] + ADVERSARIAL + ["breakfast_room"]


def _hook_refs(name):
    if name == "breakfast_room": return fixture_refs(name)[0]
    if name in ADVERSARIAL: return ref_set(name)
    n = int(name[1:])
    rng = np.random.default_rng(n)
    c = rng.random((n, 3)).astype(np.float32); e = (0.02 * rng.random((n, 1)) / max(1, n / 1000) ** (1 / 3)).astype(np.float32)
    return morton_sorted(np.concatenate([c - e, c + e], 1))


@pytest.mark.gpu
@pytest.mark.parametrize("name", HOOK_SETS)
def test_device_build_equals_restatement(pt, name):
    from vpt_b200 import binding as B
    rb = _hook_refs(name)
    T = pt.PathTracer(0)
    nodes, perm, depth, nodes4, depth4 = T.bvh2_ploc_build_query(rb)
    h_nodes, h_perm, h_depth, _ = B.bvh2_ploc_build(rb)
    assert len(nodes) == len(h_nodes) > 0
    assert nodes.tobytes() == h_nodes.tobytes(), name
    assert np.array_equal(perm, h_perm) and depth == h_depth
    c4, cd4 = B.bvh4_collapse(nodes, 0)
    assert len(nodes4) == len(c4) and nodes4.tobytes() == c4.tobytes() and depth4 == cd4, name


@pytest.mark.gpu
def test_device_build_rejects_what_the_restatement_rejects(pt):
    rb = ref_set("random")[:40]
    T = pt.PathTracer(0)
    for x in (rb[:4], rb[:1]):
        assert len(T.bvh2_ploc_build_query(x)[0]) == 0
    x = rb.copy(); x[5, 2] = np.nan
    assert len(T.bvh2_ploc_build_query(x)[0]) == 0
    x = rb.copy(); x[9, 0] = x[9, 3] + 1
    assert len(T.bvh2_ploc_build_query(x)[0]) == 0


# ---------------------------------------------------------------- GPU: rebuild == 2 in the renderer
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(iu.CASES))
def test_gpu_rebuild_equals_fresh_scene(pt, name, monkeypatch):
    fixture, env, sc, mv = iu._case(name)
    iu._env(monkeypatch, env)
    A = iu._tracer(fixture)
    A.path_trace(iu.F, iu.SEED)                             # in flight while the update runs
    A.update_instance_transforms(iu.transforms(mv), rebuild="gpu")
    assert A.samples_accumulated() == 0
    assert np.array_equal(A.get_instance_transforms(), iu.transforms(mv))
    A.path_trace(iu.F, iu.SEED)
    B = iu._tracer(fixture, scene=mv)
    B.path_trace(iu.F, iu.SEED)
    C0 = iu._tracer(fixture)
    C0.path_trace(iu.F, iu.SEED)
    a, b = A.get_hdr(), B.get_hdr()
    assert np.array_equal(iu._bits(a), iu._bits(b)), (name, int((iu._bits(a) != iu._bits(b)).any(-1).sum()))
    ca, cb, c0 = A.counters(), B.counters(), C0.counters()
    assert {k: ca[k] for k in iu.WORK} == {k: cb[k] + c0[k] for k in iu.WORK}
    R = iu._hits_on(mv, sorted(iu.CASES[name][2](sc)))
    assert np.array_equal(iu._bits(iu._shade(A, R)), iu._bits(iu._shade(B, R))), name


@pytest.mark.gpu
@pytest.mark.parametrize("fixture", ["viking_room", "breakfast_room"])
def test_gpu_rebuild_adopts_the_ploc_tree(pt, fixture, monkeypatch):
    """Closest hits do not depend on the tree, so no image or hit comparison can tell which tree the renderer walks; the traversal work can.
    A GPU rebuild that silently kept the LBVH lbvh_build made (a no-op builder, a depth rule or size guard that always trips) would walk
    exactly what a B200PT_BVH_SAH=0 handle walks.  The adopted tree must visit fewer nodes per camera ray than that LBVH (measured: BreakfastRoom
    15.0 against 26.7, Viking 6.5 against 9.3, DESIGN.md section 13) and stay close to the host level-3 tree (13.9, 6.4)."""
    from instance_refit import camera_rays
    iu._env(monkeypatch, {})
    sc = util.scene_dict(fixture)
    monkeypatch.setenv("B200PT_BVH_SAH", "0")
    L = pt.PathTracer(0); L.set_scene(sc)
    monkeypatch.delenv("B200PT_BVH_SAH")
    H = pt.PathTracer(0); H.set_scene(sc)
    G = pt.PathTracer(0); G.set_scene(sc)
    G.update_instance_transforms(iu.transforms(sc), rebuild="gpu")
    o, d = camera_rays(G)
    sl, sh, sg = (T.trace_stats(o, d, 0.0, 1e30).astype(np.float64) for T in (L, H, G))
    nl, nh, ng = sl[:, 0].mean(), sh[:, 0].mean(), sg[:, 0].mean()
    print(f"{fixture}: nodes per camera ray  LBVH {nl:.2f}  host level 3 {nh:.2f}  GPU {ng:.2f}")
    assert not np.array_equal(sg[:, :2], sl[:, :2])
    assert ng < 0.85 * nl, (ng, nl)
    assert ng < 1.2 * nh, (ng, nh)


def _gpu_rebuilt(pt, name, monkeypatch, extra_env=None):
    T, sc = tt.tracer(pt, name, monkeypatch, extra_env)
    T.update_instance_transforms(iu.transforms(sc), rebuild="gpu")
    return T, sc


@pytest.mark.gpu
@pytest.mark.parametrize("name", tt.SCENES)
def test_gpu_rebuild_ray_by_ray(pt, name, monkeypatch):
    T, sc = _gpu_rebuilt(pt, name, monkeypatch)
    ref = tt.Ref(sc)
    sets = tt.ray_sets(ref, 13)
    shapes = [s for s in tt.SHAPES if tt._has(T, s, *sets["random"])]
    assert {"shared", "global", "dyn2"} <= set(shapes) or name == "cornell_box_glass", shapes
    if name == "deep": assert {"dyn4", "dyn4_spill"} <= set(shapes), shapes      # run_case: zero refused pushes with the depth rule's stack
    tt.run_case(T, ref, f"gpu/{name}", shapes, sets)


@pytest.mark.gpu
def test_gpu_rebuild_breakfast_room_ray_by_ray(pt, monkeypatch):
    T, sc = _gpu_rebuilt(pt, "breakfast_room", monkeypatch)
    ref = tt.Ref(sc)
    rng = np.random.default_rng(23)
    sets = {"random": tt.rays_random(ref, 600, rng), "edges": tt.rays_edges(ref, 200, rng), "axis": tt.rays_axis(ref, 200, rng),
            "surface": tt.rays_from_surface(ref, 200, rng), "surface_nee": tt.rays_from_surface(ref, 200, rng), "far16": tt.rays_from_surface(ref, 150, rng, far=16.0)}
    tt.run_case(T, ref, "gpu/breakfast_room", ["global", "dyn2", "dyn4", "dyn4_spill"], sets, max_ambiguous=5e-3)


@pytest.mark.gpu
def test_refit_after_gpu_rebuild_equals_fresh_scene(pt, monkeypatch):
    """the refit's BVH4 source map is re-derived by the host collapse: a device collapse that ordered nodes differently would refit wrong boxes"""
    iu._env(monkeypatch, {})
    _, _, sc, mv = iu._case("breakfast_legs")
    mv2 = iu.moved(sc, {9: iu.about(iu.rot(1, 45), iu.centre(sc, 9)), 10: iu.trans((0.1, 0.0, 0.2))})
    A = pt.PathTracer(0); A.set_scene(sc)
    A.update_instance_transforms(iu.transforms(mv), rebuild="gpu")
    A.update_instance_transforms(iu.transforms(mv2))
    B = pt.PathTracer(0); B.set_scene(mv2)
    ref = tt.Ref(mv2)
    rng = np.random.default_rng(29)
    sets = {"random": tt.rays_random(ref, 400, rng), "edges": tt.rays_edges(ref, 150, rng), "surface_nee": tt.rays_from_surface(ref, 150, rng)}
    for set_name, (o, d) in sets.items():
        tmin = np.full(len(o), tt.TMIN[set_name], np.float32); tmax = np.full(len(o), 1e6, np.float32)
        for shape in ("dyn4", "dyn4_spill", "global"):
            ra = A.trace_query(shape, "closest", o, d, tmin, tmax, fma=True); rb = B.trace_query(shape, "closest", o, d, tmin, tmax, fma=True)
            assert all(np.array_equal(np.asarray(ra[k]).view(np.uint8), np.asarray(rb[k]).view(np.uint8)) for k in ("t", "prim", "inst", "uv")), (set_name, shape)
    tt.run_case(A, ref, "gpu+refit/breakfast_room", ["dyn4", "dyn4_spill"], sets, max_ambiguous=5e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["glass_sphere", "breakfast_legs"])
def test_gpu_rebuild_with_unchanged_transforms_keeps_the_image(pt, name, monkeypatch):
    fixture, env, sc, _ = iu._case(name)
    iu._env(monkeypatch, env)
    A = iu._tracer(fixture, variance=False)
    A.path_trace(iu.F, iu.SEED)
    before = A.get_hdr()
    A.update_instance_transforms(iu.transforms(sc), rebuild="gpu")
    A.path_trace(iu.F, iu.SEED)
    assert np.array_equal(iu._bits(A.get_hdr()), iu._bits(before))


@pytest.mark.gpu
def test_gpu_rebuild_rejected_calls_change_nothing(pt, monkeypatch):
    iu._env(monkeypatch, {})
    fixture, _, sc, mv = iu._case("glass_sphere")
    E = pt.PathTracer(0)
    with pytest.raises(pt.B200ptError) as e: E.update_instance_transforms(iu.transforms(sc), rebuild="gpu")
    assert e.value.code == pt.binding.ERR_NO_SCENE
    A = iu._tracer(fixture, variance=False)
    A.path_trace(2, iu.SEED)
    bad = [iu.transforms(mv)[:-1], np.concatenate([iu.transforms(mv), iu.transforms(mv)[:1]])]
    for v in (np.nan, np.inf, -np.inf):
        x = iu.transforms(mv).copy(); x[6, 13] = v; bad.append(x)
    x = iu.transforms(mv).copy(); x[3, 15] = np.nan; bad.append(x)
    for x in bad:
        with pytest.raises(pt.B200ptError) as e: A.update_instance_transforms(x, rebuild="gpu")
        assert e.value.code == pt.binding.ERR_WRONG_ARGUMENTS
    assert np.array_equal(A.get_instance_transforms(), iu.transforms(sc))
    A.path_trace(2, iu.SEED + 1)
    B = iu._tracer(fixture, variance=False)
    B.path_trace(2, iu.SEED); B.path_trace(2, iu.SEED + 1)
    assert np.array_equal(iu._bits(A.get_hdr()), iu._bits(B.get_hdr()))
    assert A.samples_accumulated() == B.samples_accumulated() == 4
