"""Every traversal shape and query kind the renderer issues, checked ray by ray against a float64 brute force (b200pt_trace_query).

Reference: Moeller-Trumbore in float64 on the triangle records the GPU stores (world vertices transformed in fp32 exactly as k_world_tris does,
edges rounded to fp32), over all triangles.  Each (ray, triangle) pair is classified with margins derived from the operand magnitudes of the
fp32 evaluation (u = tv.p / det, v = d.q / det, t = e2.q / det with p = d x e2, q = tv x e1).  The rounding of p and q is bounded by
the magnitudes of their operands, P = |d||e2| and Q = |tv||e1| (not by |p|, |q|, which vanish for nearly parallel operands):

    eps_u = K * 2^-24 * (|tv| P + |u||e1| P) / |det|,   eps_v = K * 2^-24 * (|d| Q + |v||e1| P) / |det|,
    eps_t = K * 2^-24 * (|e2| Q + |t||e1| P) / |det| + K * 2^-24 * tmin,   K = EPS_K

  required:   u >= eps_u, v >= eps_v, u + v <= 1 - (eps_u + eps_v), tmin + eps_t < t < tmax - eps_t
  admissible: the same bounds at -eps.

A closest-hit answer passes when its triangle is admissible, no required triangle is closer by more than eps_t, it misses only when nothing is
required, and among bit-identical duplicate triangles it names the lowest id (exact).  Any-hit answers: occluded needs an admissible occluder,
not occluded needs no required one.  TARGET (light visibility) queries also check the tie rule on duplicates of the target exactly.
The values of a required hit are checked too: |t - t_ref| <= eps_t + VALUE_ULPS ulp(t_ref), and u, v likewise with eps_u, eps_v.
Every query runs twice, through the renderer's own instantiations and through the counting ones (stats), and both must agree bit for bit.
EPS_K is tight: test_margin_is_tight asserts that EPS_K / 10 rejects some GPU answer on rays aimed at shared edges and vertices.
"""
import numpy as np
import pytest

import util
from util import gltf_ref

EPS_K = 8.0
VALUE_ULPS = 4
U = 2.0 ** -24

SHAPES = ("shared", "global", "flat", "fixed_origin", "dyn2", "dyn4", "dyn4_spill")


# ---------------------------------------------------------------- scenes (dicts for PathTracer.set_scene)
def _mesh(tris):
    tris = np.asarray(tris, np.float32).reshape(-1, 3, 3)
    v = np.zeros(3 * len(tris), gltf_ref.VERTEX_DTYPE)
    v["pos"] = tris.reshape(-1, 3); v["nrm"] = (0.0, 0.0, 1.0)
    return v, np.arange(3 * len(tris), dtype=np.uint32)


def _scene(meshes, instances=None):
    """meshes: list of [n, 3, 3] triangle arrays; instances: [(4x4 row-major transform, mesh)] (default: each mesh once, identity)"""
    mats = np.zeros(1, gltf_ref.MATERIAL_DTYPE)
    mats["BaseColor"] = 0.5; mats["Roughness"] = 0.5; mats["IOR"] = 1.5
    for k in ("BaseColorTextureIndex", "NormalTextureIndex", "RoughnessTextureIndex", "MetallicTextureIndex", "EmissiveTextureIndex"): mats[k] = 0
    if instances is None: instances = [(np.eye(4), i) for i in range(len(meshes))]
    return {"meshes": [_mesh(m) for m in meshes], "materials": mats, "textures": [np.full((1, 1, 4), 255, np.uint8)],
            "instances": [(np.asarray(x, np.float32).T.reshape(-1), m, 0) for x, m in instances],
            "camera_view": np.eye(4, dtype=np.float32).reshape(-1), "aspect": 1.0}


def _box_mesh(lo, hi, n=3):
    """closed axis-aligned box, each face an n x n grid of quads (shared edges and vertices everywhere)"""
    lo = np.asarray(lo, np.float64); hi = np.asarray(hi, np.float64); out = []
    g = np.linspace(0.0, 1.0, n + 1)
    for ax in range(3):
        a, b = [k for k in range(3) if k != ax]
        for side in (0.0, 1.0):
            for i in range(n):
                for j in range(n):
                    def P(s, t):
                        p = np.empty(3); p[ax] = side; p[a] = s; p[b] = t
                        return lo + p * (hi - lo)
                    p00, p10, p01, p11 = P(g[i], g[j]), P(g[i + 1], g[j]), P(g[i], g[j + 1]), P(g[i + 1], g[j + 1])
                    out += [[p00, p10, p11], [p00, p11, p01]]
    return np.array(out, np.float32)


def _random_tris(n, seed, size=0.4):
    rng = np.random.default_rng(seed)
    c = rng.random((n, 1, 3)) * 2 - 1
    return (c + size * (rng.random((n, 3, 3)) - 0.5)).astype(np.float32)


def deep_tris(levels=150, per=8, r=0.55):
    """clusters of small triangles at geometrically shrinking scales around the origin: the host SAH + re-insertion tree is > 62 deep"""
    rng = np.random.default_rng(1)
    out = []
    for k in range(levels):
        s = r ** k
        for _ in range(per):
            c = (rng.random(3) * 2 - 1) * s
            e = s * 0.05
            out.append([c, c + [e, 0, 0], c + [0, e, e]])
    return np.array(out, np.float32)


def _one_centroid():
    rng = np.random.default_rng(5)
    base = np.array([[1.0, 0, 0], [-0.5, 0.8, 0.1], [-0.5, -0.8, -0.1]])
    out = []
    for _ in range(40):
        q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        out.append(base @ q.T)
    out = np.array(out, np.float32)
    return np.concatenate([out, out[:6], out[:3]])                    # exact duplicates with distinct (higher) ids


def _mirror_instances():
    box = _box_mesh((-0.5, -0.3, -0.2), (0.5, 0.3, 0.2), 2)
    X = []
    for k, (sx, sy, sz) in enumerate([(1, 1, 1), (-1, 1, 1), (2.5, 0.3, 1.7), (1, -0.5, -3)]):
        m = np.diag([sx, sy, sz, 1.0]); m[:3, 3] = (1.5 * k - 2, 0.3 * k, -0.2 * k)
        X.append((m, 0))
    X.append((np.array([[0.0, 1, 0, 0.5], [-1, 0, 0, 1], [0, 0, 1, 2], [0, 0, 0, 1]]), 0))                # rotation
    X.append((np.array([[1.0, 0.4, 0, -1], [0, 1, 0, -1], [0, 0, 1, -1], [0, 0, 0, 1]]), 1))             # shear
    return _scene([box, _random_tris(12, 9)], X)


def _plane():
    g = np.linspace(-1, 1, 9); out = []
    for i in range(8):
        for j in range(8):
            p = [[g[i], g[j], 0], [g[i + 1], g[j], 0], [g[i + 1], g[j + 1], 0], [g[i], g[j + 1], 0]]
            out += [[p[0], p[1], p[2]], [p[0], p[2], p[3]]]
    return np.array(out, np.float32)


SYNTH = {
    "tris1": lambda: _scene([_random_tris(1, 1)]), "tris2": lambda: _scene([_random_tris(2, 2)]),
    "tris4": lambda: _scene([_random_tris(4, 3)]), "tris5": lambda: _scene([_random_tris(5, 4)]),
    "tris16": lambda: _scene([_box_mesh((-1, -1, -1), (1, 1, 1), 1)[:12], _random_tris(4, 6)]),
    "tris17": lambda: _scene([_box_mesh((-1, -1, -1), (1, 1, 1), 1)[:12], _random_tris(5, 7)]),
    "tris64": lambda: _scene([_box_mesh((-1, -1, -1), (1, 1, 1), 2)[:48], _random_tris(16, 8)]),
    "plane": lambda: _scene([_plane()]),
    "one_centroid": lambda: _scene([_one_centroid()]),
    "deep": lambda: _scene([deep_tris()]),
    "offset": lambda: _scene([_box_mesh((1e5 - 1, 1e5 - 2, 1e5 - 1), (1e5 + 1, 1e5 + 1, 1e5 + 2), 3)]),
    "tiny": lambda: _scene([_box_mesh((-5e-4, -5e-4, -5e-4), (5e-4, 4e-4, 5e-4), 3)]),
    "instances": _mirror_instances,
}
ENV = {"tris64": {"B200PT_FLAT_MAX": "64"}, "cornell_box_glass": {"B200PT_SMEM_BIG": "1"}}


def scene_dict(name):
    return SYNTH[name]() if name in SYNTH else util.scene_dict(name)


def world_tris(sc):
    """(v0, e1, e2) [n, 3] float32 as the GPU stores them (k_world_tris), gid order = instances x primitives"""
    v0s, e1s, e2s = [], [], []
    for xf, m, _ in sc["instances"]:
        M = np.asarray(xf, np.float32).reshape(4, 4).T                                       # column-major -> row-major o2w
        v, idx = sc["meshes"][m]
        P = v["pos"][np.asarray(idx, np.int64)].reshape(-1, 3, 3).astype(np.float32)
        W = ((M[:, 0] * P[..., 0:1] + M[:, 1] * P[..., 1:2]) + M[:, 2] * P[..., 2:3]) + M[:, 3] * np.float32(1.0)   # fp32, no FMA
        W = W[..., :3].astype(np.float32)
        v0s.append(W[:, 0]); e1s.append(W[:, 1] - W[:, 0]); e2s.append(W[:, 2] - W[:, 0])
    return np.concatenate(v0s), np.concatenate(e1s), np.concatenate(e2s)


class Ref:
    """float64 brute force with magnitude-derived margins (module docstring)"""

    def __init__(self, sc):
        self.v0, self.e1, self.e2 = [a.astype(np.float64) for a in world_tris(sc)]
        n = len(self.v0)
        rec = np.concatenate([a.view(np.uint32) for a in world_tris(sc)], 1)
        _, inv = np.unique(rec, axis=0, return_inverse=True)
        inv = inv.reshape(-1)
        self.dup_min = np.full(inv.max() + 1, n, np.int64); np.minimum.at(self.dup_min, inv, np.arange(n))
        self.dup_of = inv                                                                     # duplicate class of each gid
        self.inst_base = np.cumsum([0] + [len(sc["meshes"][m][1]) // 3 for _, m, _ in sc["instances"]])
        self.lo = np.minimum(self.v0, np.minimum(self.v0 + self.e1, self.v0 + self.e2))
        self.hi = np.maximum(self.v0, np.maximum(self.v0 + self.e1, self.v0 + self.e2))
        self.extent = float(np.abs(np.concatenate([self.lo, self.hi])).max())
        G = 64                                                                                # groups of consecutive triangles for the box prefilter
        self.groups = [np.arange(i, min(i + G, n)) for i in range(0, n, G)]
        self.glo = np.array([self.lo[g].min(0) for g in self.groups]); self.ghi = np.array([self.hi[g].max(0) for g in self.groups])

    def gid(self, prim, inst):
        return np.where(prim == 0xFFFFFFFF, -1, self.inst_base[np.minimum(inst, len(self.inst_base) - 1)] + prim.astype(np.int64))

    def classify(self, o, d, tmin, tmax, k=EPS_K):
        """per ray: (gids, t, eps_t, required, admissible, u, v, eps_u, eps_v) over candidate triangles"""
        o = o.astype(np.float64); d = d.astype(np.float64)
        out = []
        for r in range(len(o)):
            cand = self._candidates(o[r], d[r])
            v0, e1, e2 = self.v0[cand], self.e1[cand], self.e2[cand]
            p = np.cross(d[r], e2); det = (e1 * p).sum(1)
            tv = o[r] - v0; q = np.cross(tv, e1)
            with np.errstate(divide="ignore", invalid="ignore"):
                u = (tv * p).sum(1) / det; v = (d[r] * q).sum(1) / det; t = (e2 * q).sum(1) / det
                n = lambda a: np.linalg.norm(a, axis=-1)
                ad = np.abs(det); P = n(d[r]) * n(e2); Q = n(tv) * n(e1); ne1p = n(e1) * P
                eu = k * U * (n(tv) * P + np.abs(u) * ne1p) / ad
                ev = k * U * (n(d[r]) * Q + np.abs(v) * ne1p) / ad
                et = k * U * (n(e2) * Q + np.abs(t) * ne1p) / ad + k * U * abs(float(tmin[r]))
                ok = np.isfinite(u) & np.isfinite(v) & np.isfinite(t) & (ad > 0)
                req = ok & (u >= eu) & (v >= ev) & (u + v <= 1 - eu - ev) & (t > tmin[r] + et) & (t < tmax[r] - et)
                adm = ok & (u >= -eu) & (v >= -ev) & (u + v <= 1 + eu + ev) & (t > tmin[r] - et) & (t < tmax[r] + et)
            out.append((cand, np.where(ok, t, np.inf), np.where(ok, et, 0.0), req, adm, u, v, eu, ev))
        return out

    def _candidates(self, o, d):
        if len(self.groups) <= 16: return np.arange(len(self.v0))
        with np.errstate(divide="ignore", invalid="ignore"):
            inv = 1.0 / np.where(np.abs(d) < 1e-300, 1e-300, d)
            pad = 1e-6 * self.extent
            t0 = (self.glo - pad - o) * inv; t1 = (self.ghi + pad - o) * inv
            tn = np.nanmax(np.minimum(t0, t1), 1); tf = np.nanmin(np.maximum(t0, t1), 1)
        hit = np.nonzero(tn <= tf * (1 + 1e-9) + 1e-12)[0]
        return np.concatenate([self.groups[g] for g in hit]) if len(hit) else np.zeros(0, np.int64)


# ---------------------------------------------------------------- checks
def _close(a_gpu, a_ref, eps):
    return abs(float(a_gpu) - a_ref) <= eps + VALUE_ULPS * float(np.spacing(np.float32(abs(a_ref))))


def check_closest(ref, cls, gid, t_gpu, uv_gpu):
    """returns (indices of the rays whose answer fails, number of rays the margins leave ambiguous)"""
    bad, amb = [], 0
    for r, (cand, t, et, req, adm, u, v, eu, ev) in enumerate(cls):
        g = gid[r]
        best_req = t[req].min() if req.any() else np.inf
        if (adm & ~req & (t <= best_req + et)).any(): amb += 1
        if g < 0:
            if req.any(): bad.append(r)
            continue
        j = np.nonzero(cand == g)[0]
        if len(j) == 0 or not adm[j[0]]: bad.append(r); continue
        if ref.dup_min[ref.dup_of[g]] != g: bad.append(r); continue          # lowest id among bit-identical duplicates
        j = j[0]
        if req.any() and (t[req] + et[req] < t[j] - et[j]).any(): bad.append(r); continue
        if req[j] and not (_close(t_gpu[r], t[j], et[j]) and _close(uv_gpu[r, 0], u[j], eu[j]) and _close(uv_gpu[r, 1], v[j], ev[j])):
            print(f"ray {r}: t {t_gpu[r]!r} / {t[j]!r} +- {et[j]:.3g}, u {uv_gpu[r, 0]!r} / {u[j]!r} +- {eu[j]:.3g}, v {uv_gpu[r, 1]!r} / {v[j]!r} +- {ev[j]:.3g}")
            bad.append(r)                                                          # t, u, v of a required hit
    return bad, amb


def check_any(cls, occ):
    bad, amb = [], 0
    for r, (cand, t, et, req, adm, *_) in enumerate(cls):
        if adm.any() and not req.any(): amb += 1
        if occ[r] and not adm.any(): bad.append(r)
        if not occ[r] and req.any(): bad.append(r)
    return bad, amb


# ---------------------------------------------------------------- rays
def rays_random(ref, n, rng):
    lo, hi = ref.lo.min(0), ref.hi.max(0); ext = hi - lo + 1e-3 * max(ref.extent, 1e-30)
    o = lo - 0.2 * ext + 1.4 * ext * rng.random((n, 3))
    d = rng.normal(size=(n, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    return o.astype(np.float32), d.astype(np.float32)


def _surface_points(ref, n, rng, edge=False):
    g = rng.integers(0, len(ref.v0), n)
    if edge:                                                                   # on an edge, or exactly a vertex
        s = rng.random(n); s[rng.random(n) < 0.25] = 0.0
        k = rng.integers(0, 3, n)
        b = np.stack([np.where(k == 0, s, np.where(k == 1, 1 - s, 0.0)), np.where(k == 0, 1 - s, np.where(k == 2, s, 0.0))], 1)
    else:
        b = rng.random((n, 2)); f = b.sum(1) > 1; b[f] = 1 - b[f]
    p = ref.v0[g] + b[:, :1] * ref.e1[g] + b[:, 1:] * ref.e2[g]
    return p, g


def rays_edges(ref, n, rng):
    p, _ = _surface_points(ref, n, rng, edge=True)
    d = rng.normal(size=(n, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    o = p - d * (0.5 + rng.random((n, 1))) * max(ref.extent, 1e-30)
    return o.astype(np.float32), d.astype(np.float32)


def rays_axis(ref, n, rng):
    """directions with exact 0 and +-1e-31 components; aimed at triangle points, and from random origins inside / around the boxes"""
    p, _ = _surface_points(ref, n, rng)
    ax = rng.integers(0, 3, n)
    d = np.zeros((n, 3)); d[np.arange(n), ax] = np.where(rng.random(n) < 0.5, -1.0, 1.0)
    tiny = rng.random((n, 3)) < 0.4
    d = np.where((d == 0) & tiny, np.where(rng.random((n, 3)) < 0.5, -1e-31, 1e-31), d)
    o = p - d * max(ref.extent, 1e-30) * (0.2 + rng.random((n, 1)))
    o2, _ = rays_random(ref, n, rng)
    half = rng.random(n) < 0.5
    o = np.where(half[:, None], o, o2)
    return o.astype(np.float32), d.astype(np.float32)


def rays_from_surface(ref, n, rng, far=0.0):
    p, _ = _surface_points(ref, n, rng)
    if far:
        u = rng.normal(size=(n, 3)); u /= np.linalg.norm(u, axis=1, keepdims=True)
        p = p + u * far * ref.extent * rng.random((n, 1))
    q, _ = _surface_points(ref, n, rng)
    d = q - p; d /= np.maximum(np.linalg.norm(d, axis=1, keepdims=True), 1e-300)
    m = rng.random(n) < 0.3                                                   # and some random directions
    r = rng.normal(size=(n, 3)); r /= np.linalg.norm(r, axis=1, keepdims=True)
    d = np.where(m[:, None], r, d)
    return p.astype(np.float32), d.astype(np.float32)


def ray_sets(ref, seed, n=600):
    rng = np.random.default_rng(seed)
    return {"random": rays_random(ref, 4 * n, rng), "edges": rays_edges(ref, n, rng), "axis": rays_axis(ref, n, rng),
            "surface": rays_from_surface(ref, n, rng), "surface_nee": rays_from_surface(ref, n, rng), "far16": rays_from_surface(ref, n, rng, far=16.0)}


# ---------------------------------------------------------------- the GPU side
@pytest.fixture(scope="module")
def pt():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import vpt_b200
    return vpt_b200


def tracer(pt, name, monkeypatch, extra_env=None):
    for k in ("B200PT_FLAT_MAX", "B200PT_SMEM_BIG", "B200PT_BVH_SAH", "B200PT_WIDE_STACK", "B200PT_TRAV", "B200PT_WIDE"): monkeypatch.delenv(k, raising=False)
    for k, v in {**ENV.get(name, {}), **(extra_env or {})}.items(): monkeypatch.setenv(k, v)
    sc = scene_dict(name)
    T = pt.PathTracer(0)
    T.set_scene(sc)
    return T, sc


# tmin: extension rays leave a surface at 0.01, shadow rays at 1e-4 (k_extend / k_connect / k_shade_hit)
TMIN = {"random": 1e-4, "edges": 1e-4, "axis": 1e-4, "surface": 0.01, "surface_nee": 1e-4, "far16": 1e-4}


def query(T, shape, kind, o, d, tmin, tmax, **kw):
    """the query through the counting instantiations (returned) and through the renderer's own ones: the answers must be identical"""
    r = T.trace_query(shape, kind, o, d, tmin, tmax, **kw)
    p = T.trace_query(shape, kind, o, d, tmin, tmax, stats=False, **kw)
    keys = ("t", "prim", "inst", "uv") if kind == "closest" else ("occluded",)
    assert all(np.array_equal(np.asarray(r[k]).view(np.uint8), np.asarray(p[k]).view(np.uint8)) for k in keys), (shape, kind, kw)
    return r


def run_case(T, ref, name, shapes, sets, kinds=("closest", "any", "target"), max_ambiguous=1e-3):
    """every shape x kind x ray set: 100 % of the answers pass, zero refused pushes, and at most max_ambiguous of the random rays are
    left undecided by the margins"""
    failures = []
    for set_name, (o, d) in sets.items():
        tmin = np.full(len(o), TMIN[set_name], np.float32)
        tmax = np.full(len(o), 1e6, np.float32)
        cls = ref.classify(o, d, tmin, tmax)
        closest0 = None
        for shape in shapes:
            for fma in ((False, True) if shape not in ("flat", "fixed_origin") else (False,)):
                if shape == "fixed_origin" or (set_name == "far16" and not fma):
                    continue
                r = query(T, shape, "closest", o, d, tmin, tmax, fma=fma)
                gid = ref.gid(r["prim"], r["inst"])
                bad, amb = check_closest(ref, cls, gid, r["t"], r["uv"])
                refused = int(r["stats"][:, 2].sum())
                print(f"{name:18s} {set_name:8s} {shape:11s} fma={int(fma)} closest  ambiguous {amb / len(o):.4%}  failed {len(bad)}  refused {refused}")
                if set_name == "random": assert amb / len(o) < max_ambiguous, (name, amb)
                if bad or refused: failures.append((set_name, shape, fma, "closest", bad[:5], refused))
                cur = (r["t"].view(np.uint32), r["prim"], r["inst"], r["uv"].view(np.uint32))
                if closest0 is None: closest0 = (shape, fma, cur)
                elif not all(np.array_equal(a, b) for a, b in zip(cur, closest0[2])):   # the shapes are interchangeable bit for bit
                    failures.append((set_name, shape, fma, "closest differs from " + str(closest0[:2]), None, 0))
                # tmax at, and one ulp on either side of, each hit distance: t < tmax is strict and decided by the same fp32 t
                hit = r["t"] > 0
                if hit.any() and shape in ("shared", "global", "dyn2", "dyn4", "flat"):
                    th = r["t"][hit]
                    at = query(T, shape, "closest", o[hit], d[hit], tmin[hit], th, fma=fma)
                    above = query(T, shape, "closest", o[hit], d[hit], tmin[hit], np.nextafter(th, np.float32(np.inf)), fma=fma)
                    below = query(T, shape, "closest", o[hit], d[hit], tmin[hit], np.nextafter(th, np.float32(0)), fma=fma)
                    if not (np.all(at["t"] < th) and np.array_equal(above["t"], th) and np.array_equal(above["prim"], r["prim"][hit])
                            and np.all(below["t"] < np.nextafter(th, np.float32(0)))):
                        failures.append((set_name, shape, fma, "tmax ulp", None, 0))
                if "target" in kinds and hit.any():
                    failures += check_target(T, ref, shape, o[hit], d[hit], tmin[hit], r["t"][hit], gid[hit], fma, name, set_name)
            if "any" in kinds and shape != "fixed_origin":
                for fma in ((False, True) if shape != "flat" else (False,)):
                    if set_name == "far16" and not fma: continue
                    r = query(T, shape, "any", o, d, tmin, tmax, fma=fma)
                    bad, amb = check_any(cls, r["occluded"])
                    refused = int(r["stats"][:, 2].sum())
                    print(f"{name:18s} {set_name:8s} {shape:11s} fma={int(fma)} any      ambiguous {amb / len(o):.4%}  failed {len(bad)}  refused {refused}")
                    if bad or refused: failures.append((set_name, shape, fma, "any", bad[:5], refused))
        if "fixed_origin" in shapes:                                            # one origin, many directions: k_camera's table
            oo = np.repeat(o[:1], len(o), 0)
            c2 = ref.classify(oo, d, tmin, tmax)
            r = query(T, "fixed_origin", "closest", oo, d, tmin, tmax)
            bad, amb = check_closest(ref, c2, ref.gid(r["prim"], r["inst"]), r["t"], r["uv"])
            r2 = T.trace_query("flat", "closest", oo, d, tmin, tmax)
            print(f"{name:18s} {set_name:8s} fixed_origin      closest  ambiguous {amb / len(o):.4%}  failed {len(bad)}")
            if bad or not np.array_equal(r["t"].view(np.uint32), r2["t"].view(np.uint32)) or not np.array_equal(r["prim"], r2["prim"]):
                failures.append((set_name, "fixed_origin", False, "closest", bad[:5], 0))
    assert not failures, failures


def check_target(T, ref, shape, o, d, tmin, t_hit, g_hit, fma, name, set_name):
    """light visibility towards the triangle the closest-hit query found, at tmax = its fp32 t (the renderer's tL): the target and its
    higher-id duplicates never occlude, a lower-id duplicate at the same t always does (exact); everything else by the margins.  Also the
    fused kernel's sky form of the same query (target 0xFFFFFFFF, tmax_test = tmax): only triangles strictly before tmax occlude."""
    fails = []
    n = len(o)
    dup = ref.dup_of[g_hit]
    members = [np.nonzero(ref.dup_of == c)[0] for c in dup]
    # target = the hit itself (the lowest duplicate) or its highest duplicate
    hi_dup = np.array([m.max() for m in members]); lo_dup = np.array([m.min() for m in members])
    tmax_next = np.nextafter(t_hit, np.float32(np.inf))
    cls = ref.classify(o, d, tmin, t_hit)
    sky = np.full(n, 0xFFFFFFFF, np.int64)
    for label, target, forms in (("lowest", lo_dup, ("default", "nextafter")), ("highest", hi_dup, ("default", "nextafter")), ("sky", sky, ("tmax",))):
        for tt_label in forms:
            tt = {"default": np.full(n, -1.0, np.float32), "nextafter": tmax_next, "tmax": t_hit}[tt_label]
            r = query(T, shape, "target", o, d, tmin, t_hit, target=target.astype(np.uint32), tmax_test=tt, fma=fma)
            occ = r["occluded"]
            bad = []
            for k in range(n):
                cand, t, et, req, adm = cls[k][:5]
                if label == "sky":                                              # nothing at t == tmax passes tmax_test = tmax
                    req_occ, adm_occ = req.any(), adm.any()
                else:
                    same = ref.dup_of[cand] == dup[k]
                    lower_dup = (same & (cand < target[k])).any()
                    req_occ = (req & ~same).any() or lower_dup
                    adm_occ = (adm & ~same).any() or lower_dup
                if occ[k] and not adm_occ: bad.append(k)
                if not occ[k] and req_occ: bad.append(k)
            refused = int(r["stats"][:, 2].sum())
            print(f"{name:18s} {set_name:8s} {shape:11s} fma={int(fma)} target({label},{tt_label})  failed {len(bad)}  refused {refused}")
            if bad or refused: fails.append((set_name, shape, fma, f"target {label} {tt_label}", bad[:5], refused))
    return fails


SCENES = ["tris1", "tris2", "tris4", "tris5", "tris16", "tris17", "tris64", "plane", "one_centroid", "deep", "offset", "tiny", "instances",
          "cornell_box", "cornell_box_glass"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", SCENES)
def test_every_shape_and_kind_matches_float64_reference(pt, name, monkeypatch):
    T, sc = tracer(pt, name, monkeypatch)
    ref = Ref(sc)
    sets = ray_sets(ref, 11)
    o, d = sets["random"]
    shapes = [s for s in SHAPES if _has(T, s, o, d)]
    assert {"shared", "global", "dyn2"} <= set(shapes) or name == "cornell_box_glass", shapes
    if name in ("tris1", "tris2", "tris4", "tris5", "tris16", "tris64", "cornell_box"): assert {"flat", "fixed_origin"} <= set(shapes)
    if name == "deep": assert {"dyn4", "dyn4_spill"} <= set(shapes), shapes           # its BVH is big enough for the BVH4 (> 64 KiB)
    run_case(T, ref, name, shapes, sets)


def _has(T, shape, o, d):
    import vpt_b200
    try:
        T.trace_query(shape, "closest", o[:1], d[:1], 0.01, 1e5)
        return True
    except vpt_b200.B200ptError:
        return False


@pytest.mark.gpu
@pytest.mark.parametrize("wide_stack", [None, "4"])
def test_breakfast_room_bvh4(pt, wide_stack, monkeypatch):
    T, sc = tracer(pt, "breakfast_room", monkeypatch, {"B200PT_WIDE_STACK": wide_stack} if wide_stack else None)
    ref = Ref(sc)
    rng = np.random.default_rng(3)
    sets = {"random": rays_random(ref, 600, rng), "edges": rays_edges(ref, 200, rng), "axis": rays_axis(ref, 200, rng),
            "surface": rays_from_surface(ref, 200, rng), "surface_nee": rays_from_surface(ref, 200, rng), "far16": rays_from_surface(ref, 150, rng, far=16.0)}
    # the chair legs are slivers (aspect ratio 240 at p90): their margins are wide, 2 of 600 random rays pass within them (H100, K = 8)
    run_case(T, ref, "breakfast_room", ["global", "dyn2", "dyn4", "dyn4_spill"], sets, max_ambiguous=5e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("sah", ["0", "1", "2", "3", "4", "5"])
@pytest.mark.parametrize("name", ["one_centroid", "deep", "instances"])
def test_tree_builders(pt, name, sah, monkeypatch):
    T, sc = tracer(pt, name, monkeypatch, {"B200PT_BVH_SAH": sah})
    ref = Ref(sc)
    rng = np.random.default_rng(int(sah) + 20)
    sets = {"random": rays_random(ref, 1500, rng), "edges": rays_edges(ref, 400, rng), "surface_nee": rays_from_surface(ref, 300, rng)}
    run_case(T, ref, f"{name}/sah{sah}", [s for s in ("shared", "global", "dyn2", "dyn4", "dyn4_spill") if _has(T, s, *sets["random"])], sets,
             kinds=("closest", "any"))


@pytest.mark.gpu
def test_margin_is_tight(pt, monkeypatch):
    """EPS_K / 10 rejects some GPU answer on edge / vertex rays; EPS_K accepts all of them"""
    worst = 0
    for name in ("plane", "offset", "instances", "one_centroid"):
        T, sc = tracer(pt, name, monkeypatch)
        ref = Ref(sc)
        o, d = rays_edges(ref, 3000, np.random.default_rng(7))
        tmin = np.full(len(o), 1e-4, np.float32); tmax = np.full(len(o), 1e6, np.float32)
        r = query(T, "global", "closest", o, d, tmin, tmax)
        gid = ref.gid(r["prim"], r["inst"])
        assert not check_closest(ref, ref.classify(o, d, tmin, tmax), gid, r["t"], r["uv"])[0]
        fails = len(check_closest(ref, ref.classify(o, d, tmin, tmax, k=EPS_K / 10), gid, r["t"], r["uv"])[0])
        print(f"{name}: {fails} of {len(o)} edge rays fail at EPS_K / 10")
        worst = max(worst, fails)
    assert worst > 0


def test_deep_scene_premise():
    """the host builders (full binned SAH + the default re-insertion pass) make the deep fixture's tree deeper than the 62 levels a
    64-entry traversal stack serves; lbvh_refine_sah must keep the shallower tree there (the GPU tests check zero refused pushes)"""
    from vpt_b200 import binding as B
    tri = deep_tris()
    rb = np.concatenate([tri.min(1), tri.max(1)], 1).astype(np.float32)
    nodes, perm, depth, cost = B.bvh2_sah_build(rb, 1.0)
    _, d2, _ = B.bvh2_reinsert(nodes, 0, 2, 0.1)
    assert max(depth, d2) > 62, (depth, d2)
