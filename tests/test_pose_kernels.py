"""The pose kernels (k_pose_vertices, k_pose_normals) vertex by vertex against the float64 model of test_gltf_animation, at the sizes where
they can go wrong: multi-block meshes, 512- and 513-joint palettes, 16 influences and 256 morph targets.

Two generated files differ only in the size of one skin: 512 joints ("shared": the 24 KiB palette is staged in shared memory) and 513
("global": launch_pose reads every palette of the launch, small skins included, from global memory).  Both hold the same deformable meshes,
in this order (product mesh index):
  2-4   one glTF mesh of three primitives (42, 300 and 90 vertices), skinned and morphed; the 300-vertex one has no NORMAL
  5     577 vertices without NORMAL, faces in reverse order (a vertex's last face reaches into the previous block), one vertex no face uses
  6-11  3, 255, 256, 257, 1,000 and 20,000 vertices: 1, 3 (12 influences), 4 (16 influences), 0, 2 and 1 influence sets; the 257-vertex
        mesh has 256 morph targets, each with its own subset of POSITION / NORMAL / TEXCOORD_0, the 1,000-vertex one 24 and a skin; the
        20,000-vertex one is skinned to the big skin and reaches joint 511.  The 255-vertex mesh is instanced twice under the same skin.
Joints are u8 and u16, weights float (zeros, -0.0), normalized u16 and normalized u8; influence weights do not sum to 1 (nothing
renormalises), morph weights are negative, zero and above 1.

Bound: a float sum of n terms is within (n - 1) 2^-24 of the sum of their absolute values (recursive summation).  The longest chain here is
a rest position plus 256 morph terms (a skinned vertex: 16 influences x 12 palette entries, each the end of a product chain), so positions,
normals and UVs must be within K = 256 x 2^-24 of the model's sum of absolute terms, in the forms test_gltf_animation uses (generated
normals: the terms of the face's cross product).  Vertex 256 of the 256-target mesh is built so that every morph term loses almost half an ulp: K / 10 rejects it (test_margin_is_tight).
"""
import copy

import numpy as np
import pytest

import test_gltf_animation as ga
import test_instance_updates as ti
from test_gltf_animation import EPS, Gltf, _acc, _model_vertices, _rows, model_pose, quat, trs, write

K = 256
F32, U8, U16, U32 = 5126, 5121, 5123, 5125
CHAINS, LINKS = 27, 19                                  # the big skin: 27 chains of 19 joints, the last one cut to 18 for 512 joints
SMALL = 16                                              # the small skin: a binary tree of 16 joints
OVERFLOW_JOINT = LINKS - 1                              # leaf of chain 0; only the last block of the last mesh weights it
BIG_WEIGHT_TARGET = 5                                   # of the 1,000-vertex mesh; its POSITION deltas reach 2
A_SKIN, A_LONG, A_JOINT_OVERFLOW, A_WEIGHT_OVERFLOW = 0, 1, 2, 3
TIMES = {-1: [0.0], A_SKIN: [-0.5, 0.0, 0.4, 1.0, 1.55, 2.0, 3.0], A_LONG: [-1.0, 0.0, 3.33, 4.5, 9.99, 12.0]}
LONG_KEYS = 1000


# ---------------------------------------------------------------- geometry and influences
def grid(nx, ny, origin, du, dv, rng):
    """nx x ny vertices (row-major), two triangles per cell, normals near du x dv, uvs in [0, 1]"""
    o, du, dv = (np.asarray(x, np.float64) for x in (origin, du, dv))
    jj, ii = np.meshgrid(np.arange(nx), np.arange(ny))
    P = o + jj.reshape(-1, 1) * du + ii.reshape(-1, 1) * dv + rng.normal(0, 0.01, (nx * ny, 3))
    n = np.cross(du, dv); n /= np.linalg.norm(n)
    N = n + rng.normal(0, 0.1, (nx * ny, 3))
    U = np.stack([jj.reshape(-1) / max(nx - 1, 1), ii.reshape(-1) / max(ny - 1, 1)], 1)
    I = []
    for i in range(ny - 1):
        for j in range(nx - 1):
            a, b, c, d = i * nx + j, i * nx + j + 1, (i + 1) * nx + j, (i + 1) * nx + j + 1
            I += [a, b, c, b, d, c]
    return P.astype(np.float32), N.astype(np.float32), U.astype(np.float32), np.array(I, np.uint32)


def encode_set(G, J, W, jtype, wtype):
    """one JOINTS_n / WEIGHTS_n pair -> (accessors, joints and weights as the loader decodes them)"""
    if wtype == "f32":
        w = W.astype(np.float32); wa = G.acc(w, F32, "VEC4", 1); wd = w.astype(np.float64)
    else:
        top = 255 if wtype == "u8" else 65535
        w = np.round(np.clip(W, 0, 1) * top).astype(np.uint8 if wtype == "u8" else np.uint16)
        wa = G.acc(w, U8 if wtype == "u8" else U16, "VEC4", 1, normalized=True); wd = w.astype(np.float64) / top
    j = J.astype(np.uint8 if jtype == "u8" else np.uint16)
    return G.acc(j, U8 if jtype == "u8" else U16, "VEC4", 1), wa, j.astype(np.int64), wd


def influences(G, rng, n, types, n_joints):
    """random influences over len(types) sets: ~20% zero weights, -0.0 in float sets, sums spread around 1, the first weight at least 0.1"""
    attr, Js, Ws = {}, [], []
    for s, (jt, wt) in enumerate(types):
        J = rng.integers(0, n_joints, (n, 4))
        W = rng.random((n, 4)) * 2 / (4 * len(types)); W[rng.random((n, 4)) < 0.2] = 0.0
        if wt == "f32": W[rng.random((n, 4)) < 0.05] = -0.0
        if s == 0: W[:, 0] = np.maximum(W[:, 0], 0.1)                # no vertex without weight: a zero skin matrix has no normal
        ja, wa, jd, wd = encode_set(G, J, W, jt, wt)
        attr[f"JOINTS_{s}"] = ja; attr[f"WEIGHTS_{s}"] = wa; Js.append(jd); Ws.append(wd)
    return attr, dict(joints=np.concatenate(Js, 1), weights=np.concatenate(Ws, 1))


def morph(G, rng, n, n_targets, scale=0.02, subsets=lambda t: t % 7 + 1, fix=None):
    """n_targets targets; target t carries the attributes of bit set subsets(t) (1 POSITION, 2 NORMAL, 4 TEXCOORD_0); fix(t, key, deltas)
    may edit a target's deltas before they are written"""
    targets, M = [], dict(dpos=[], dnrm=[], duv=[])
    for t in range(n_targets):
        tg = {}
        for bit, key, nc, name in ((1, "POSITION", 3, "dpos"), (2, "NORMAL", 3, "dnrm"), (4, "TEXCOORD_0", 2, "duv")):
            if subsets(t) & bit:
                d = rng.normal(0, scale, (n, nc)).astype(np.float32)
                if fix: fix(t, key, d)
                tg[key] = G.acc(d, F32, f"VEC{nc}", 1); M[name].append(d)
            else:
                M[name].append(None)
        targets.append(tg)
    return targets, M


def morph_weights(rng, n):
    """negative, zero, -0.0 and above-1 weights"""
    w = rng.uniform(-1.5, 2.5, n); w[rng.random(n) < 0.15] = 0.0; w[rng.random(n) < 0.05] = -0.0
    return [float(np.float32(x)) for x in w]


# ---------------------------------------------------------------- the file
def rest_worlds(nodes):
    parent = {c: i for i, n in enumerate(nodes) for c in n.get("children", [])}
    memo = {}
    def w(i):
        if i not in memo:
            n = nodes[i]; loc = trs(n.get("translation", [0, 0, 0]), n.get("rotation", [0, 0, 0, 1]), n.get("scale", [1, 1, 1]))
            memo[i] = (w(parent[i]) if i in parent else np.eye(4)) @ loc
        return memo[i]
    return w


def build_scene(big_joints):
    """(gltf dict, [geometry bin, animation bin], model) of the module docstring's file with a big skin of `big_joints` (512 or 513)"""
    G = Gltf(); rng = np.random.default_rng(2026)
    meshes, model = [], {}

    def prim(P, N, U, I, material, attr=None, targets=None):
        a = {"POSITION": G.acc(P, F32, "VEC3")}
        if N is not None: a["NORMAL"] = G.acc(N, F32, "VEC3")
        a["TEXCOORD_0"] = G.acc(U, F32, "VEC2")
        a.update(attr or {})
        p = {"attributes": a, "indices": G.acc(I, U32, "SCALAR"), "material": material}
        if targets: p["targets"] = targets
        return p

    materials = [{"pbrMetallicRoughness": {"baseColorFactor": [0.8, 0.8, 0.8, 1], "metallicFactor": 0.0, "roughnessFactor": 0.7}},
                 {"emissiveFactor": [1, 1, 1], "extensions": {"KHR_materials_emissive_strength": {"emissiveStrength": 6.0}},
                  "pbrMetallicRoughness": {"metallicFactor": 0.0}},
                 {"pbrMetallicRoughness": {"baseColorFactor": [0.8, 0.2, 0.1, 1], "metallicFactor": 0.0, "roughnessFactor": 0.4}}]
    meshes.append({"name": "room", "primitives": [prim(*ga.box((0, 0, -1), (6, 4, 7), inward=True), 0)]})           # 0
    meshes.append({"name": "light", "primitives": [prim(*ga.box((0, 0, 0), (1.2, 0.05, 0.8)), 1)]})                 # 1

    # 2: three primitives, skinned (small skin) and morphed with 3 shared weights; the middle one has no NORMAL
    prims = []
    for k, (nx, ny, normals) in enumerate(((7, 6, True), (20, 15, False), (9, 10, True))):
        P, N, U, I = grid(nx, ny, (-3.5 + 1.2 * k, -1.8, -3.0), (0.05, 0, 0), (0, 0.08, 0.01), rng)
        attr, M = influences(G, rng, len(P), [("u8", "f32"), ("u16", "u8")] if k == 1 else [("u8", "f32")], SMALL)
        tg, D = morph(G, rng, len(P), 3, 0.05, lambda t: (1, 3, 5)[t] if normals else (1, 5, 4)[t])
        prims.append(prim(P, N if normals else None, U, I, 2, attr, tg)); model[(2, k)] = {**M, **D}
    meshes.append({"name": "multi", "primitives": prims, "weights": [0.3, -0.2, 0.7]})
    # 3: 577 vertices without NORMAL, faces in reverse order, vertex 576 used by no face
    P, _, U, I = grid(24, 24, (0.5, -1.8, -3.2), (0.06, 0, 0), (0, 0.06, 0.02), rng)
    P = np.concatenate([P, [[1.0, -1.0, -3.0]]]).astype(np.float32); U = np.concatenate([U, [[0.5, 0.5]]]).astype(np.float32)
    I = I.reshape(-1, 3)[::-1].reshape(-1).copy()
    attr, M = influences(G, rng, len(P), [("u16", "u16")], SMALL)
    meshes.append({"name": "reversed", "primitives": [prim(P, None, U, I, 0, attr)]}); model[(3, 0)] = {**M, "dpos": [], "dnrm": [], "duv": []}
    # 4: one triangle
    P, N, U = (np.array(x, np.float32) for x in ([[-1, 0.5, -2.5], [-0.5, 0.5, -2.5], [-0.8, 1.0, -2.6]], [[0, 0, 1]] * 3, [[0, 0], [1, 0], [0, 1]]))
    attr, M = influences(G, rng, 3, [("u8", "u8")], SMALL)
    meshes.append({"name": "tri", "primitives": [prim(P, N, U, np.array([0, 1, 2], np.uint32), 2, attr)]}); model[(4, 0)] = {**M, "dpos": [], "dnrm": [], "duv": []}
    # 5: 255 vertices, 3 sets (12 influences), instanced twice
    P, N, U, I = grid(15, 17, (-2.0, 0.2, -3.4), (0.07, 0, 0), (0, 0.06, 0.01), rng)
    attr, M = influences(G, rng, len(P), [("u8", "f32"), ("u16", "u8"), ("u8", "u16")], SMALL)
    meshes.append({"name": "g255", "primitives": [prim(P, N, U, I, 0, attr)]}); model[(5, 0)] = {**M, "dpos": [], "dnrm": [], "duv": []}
    # 6: 256 vertices, 4 sets (16 influences)
    P, N, U, I = grid(16, 16, (-0.8, 0.2, -3.4), (0.07, 0, 0), (0, 0.06, -0.01), rng)
    attr, M = influences(G, rng, len(P), [("u16", "u16"), ("u8", "f32"), ("u16", "u8"), ("u8", "f32")], SMALL)
    meshes.append({"name": "g256", "primitives": [prim(P, N, U, I, 2, attr)]}); model[(6, 0)] = {**M, "dpos": [], "dnrm": [], "duv": []}
    # 7: 257 vertices, 256 morph targets, not skinned; vertex 256 (one extra triangle) loses almost half an ulp at every POSITION term
    P, N, U, I = grid(16, 16, (0.6, 0.2, -3.0), (0.07, 0, 0), (0, 0.06, 0.0), rng)
    P = np.concatenate([P, [[1.0, 1.5, -3.0]]]).astype(np.float32); N = np.concatenate([N, [[0, 0, 1]]]).astype(np.float32)
    U = np.concatenate([U, [[0.25, 0.75]]]).astype(np.float32); I = np.concatenate([I, [0, 1, 256]]).astype(np.uint32)
    w257 = morph_weights(rng, 256)

    def lose_half_ulps(t, key, d):
        if key == "POSITION":
            d[256] = 0.0
            if w257[t] != 0.0: d[256, 0] = np.float32(0.45 * 2.0 ** -23 / w257[t])    # w d = +0.45 ulp(1): the float sum stays 1
    tg, D = morph(G, rng, len(P), 256, 0.01, fix=lose_half_ulps)
    meshes.append({"name": "g257", "primitives": [prim(P, N, U, I, 0, None, tg)], "weights": w257}); model[(7, 0)] = D
    # 8: 1,000 vertices, 24 targets, 2 sets; target BIG_WEIGHT_TARGET moves a few vertices by 2
    P, N, U, I = grid(25, 40, (2.0, -1.8, -3.3), (0.06, 0, 0), (0, 0.09, 0.0), rng)
    attr, M = influences(G, rng, len(P), [("u8", "u16"), ("u16", "f32")], SMALL)
    def far(t, key, d):
        if t == BIG_WEIGHT_TARGET and key == "POSITION": d[::97] = 2.0
    tg, D = morph(G, rng, len(P), 24, 0.03, lambda t: 1 | (2 if t % 2 else 0) | (4 if t % 3 == 0 else 0), far)
    w1000 = morph_weights(rng, 24); w1000[BIG_WEIGHT_TARGET] = 0.1
    meshes.append({"name": "g1000", "primitives": [prim(P, N, U, I, 2, attr, tg)], "weights": w1000}); model[(8, 0)] = {**M, **D}
    # 9: 20,000 vertices on the big skin, 1 set: joint (chain by column, link by row), its neighbours along and across the chain
    nx, ny = 100, 200
    P, N, U, I = grid(nx, ny, (-4.0, -2.0, -3.8), (8.0 / (nx - 1), 0, 0), (0, 3.6 / (ny - 1), 0.0), rng)
    jj, ii = np.meshgrid(np.arange(nx), np.arange(ny)); jj, ii = jj.reshape(-1), ii.reshape(-1)
    c = np.minimum(jj * CHAINS // nx, CHAINS - 1); k = np.minimum(ii * LINKS // ny, LINKS - 1)
    J0 = np.minimum(c * LINKS + k, 511)
    J = np.stack([J0, np.minimum(c * LINKS + np.maximum(k - 1, 0), 511), np.minimum(np.minimum(c + 1, CHAINS - 1) * LINKS + k, 511), J0], 1)
    J[J == OVERFLOW_JOINT] = OVERFLOW_JOINT - 1
    W = np.stack([0.6 + 0.1 * rng.random(len(P)), 0.25 * rng.random(len(P)), 0.15 * rng.random(len(P)), np.zeros(len(P))], 1)
    last = (len(P) - 1) // 256 * 256
    J[last:, 3] = OVERFLOW_JOINT; W[last:, 3] = 0.05
    assert (J == 511).any() and (J[:last] != OVERFLOW_JOINT).all()
    ja, wa, jd, wd = encode_set(G, J, W, "u16", "f32")
    meshes.append({"name": "g20k", "primitives": [prim(P, N, U, I, 0, {"JOINTS_0": ja, "WEIGHTS_0": wa})]})
    model[(9, 0)] = dict(joints=jd, weights=wd, dpos=[], dnrm=[], duv=[])

    # nodes: meshes, the small skin's tree, the big skin's chains (joint j is node JB + j; joint 512, when present, the last node)
    nodes = [{"name": "room", "mesh": 0}, {"name": "light", "mesh": 1, "translation": [0, -3.8, -1]},
             {"name": "multi", "mesh": 2, "skin": 0}, {"name": "reversed", "mesh": 3, "skin": 0}, {"name": "tri", "mesh": 4, "skin": 0},
             {"name": "g255a", "mesh": 5, "skin": 0}, {"name": "g255b", "mesh": 5, "skin": 0}, {"name": "g256", "mesh": 6, "skin": 0},
             {"name": "g257", "mesh": 7}, {"name": "g1000", "mesh": 8, "skin": 0}, {"name": "g20k", "mesh": 9, "skin": 1}]
    SB = len(nodes)
    for s in range(SMALL):
        n = {"name": f"s{s}", "translation": [0.4 * (-1) ** s, 0.35, 0.05 * s] if s else [0.0, -1.5, -3.0],
             "rotation": list(quat((0.3, 0.2, 1), 4 * s - 20))}
        if s == 5: n["scale"] = [1.0, 1.2, 0.9]
        ch = [c_ for c_ in (2 * s + 1, 2 * s + 2) if c_ < SMALL]
        if ch: n["children"] = [SB + c_ for c_ in ch]
        nodes.append(n)
    JB = len(nodes)
    for j in range(512):
        c_, k_ = divmod(j, LINKS)
        n = {"name": f"j{j}", "rotation": list(quat((1, 0, 0.3), 2 + k_ % 3))}
        n["translation"] = [-4.0 + 8.0 * c_ / (CHAINS - 1), -2.0, -3.8] if k_ == 0 else [0.0, 0.19, 0.0]
        if k_ < LINKS - 1 and j + 1 < 512: n["children"] = [JB + j + 1]
        nodes.append(n)
    big = [JB + j for j in range(512)]
    if big_joints == 513:
        nodes.append({"name": "j512", "translation": [0.0, 0.19, 0.0]}); nodes[JB + 511]["children"] = [len(nodes) - 1]; big.append(len(nodes) - 1)
    rw = rest_worlds(nodes)
    ib = lambda js: G.acc(np.stack([np.linalg.inv(rw(j)).T.reshape(16) for j in js]).astype(np.float32), F32, "MAT4", 1)
    skins = [{"joints": [SB + s for s in range(SMALL)], "inverseBindMatrices": ib([SB + s for s in range(SMALL)])},
             {"joints": big, "inverseBindMatrices": ib(big)}]

    def sampler(times, values, interp, typ):
        vals = np.asarray(values, np.float32)
        if typ == "SCALAR": vals = vals.reshape(-1)
        return {"input": G.acc(np.asarray(times, np.float32), F32, "SCALAR", 1), "output": G.acc(vals, F32, typ, 1), "interpolation": interp}
    cubic = lambda vals, tan: np.concatenate([np.stack([-np.asarray(t, np.float64), np.asarray(v, np.float64), np.asarray(t, np.float64)]) for v, t in zip(vals, tan)])
    kt = [0.0, 1.0, 2.0]
    # animation 0: every small-skin joint, every other big-skin joint (two shared samplers), chain 0's root, and all three meshes' weights
    s0 = [sampler(kt, [quat((0, 0, 1), 0), quat((0, 0, 1), 25), quat((1, 0, 1), -15)], "LINEAR", "VEC4"),
          sampler(kt, [quat((1, 0, 0), 2), quat((1, 0, 0), 6), quat((0, 1, 1), 4)], "LINEAR", "VEC4"),
          sampler(kt, cubic([[-4.0, -2.0, -3.8], [-3.9, -1.8, -3.7], [-4.1, -2.1, -3.9]], [[0.2, 0.1, 0]] * 3), "CUBICSPLINE", "VEC3"),
          sampler(kt, [w257, morph_weights(rng, 256), morph_weights(rng, 256)], "LINEAR", "SCALAR"),
          sampler(kt, [w1000, [x if i != BIG_WEIGHT_TARGET else -0.2 for i, x in enumerate(morph_weights(rng, 24))], w1000], "STEP", "SCALAR"),
          sampler(kt, cubic([[0.3, -0.2, 0.7], [1.4, 0.0, -0.6], [-0.3, 0.9, 0.2]], [[0.5, -0.4, 0.3]] * 3), "CUBICSPLINE", "SCALAR")]
    c0 = [(SB + s, "rotation", 0) for s in range(SMALL)] + [(JB + j, "rotation", 1) for j in range(0, 512, 2) if j % LINKS] + \
         [(JB, "translation", 2), (8, "weights", 3), (9, "weights", 4), (2, "weights", 5)]
    # animation 1: 1,000 keys on chain 1's root (translation LINEAR, rotation LINEAR and slerp)
    lk = np.arange(LONG_KEYS, dtype=np.float32) * np.float32(0.01)
    ph = np.arange(LONG_KEYS) * 0.05
    s1 = [sampler(lk, np.stack([-4.0 + 8.0 / (CHAINS - 1) + 0.1 * np.sin(ph), -2.0 + 0.1 * np.cos(ph), -3.8 + 0.05 * np.sin(3 * ph)], 1), "LINEAR", "VEC3"),
          sampler(lk, [quat((np.sin(p), 1, np.cos(p)), 30 * np.sin(p)) * (-1) ** i for i, p in enumerate(ph)], "LINEAR", "VEC4")]
    c1 = [(JB + LINKS, "translation", 0), (JB + LINKS, "rotation", 1)]
    # animation 2: the leaf joint scaled by 1e30 from t = 1; animation 3: a morph weight of 3e38 from t = 1
    s2 = [sampler([0.0, 1.0], [[1, 1, 1], [1e30, 1e30, 1e30]], "STEP", "VEC3")]
    s3 = [sampler([0.0, 1.0], [w1000, [3e38 if i == BIG_WEIGHT_TARGET else x for i, x in enumerate(w1000)]], "STEP", "SCALAR")]
    anims = [{"name": name, "samplers": s, "channels": [{"sampler": i, "target": {"node": n, "path": p}} for n, p, i in c]}
             for name, s, c in (("skin", s0, c0), ("long", s1, c1), ("joint_overflow", s2, [(JB + OVERFLOW_JOINT, "scale", 0)]),
                                ("weight_overflow", s3, [(9, "weights", 0)]))]
    g = {"asset": {"version": "2.0"}, "scene": 0, "scenes": [{"nodes": list(range(SB)) + [SB] + [JB + c_ * LINKS for c_ in range(CHAINS)]}],
         "nodes": nodes, "meshes": meshes, "materials": materials, "skins": skins, "animations": anims,
         "accessors": G.accs, "bufferViews": G.views,
         "buffers": [{"uri": "geo.bin", "byteLength": len(G.blob[0])}, {"uri": "anim.bin", "byteLength": len(G.blob[1])}]}
    return g, G.blob, model


def product_meshes(g):
    """(glTF mesh, primitive) of every loaded mesh, in load order"""
    return [(mi, pi) for mi, m in enumerate(g["meshes"]) for pi in range(len(m["primitives"]))]


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    out = {}
    for name, nj in (("shared", 512), ("global", 513)):
        d = tmp_path_factory.mktemp(name); g, blobs, model = build_scene(nj)
        out[name] = (write(d, g, blobs, name), g, blobs, model)
    return out


# ---------------------------------------------------------------- CPU
def test_hook_matches_the_model_on_513_joints_and_1000_keys(files):
    import vpt_b200 as pt
    path, g, blobs, _ = files["global"]
    assert len(g["skins"][1]["joints"]) == 513 and len(g["animations"][A_LONG]["channels"]) == 2
    keys = _acc(g, blobs, g["animations"][A_LONG]["samplers"][0]["input"])[:, 0]
    assert len(keys) == LONG_KEYS
    for a, times in ((-1, [0.0]), (A_SKIN, TIMES[A_SKIN]), (A_LONG, TIMES[A_LONG] + [float(keys[1]), float(keys[517]), float(keys[-1])])):
        for t in times:
            world, weights = pt.gltf_pose_nodes(path, a, t)
            ref_w, ref_wt = model_pose(g, blobs, a, t)
            got = world.reshape(-1, 4, 4).transpose(0, 2, 1).astype(np.float64)
            scale = np.abs(ref_w).max(axis=(1, 2), keepdims=True)
            assert (np.abs(got - ref_w) <= 64 * EPS * 4 * np.maximum(scale, 1)).all(), (a, t, np.abs(got - ref_w).max())
            for x, y in zip(weights, ref_wt):
                assert x.shape == y.shape and np.allclose(x, y, rtol=0, atol=1e-6 * max(1.0, np.abs(y).max(initial=0))), (a, t)
    d = pt.load_gltf(path)
    assert len(d["meshes"]) == len(product_meshes(g)) == 12
    assert [len(d["meshes"][m][0]) for m in range(2, 12)] == [42, 300, 90, 577, 3, 255, 256, 257, 1000, 20000]


def _small_file(tmp_path, edit, name):
    g, blobs, _ = ga.build_scene(); g = copy.deepcopy(g); edit(g)
    return write(tmp_path, g, blobs, name)


def test_too_many_targets_or_sets_are_rejected_by_the_pose(tmp_path):
    """257 targets and a 17th influence set never fail a load; the pose that needs them names them.  16 sets pose."""
    import vpt_b200 as pt
    g0, blobs, _ = ga.build_scene(); ref = pt.load_gltf(write(tmp_path, g0, blobs, "ref"))

    def targets257(g):
        p = g["meshes"][5]["primitives"][0]; p["targets"] = [p["targets"][k % 2] for k in range(257)]; g["meshes"][5].pop("weights")

    def sets(n):                                                    # sets 2 .. n - 1 repeat set 1
        def edit(g):
            at = g["meshes"][4]["primitives"][0]["attributes"]
            for s in range(2, n): at[f"JOINTS_{s}"] = at["JOINTS_1"]; at[f"WEIGHTS_{s}"] = at["WEIGHTS_1"]
        return edit

    def gap(g):
        at = g["meshes"][4]["primitives"][0]["attributes"]; at["JOINTS_2"] = at.pop("JOINTS_1"); at["WEIGHTS_2"] = at.pop("WEIGHTS_1")
    for edit, what in ((targets257, "more than 256 morph targets"), (sets(17), "JOINTS_16"), (gap, "JOINTS_2")):
        p = _small_file(tmp_path, edit, what.replace(" ", "_"))
        ga._same_load(ref, pt.load_gltf(p))
        for a in (-1, 0):
            with pytest.raises(pt.B200ptError) as e: pt.gltf_pose_nodes(p, a, 0.5)
            assert e.value.code == pt.ERR_WRONG_ARGUMENTS and what in pt.lib().b200pt_last_error(None).decode(), (what, str(e.value))
    p = _small_file(tmp_path, sets(16), "sets16")
    ga._same_load(ref, pt.load_gltf(p)); pt.gltf_pose_nodes(p, 1, 0.5)


# ---------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def pt():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import vpt_b200
    return vpt_b200


def check_pose(pt, T, path, g, blobs, model, a, t):
    """per (product mesh, quantity) the worst |GPU - model| / (2^-24 x sum of absolute terms) (the K a vertex needs), after asserting the
    instance transforms.  Generated normals are checked against the last face's normal of the GPU's own posed positions, with the absolute
    terms of that cross product over its length, and a vertex no face uses must stay NaN."""
    world, weights, wabs = model_pose(g, blobs, a, t, with_abs=True)
    d = pt.load_gltf(path); xf = T.get_instance_transforms()
    flip = np.diag([1.0, -1.0, 1.0, 1.0]); need = {}
    for mesh, (gm, pi) in enumerate(product_meshes(g)):
        if (gm, pi) not in model: continue
        node = next(i for i, nd in enumerate(g["nodes"]) if nd.get("mesh") == gm)
        skinned = "skin" in g["nodes"][node]
        Xm = flip if skinned else flip @ world[node]
        Xa = np.eye(4) if skinned else wabs[node]
        insts = [i for i, (_, m, _) in enumerate(d["instances"]) if m == mesh]
        assert len(insts) == (2 if gm == 5 else 1)
        for i in insts:
            X = xf[i].reshape(4, 4).T.astype(np.float64)
            assert np.abs(X - Xm).max() <= 64 * EPS * 4 * max(1.0, np.abs(Xm).max()), (mesh, a, t)
        got = _rows(T.get_mesh_vertices(mesh)).astype(np.float64)
        p, n, uv, pa, ua, na = _model_vertices(g, blobs, model[(gm, pi)], gm, pi, world, weights, wabs)
        gp = got[:, :3] @ X[:3, :3].T + X[:3, 3]; rp = p @ Xm[:3, :3].T + Xm[:3, 3]
        need[mesh, "position"] = (np.abs(gp - rp) / (EPS * (pa @ Xa[:3, :3].T + Xa[:3, 3]))).max()
        need[mesh, "uv"] = (np.abs(got[:, 6:8] - uv) / (EPS * np.maximum(ua, 1e-300))).max()
        if "NORMAL" not in g["meshes"][gm]["primitives"][pi]["attributes"]:   # generated: the last face's normal of the posed positions
            idx = np.asarray(d["meshes"][mesh][1], np.int64).reshape(-1, 3); P = got[:, :3]
            last = np.full(len(P), -1); last[idx.reshape(-1)] = np.repeat(np.arange(len(idx)), 3)
            e1, e2 = P[idx[:, 1]] - P[idx[:, 0]], P[idx[:, 2]] - P[idx[:, 0]]
            fn = np.cross(e1, e2); fl = np.linalg.norm(fn, axis=1, keepdims=True)
            fa = np.abs(e1[:, [1, 2, 0]] * e2[:, [2, 0, 1]]) + np.abs(e1[:, [2, 0, 1]] * e2[:, [1, 2, 0]])   # abs terms of the cross product
            assert np.isnan(got[last < 0, 3:6]).all() and (last < 0).sum() == (1 if gm == 3 else 0), (mesh, a, t)
            u = last >= 0
            need[mesh, "normal"] = (np.abs(got[u, 3:6] - fn[last[u]] / fl[last[u]]) / (EPS * (fa[last[u]] / fl[last[u]] + 1))).max()
            continue
        nrm = n / np.linalg.norm(n, axis=1, keepdims=True)
        gn = got[:, 3:6] @ ga.cofactor(X[:3, :3]).T; rn = nrm @ ga.cofactor(Xm[:3, :3]).T
        gn /= np.linalg.norm(gn, axis=1, keepdims=True); rn /= np.linalg.norm(rn, axis=1, keepdims=True)
        need[mesh, "normal"] = (np.abs(gn - rn) / (EPS * 4 * (na.max(1, keepdims=True) + 1))).max()
    assert all(np.isfinite(v) for v in need.values()), need
    return need


def _tracer(pt, path):
    return ga._file_tracer(pt, path)


def _poses():
    return [(a, t) for a in (-1, A_SKIN, A_LONG) for t in TIMES[a]]


@pytest.mark.gpu
@pytest.mark.parametrize("palette", ["shared", "global"])
def test_posed_vertices_match_the_float64_model(pt, files, palette):
    path, g, blobs, model = files[palette]
    T = _tracer(pt, path); worst = {}
    for a, t in _poses():
        T.pose(a, t)
        for key, v in check_pose(pt, T, path, g, blobs, model, a, t).items():
            assert v <= K, (key, a, t, v)
            worst[key] = max(worst.get(key, 0.0), v)
    print(f"\n{palette}: worst error / (2^-24 x sum of absolute terms), K = {K}:")
    for key in sorted(worst): print(f"  mesh {key[0]:2d} {key[1]:8s} {worst[key]:8.2f}")


@pytest.mark.gpu
def test_margin_is_tight(pt, files):
    """K / 10 rejects a vertex: vertex 256 of the 256-target mesh, whose float sum loses almost half an ulp at every term"""
    path, g, blobs, model = files["global"]
    T = _tracer(pt, path); T.pose(-1, 0.0)
    need = check_pose(pt, T, path, g, blobs, model, -1, 0.0)
    assert max(need.values()) > K / 10, need
    assert need[9, "position"] > K / 10 and need[9, "position"] <= K


@pytest.mark.gpu
def test_shared_and_global_palettes_agree_byte_for_byte(pt, files):
    S, G_ = _tracer(pt, files["shared"][0]), _tracer(pt, files["global"][0])
    for a, t in _poses():
        S.pose(a, t); G_.pose(a, t)
        for m in range(2, 12): assert _rows(S.get_mesh_vertices(m)).tobytes() == _rows(G_.get_mesh_vertices(m)).tobytes(), (m, a, t)
        assert S.get_instance_transforms().tobytes() == G_.get_instance_transforms().tobytes(), (a, t)


@pytest.mark.gpu
@pytest.mark.parametrize("palette", ["shared", "global"])
@pytest.mark.parametrize("rebuild", list(ga.REBUILDS))
def test_pose_equals_a_fresh_handle(pt, files, palette, rebuild):
    path = files[palette][0]
    A = _tracer(pt, path)
    A.path_trace(ga.F, ga.SEED)                      # in flight while the pose runs
    A.pose(A_SKIN, 1.55, rebuild=ga.REBUILDS[rebuild])
    assert A.samples_accumulated() == 0
    A.path_trace(ga.F, ga.SEED)
    B = pt.PathTracer(0); B.set_scene(ga._array_scene(pt, path, A)); ga._configure(B)
    B.path_trace(ga.F, ga.SEED)
    C0 = _tracer(pt, path); C0.path_trace(ga.F, ga.SEED)
    a, b = A.get_hdr(), B.get_hdr()
    assert np.array_equal(ti._bits(a), ti._bits(b)), int((ti._bits(a) != ti._bits(b)).any(-1).sum())
    assert np.isfinite(a).all() and a[..., :3].max() > 0
    ca, cb, c0 = A.counters(), B.counters(), C0.counters()
    assert {k: ca[k] for k in ti.WORK} == {k: cb[k] + c0[k] for k in ti.WORK}


@pytest.mark.gpu
@pytest.mark.parametrize("palette", ["shared", "global"])
def test_non_finite_pose_is_rejected_and_changes_nothing(pt, files, palette):
    """a joint scaled by 1e30 (its cofactor overflows on the device) and a morph weight of 3e38 (w x delta overflows) pass every host check;
    the device flag rejects the pose, nothing changes, and the next pose is computed in full"""
    path, g, blobs, model = files[palette]
    for a in (A_JOINT_OVERFLOW, A_WEIGHT_OVERFLOW): pt.gltf_pose_nodes(path, a, 1.0)
    T = _tracer(pt, path); T.pose(A_SKIN, 0.4); T.path_trace(2, ga.SEED)
    state = lambda: [_rows(T.get_mesh_vertices(m)).tobytes() for m in range(12)] + [T.get_instance_transforms().tobytes()]
    before = state(); img = T.get_hdr(); acc = T.samples_accumulated()
    for a in (A_JOINT_OVERFLOW, A_WEIGHT_OVERFLOW):
        for rebuild in ga.REBUILDS.values():
            with pytest.raises(pt.B200ptError) as e: T.pose(a, 1.0, rebuild=rebuild)
            assert e.value.code == pt.ERR_WRONG_ARGUMENTS and "not finite" in str(e.value), (a, str(e.value))
        assert state() == before, a
        assert T.samples_accumulated() == acc and np.array_equal(ti._bits(T.get_hdr()), ti._bits(img))
    for a, t in ((A_JOINT_OVERFLOW, 0.5), (A_WEIGHT_OVERFLOW, 0.5), (A_SKIN, 1.0)):    # the flag is reset: these pose and match the model
        T.pose(a, t)
        assert all(v <= K for v in check_pose(pt, T, path, g, blobs, model, a, t).values())
