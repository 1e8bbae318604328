"""glTF node animations, skins and morph targets (b200pt_pose): loader, host evaluation and the GPU pose kernels.

The glTF files are generated here: a lit box, a rigidly animated node chain (T / R / S on STEP, LINEAR and CUBICSPLINE), a two-bone skinned
tube (u8 joints, normalized u16 weights, a non-uniform-scale joint), an 8-influence skin (JOINTS_1), a morphing box (sparse deltas,
CUBICSPLINE weights), a mesh both morphed and skinned, a skinned mesh without normals and an emissive skinned mesh (normalized u8 weights).  Everything a pose reads
lives in a second buffer, so corrupting it cannot touch what the loader returns.

The model is a float64 restatement of glTF 2.0 Appendix C and of skinning / morphing.  The exact checks: a node no channel touches keeps its
load-time transform byte for byte, and after a pose the image equals, bit for bit, that of a fresh handle loaded with the posed arrays.
"""
import copy
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

import util
import test_instance_updates as ti

W, H, F, DEPTH = 96, 54, 4, 6
SEED = util.BASE_SEED
REBUILDS = {"refit": False, "gpu": "gpu", "host": True}
EPS = 2.0 ** -24


# ---------------------------------------------------------------- quaternions and matrices (float64)
def quat(axis, deg):
    a = np.radians(deg) / 2; ax = np.asarray(axis, np.float64); ax = ax / np.linalg.norm(ax)
    return np.array([*(np.sin(a) * ax), np.cos(a)])


def qmat(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def trs(t, r, s):
    m = np.eye(4); m[:3, :3] = qmat(r) @ np.diag(s); m[:3, 3] = t
    return m


def cofactor(m):
    """det(m) m^-T: its columns are the cross products of m's columns"""
    return np.stack([np.cross(m[:, 1], m[:, 2]), np.cross(m[:, 2], m[:, 0]), np.cross(m[:, 0], m[:, 1])], axis=1)


# ---------------------------------------------------------------- geometry
def box(c=(0, 0, 0), h=(1, 1, 1), inward=False):
    """24 vertices (per-face normals and uvs), 36 indices"""
    c = np.asarray(c, np.float64); h = np.asarray(h, np.float64)
    P, N, U, I = [], [], [], []
    for ax in range(3):
        for sgn in (-1.0, 1.0):
            n = np.zeros(3); n[ax] = sgn
            u, v = [k for k in range(3) if k != ax]
            base = len(P)
            for a, b in ((-1, -1), (1, -1), (1, 1), (-1, 1)):
                p = np.zeros(3); p[ax] = sgn; p[u] = a; p[v] = b
                P.append(c + p * h); N.append(-n if inward else n); U.append(((a + 1) / 2, (b + 1) / 2))
            q = [base, base + 1, base + 2, base, base + 2, base + 3]
            if (sgn < 0) != inward: q = [q[0], q[2], q[1], q[3], q[5], q[4]]
            I += q
    return np.array(P, np.float32), np.array(N, np.float32), np.array(U, np.float32), np.array(I, np.uint32)


def tube(rings=6, seg=8, r=0.25, length=2.0):
    P, N, U, I = [], [], [], []
    for i in range(rings + 1):
        y = length * i / rings
        for k in range(seg):
            a = 2 * np.pi * k / seg
            P.append((r * np.cos(a), y, r * np.sin(a))); N.append((np.cos(a), 0.0, np.sin(a))); U.append((k / seg, i / rings))
    for i in range(rings):
        for k in range(seg):
            a, b, c, d = i * seg + k, i * seg + (k + 1) % seg, (i + 1) * seg + k, (i + 1) * seg + (k + 1) % seg
            I += [a, c, b, b, c, d]
    return np.array(P, np.float32), np.array(N, np.float32), np.array(U, np.float32), np.array(I, np.uint32)


# ---------------------------------------------------------------- the glTF writer
class Gltf:
    def __init__(self):
        self.blob = [b"", b""]; self.views = []; self.accs = []; self.anim_accs = set()

    def acc(self, arr, comp, typ, buffer=0, normalized=False, sparse=None):
        arr = np.ascontiguousarray(arr)
        count = len(arr)
        a = {"componentType": comp, "count": count, "type": typ}
        if normalized: a["normalized"] = True
        if sparse is None:
            a["bufferView"] = self._view(arr, buffer)
        else:                                           # sparse without a bufferView: zeros, then the listed elements
            idx = np.asarray(sparse, np.uint16)
            a["sparse"] = {"count": len(idx), "indices": {"bufferView": self._view(idx, buffer), "componentType": 5123},
                           "values": {"bufferView": self._view(arr[idx.astype(np.int64)], buffer)}}
        self.accs.append(a)
        if buffer == 1: self.anim_accs.add(len(self.accs) - 1)
        return len(self.accs) - 1

    def _view(self, arr, buffer):
        b = self.blob[buffer]
        b += b"\0" * (-len(b) % 4)
        self.views.append({"buffer": buffer, "byteOffset": len(b), "byteLength": arr.nbytes}); self.blob[buffer] = b + arr.tobytes()
        return len(self.views) - 1


def build_scene():
    """(gltf dict, [geometry bin, animation bin], model) of the scene described in the module docstring"""
    G = Gltf(); F32 = 5126
    meshes, nodes, skins, anims, model = [], [], [], [], {}

    def prim(P, N, U, I, material, **attr):
        a = {"POSITION": G.acc(P, F32, "VEC3")}
        if N is not None: a["NORMAL"] = G.acc(N, F32, "VEC3")
        a["TEXCOORD_0"] = G.acc(U, F32, "VEC2")
        a.update(attr)
        return {"attributes": a, "indices": G.acc(I, 5125, "SCALAR"), "material": material}

    # materials: 0 white, 1 light, 2 red, 3 emissive skin
    materials = [{"pbrMetallicRoughness": {"baseColorFactor": [0.8, 0.8, 0.8, 1], "metallicFactor": 0.0, "roughnessFactor": 0.7}},
                 {"emissiveFactor": [1, 1, 1], "extensions": {"KHR_materials_emissive_strength": {"emissiveStrength": 6.0}},
                  "pbrMetallicRoughness": {"metallicFactor": 0.0}},
                 {"pbrMetallicRoughness": {"baseColorFactor": [0.8, 0.2, 0.1, 1], "metallicFactor": 0.0, "roughnessFactor": 0.4}},
                 {"emissiveFactor": [0.2, 0.6, 1.0], "extensions": {"KHR_materials_emissive_strength": {"emissiveStrength": 4.0}},
                  "pbrMetallicRoughness": {"metallicFactor": 0.0}}]
    # 0 room, 1 light
    meshes.append({"name": "room", "primitives": [prim(*box((0, 0, -1), (6, 4, 7), inward=True), 0)]})
    meshes.append({"name": "light", "primitives": [prim(*box((0, 0, 0), (1.2, 0.05, 0.8)), 1)]})
    # 2 cube of the node chain
    meshes.append({"name": "cube", "primitives": [prim(*box((0, 0, 0), (0.3, 0.3, 0.3)), 2)]})
    # 3 two-bone tube: u8 joints, normalized u16 weights
    tP, tN, tU, tI = tube()
    y = tP[:, 1].astype(np.float64) / 2.0
    w1 = np.clip((y - 0.3) / 0.4, 0, 1); w16 = np.round(np.stack([1 - w1, w1, 0 * w1, 0 * w1], 1) * 65535).astype(np.uint16)
    w16[:, 0] = 65535 - w16[:, 1]
    j8 = np.tile(np.array([0, 1, 0, 0], np.uint8), (len(tP), 1))
    meshes.append({"name": "tube", "primitives": [prim(tP, tN, tU, tI, 0, JOINTS_0=G.acc(j8, 5121, "VEC4", 1), WEIGHTS_0=G.acc(w16, 5123, "VEC4", 1, normalized=True))]})
    model["tube"] = dict(joints=j8.astype(np.int64), weights=w16.astype(np.float64) / 65535.0)
    # 4 tube with 8 influences (JOINTS_0 + JOINTS_1, u16 joints, float weights)
    P8, N8, U8, I8 = tube(rings=8, seg=6, r=0.2, length=1.6)
    rng = np.random.default_rng(11)
    w8 = rng.random((len(P8), 8)); w8 /= w8.sum(1, keepdims=True); w8 = w8.astype(np.float32)
    j8b = np.stack([rng.permutation(8) for _ in range(len(P8))]).astype(np.uint16)
    meshes.append({"name": "tube8", "primitives": [prim(P8, N8, U8, I8, 2, JOINTS_0=G.acc(j8b[:, :4], 5123, "VEC4", 1), JOINTS_1=G.acc(j8b[:, 4:], 5123, "VEC4", 1),
                                                        WEIGHTS_0=G.acc(w8[:, :4], F32, "VEC4", 1), WEIGHTS_1=G.acc(w8[:, 4:], F32, "VEC4", 1))]})
    model["tube8"] = dict(joints=j8b.astype(np.int64), weights=w8.astype(np.float64))
    # 5 morphing box: target 0 sparse POSITION + NORMAL, target 1 POSITION + TEXCOORD_0; mesh.weights default
    bP, bN, bU, bI = box((0, 0, 0), (0.4, 0.4, 0.4))
    d0 = np.zeros_like(bP); sp = np.array([1, 2, 5, 9, 17, 22]); d0[sp] = rng.normal(0, 0.2, (len(sp), 3))
    dn0 = rng.normal(0, 0.3, bN.shape).astype(np.float32)
    d1 = rng.normal(0, 0.1, bP.shape).astype(np.float32); du1 = rng.normal(0, 0.2, bU.shape).astype(np.float32)
    t0 = {"POSITION": G.acc(d0, F32, "VEC3", 1, sparse=sp), "NORMAL": G.acc(dn0, F32, "VEC3", 1)}
    t1 = {"POSITION": G.acc(d1, F32, "VEC3", 1), "TEXCOORD_0": G.acc(du1, F32, "VEC2", 1)}
    p5 = prim(bP, bN, bU, bI, 2); p5["targets"] = [t0, t1]
    meshes.append({"name": "morphbox", "primitives": [p5], "weights": [0.25, 0.0]})
    model["morphbox"] = dict(dpos=[d0, d1], dnrm=[dn0, None], duv=[None, du1])
    # 6 morphed and skinned tube
    mP, mN, mU, mI = tube(rings=4, seg=6, r=0.3, length=1.5)
    dm = (rng.normal(0, 0.05, mP.shape)).astype(np.float32)
    wm = np.clip(mP[:, 1:2].astype(np.float64) / 1.5, 0, 1); wm = np.concatenate([1 - wm, wm, 0 * wm, 0 * wm], 1).astype(np.float32)
    jm = np.tile(np.array([0, 1, 0, 0], np.uint8), (len(mP), 1))
    p6 = prim(mP, mN, mU, mI, 0, JOINTS_0=G.acc(jm, 5121, "VEC4", 1), WEIGHTS_0=G.acc(wm, F32, "VEC4", 1)); p6["targets"] = [{"POSITION": G.acc(dm, F32, "VEC3", 1)}]
    meshes.append({"name": "morphskin", "primitives": [p6]})
    model["morphskin"] = dict(joints=jm.astype(np.int64), weights=wm.astype(np.float64), dpos=[dm], dnrm=[None], duv=[None])
    # 7 skinned tube without normals, plus one vertex no face uses (its loaded normal is NaN)
    nP, _, nU, nI = tube(rings=3, seg=5, r=0.2, length=1.0)
    nP = np.concatenate([nP, [[0.0, 0.5, 0.0]]]).astype(np.float32); nU = np.concatenate([nU, [[0.5, 0.5]]]).astype(np.float32)
    wn = np.clip(nP[:, 1:2].astype(np.float64), 0, 1); wn = np.concatenate([1 - wn, wn, 0 * wn, 0 * wn], 1).astype(np.float32)
    jn = np.tile(np.array([0, 1, 0, 0], np.uint8), (len(nP), 1))
    meshes.append({"name": "nonormals", "primitives": [prim(nP, None, nU, nI, 2, JOINTS_0=G.acc(jn, 5121, "VEC4", 1), WEIGHTS_0=G.acc(wn, F32, "VEC4", 1))]})
    model["nonormals"] = dict(joints=jn.astype(np.int64), weights=wn.astype(np.float64))
    # 8 emissive skinned slab
    eP, eN, eU, eI = box((0, 0.6, 0), (0.5, 0.6, 0.05))
    we = np.clip(eP[:, 1:2].astype(np.float64) / 1.2, 0, 1); we = np.round(np.concatenate([1 - we, we, 0 * we, 0 * we], 1) * 255).astype(np.uint8)
    we[:, 0] = 255 - we[:, 1]                                                                               # normalized u8 weights
    je = np.tile(np.array([0, 1, 0, 0], np.uint8), (len(eP), 1))
    meshes.append({"name": "emissive", "primitives": [prim(eP, eN, eU, eI, 3, JOINTS_0=G.acc(je, 5121, "VEC4", 1), WEIGHTS_0=G.acc(we, 5121, "VEC4", 1, normalized=True))]})
    model["emissive"] = dict(joints=je.astype(np.int64), weights=we.astype(np.float64) / 255.0)

    # nodes
    nodes = [{"name": "room", "mesh": 0},                                                                   # 0
             {"name": "light", "mesh": 1, "translation": [0, -3.8, -1]},                                    # 1
             {"name": "chain0", "mesh": 2, "translation": [-2.5, 0.5, -2], "children": [3]},                # 2
             {"name": "chain1", "mesh": 2, "translation": [0.8, 0, 0], "rotation": list(quat((0, 0, 1), 20)), "children": [4]},   # 3
             {"name": "chain2", "mesh": 2, "translation": [0.8, 0, 0], "scale": [1, 0.5, 1.5]},            # 4
             {"name": "tube", "mesh": 3, "skin": 0, "translation": [5, 5, 5]},                              # 5 (its transform is ignored)
             {"name": "bone0", "translation": [0.5, -1.0, -2.5], "children": [7]},                          # 6
             {"name": "bone1", "translation": [0, 1.0, 0], "scale": [1.0, 1.3, 0.8]},                       # 7
             {"name": "tube8", "mesh": 4, "skin": 1},                                                       # 8
             {"name": "b8root", "translation": [2.0, -0.8, -2.0], "children": list(range(10, 18))}]        # 9
    for k in range(8):                                                                                      # 10 .. 17
        nodes.append({"name": f"b8_{k}", "translation": [0.05 * k, 0.2 * k, 0], "rotation": list(quat((0, 0, 1), 3 * k))})
    nodes += [{"name": "morphbox", "mesh": 5, "translation": [-1.0, 1.5, -1.5], "rotation": list(quat((1, 1, 0), 30))},   # 18
              {"name": "morphskin", "mesh": 6, "skin": 2},                                                  # 19
              {"name": "nonormals", "mesh": 7, "skin": 3},                                                  # 20
              {"name": "emissive", "mesh": 8, "skin": 4},                                                   # 21
              {"name": "mbone0", "translation": [-2.5, 1.0, -3.0], "children": [23]},                       # 22
              {"name": "mbone1", "translation": [0, 0.75, 0]}]                                              # 23
    ib = lambda ms: G.acc(np.stack([np.linalg.inv(m).T.reshape(16) for m in ms]).astype(np.float32), F32, "MAT4", 1)
    skins = [{"joints": [6, 7], "inverseBindMatrices": ib([trs((0.5, -1.0, -2.5), (0, 0, 0, 1), (1, 1, 1)), trs((0.5, 0.0, -2.5), (0, 0, 0, 1), (1, 1.3, 0.8))])},
             {"joints": list(range(10, 18))},                                                               # identity inverse binds
             {"joints": [22, 23], "inverseBindMatrices": ib([trs((-2.5, 1.0, -3.0), (0, 0, 0, 1), (1, 1, 1)), trs((-2.5, 1.75, -3.0), (0, 0, 0, 1), (1, 1, 1))])},
             {"joints": [22, 23]},
             {"joints": [6, 7], "inverseBindMatrices": ib([np.eye(4), trs((0, 0.6, 0), (0, 0, 0, 1), (1, 1, 1))])}]

    def sampler(times, values, interp, typ):
        vals = np.asarray(values, np.float32)
        if typ == "SCALAR": vals = vals.reshape(-1)                  # morph weights: keys x targets scalars
        return {"input": G.acc(np.asarray(times, np.float32), F32, "SCALAR", 1), "output": G.acc(vals, F32, typ, 1), "interpolation": interp}

    # animation 0: the node chain, T / R / S on all three modes
    kt = [0.0, 0.5, 1.2, 2.0]
    qa = [quat((0, 1, 0), 0), quat((0, 1, 0), 80), quat((0, 1, 0), 170), quat((0, 1, 0), 260)]
    qb = [quat((1, 0, 0), 10), -quat((1, 0, 0), 60), quat((1, 0, 0), 140), -quat((1, 0, 0), 200)]   # sign flips: slerp takes the short way
    cubic = lambda vals, tan: np.concatenate([np.stack([-np.asarray(t, np.float64), np.asarray(v, np.float64), np.asarray(t, np.float64)]) for v, t in zip(vals, tan)])
    s0 = [sampler(kt, [[-2.5, 0.5, -2], [-2.2, 0.9, -2.1], [-2.6, 0.2, -1.8], [-2.4, 0.6, -2.2]], "LINEAR", "VEC3"),
          sampler(kt, qa, "STEP", "VEC4"),
          sampler(kt, qb, "LINEAR", "VEC4"),
          sampler(kt, cubic([[1, 1, 1], [1.4, 0.8, 1.1], [0.7, 1.2, 0.9], [1, 1, 1]], [[0.5, -0.2, 0.1]] * 4), "CUBICSPLINE", "VEC3"),
          sampler(kt, [[0.8, 0, 0], [0.9, 0.2, 0], [0.7, -0.1, 0.2], [0.8, 0, 0]], "STEP", "VEC3"),
          sampler(kt, cubic([quat((0, 0, 1), 0), quat((0, 0, 1), 45), quat((0, 1, 1), 90), quat((0, 0, 1), 10)], [[0.1, 0.2, -0.1, 0.05]] * 4), "CUBICSPLINE", "VEC4"),
          sampler(kt, [[1, 0.5, 1.5], [1.2, 0.7, 1.0], [0.9, 0.4, 1.3], [1, 0.5, 1.5]], "LINEAR", "VEC3")]
    c0 = [(2, "translation", 0), (2, "rotation", 1), (3, "rotation", 2), (3, "scale", 3), (4, "translation", 4), (4, "rotation", 5), (4, "scale", 6)]
    anims.append({"name": "chain", "samplers": s0, "channels": [{"sampler": s, "target": {"node": n, "path": p}} for n, p, s in c0]})
    # animation 1: skins and morph weights
    kb = [0.2, 1.0, 1.7]
    s1 = [sampler(kb, [quat((0, 0, 1), 0), quat((0, 0, 1), 50), quat((1, 0, 1), -40)], "LINEAR", "VEC4"),               # bone1 rotation
          sampler(kb, cubic([[0.5, -1.0, -2.5], [0.7, -0.9, -2.4], [0.4, -1.1, -2.6]], [[0.3, 0.1, 0]] * 3), "CUBICSPLINE", "VEC3"),   # bone0 translation
          sampler(kb, cubic([[0.25, 0.0], [0.8, 0.5], [0.1, 1.0]], [[0.4, -0.3]] * 3), "CUBICSPLINE", "SCALAR"),          # morphbox weights
          sampler(kb, [[0.0], [1.0], [0.5]], "LINEAR", "SCALAR"),                                                          # morphskin weights
          sampler(kb, [quat((0, 0, 1), 0), quat((0, 0, 1), 35), quat((0, 0, 1), -20)], "LINEAR", "VEC4"),              # mbone1 rotation
          sampler(kb, [quat((0, 0, 1), 0), quat((1, 0, 0), 25), quat((0, 1, 0), 15)], "LINEAR", "VEC4")]               # the 8 joints
    c1 = [(7, "rotation", 0), (6, "translation", 1), (18, "weights", 2), (19, "weights", 3), (23, "rotation", 4)] + [(10 + k, "rotation", 5) for k in range(0, 8, 2)]
    anims.append({"name": "bend", "samplers": s1, "channels": [{"sampler": s, "target": {"node": n, "path": p}} for n, p, s in c1]})
    anims.append({"name": "empty", "samplers": [], "channels": []})
    g = {"asset": {"version": "2.0"}, "scene": 0, "scenes": [{"nodes": [0, 1, 2, 5, 6, 8, 9, 18, 19, 20, 21, 22]}],
         "nodes": nodes, "meshes": meshes, "materials": materials, "skins": skins, "animations": anims,
         "accessors": G.accs, "bufferViews": G.views,
         "buffers": [{"uri": "geo.bin", "byteLength": len(G.blob[0])}, {"uri": "anim.bin", "byteLength": len(G.blob[1])}]}
    model["anim_accessors"] = sorted(G.anim_accs)
    return g, G.blob, model


def write(tmp_path, g, blobs, name="anim"):
    (tmp_path / "geo.bin").write_bytes(blobs[0]); (tmp_path / "anim.bin").write_bytes(blobs[1])
    p = tmp_path / f"{name}.gltf"; p.write_text(json.dumps(g))
    return str(p)


@pytest.fixture
def scene(tmp_path):
    g, blobs, model = build_scene()
    return write(tmp_path, g, blobs), g, blobs, model


def stripped(g):
    """the same file without skins, animations, morph targets and morph weights"""
    g = copy.deepcopy(g)
    g.pop("skins", None); g.pop("animations", None)
    for m in g["meshes"]:
        m.pop("weights", None)
        for p in m["primitives"]: p.pop("targets", None)
    for n in g["nodes"]: n.pop("skin", None); n.pop("weights", None)
    return g


# ---------------------------------------------------------------- the float64 model (glTF 2.0 Appendix C)
def _acc(g, blobs, i):
    a = g["accessors"][i]
    nc = {"SCALAR": 1, "VEC2": 2, "VEC3": 3, "VEC4": 4, "MAT4": 16}[a["type"]]
    dt = {5126: np.float32, 5121: np.uint8, 5123: np.uint16, 5125: np.uint32}[a["componentType"]]
    out = np.zeros((a["count"], nc), np.float64)
    def view(v, off, n, dtype, k):
        bv = g["bufferViews"][v]
        return np.frombuffer(blobs[bv["buffer"]], dtype, n * k, bv["byteOffset"] + off).reshape(n, k).astype(np.float64)
    if "bufferView" in a: out = view(a["bufferView"], a.get("byteOffset", 0), a["count"], dt, nc)
    if "sparse" in a:
        s = a["sparse"]; idt = {5121: np.uint8, 5123: np.uint16, 5125: np.uint32}[s["indices"]["componentType"]]
        ix = view(s["indices"]["bufferView"], 0, s["count"], idt, 1)[:, 0].astype(np.int64)
        out[ix] = view(s["values"]["bufferView"], 0, s["count"], dt, nc)
    if a.get("normalized"): out = out / {5121: 255.0, 5123: 65535.0}[a["componentType"]]
    return out


def sample(g, blobs, smp, t, rotation):
    ti_ = _acc(g, blobs, smp["input"])[:, 0]; out = _acc(g, blobs, smp["output"])
    K = len(ti_); interp = smp.get("interpolation", "LINEAR"); cubic = interp == "CUBICSPLINE"
    n = out.size // (K * (3 if cubic else 1))
    out = out.reshape(K, 3, n) if cubic else out.reshape(K, n)
    val = (lambda k: out[k, 1]) if cubic else (lambda k: out[k])
    if K == 1 or t <= ti_[0]: return val(0).copy()
    if t >= ti_[-1]: return val(K - 1).copy()
    k = int(np.searchsorted(ti_, t, side="right")) - 1
    td = ti_[k + 1] - ti_[k]; u = (t - ti_[k]) / td
    a, b = val(k), val(k + 1)
    if interp == "STEP": return a.copy()
    if interp == "LINEAR":
        if not rotation: return (1 - u) * a + u * b
        d = float(np.dot(a, b)); s = -1.0 if d < 0 else 1.0
        if abs(d) > 1 - 1e-9: return (1 - u) * a + s * u * b
        ang = np.arccos(abs(d))
        return np.sin(ang * (1 - u)) / np.sin(ang) * a + s * np.sin(ang * u) / np.sin(ang) * b
    u2, u3 = u * u, u * u * u
    v = (2 * u3 - 3 * u2 + 1) * a + td * (u3 - 2 * u2 + u) * out[k, 2] + (-2 * u3 + 3 * u2) * b + td * (u3 - u2) * out[k + 1, 0]
    return v / np.linalg.norm(v) if rotation else v


def model_pose(g, blobs, animation, t, with_abs=False):
    """(world [nodes, 4, 4], weights per node) in float64; with_abs: also the world matrices of the absolute values of every factor, the
    per-entry sum of absolute terms of the product chain"""
    N = g["nodes"]
    T = [np.array(n.get("translation", [0, 0, 0]), np.float64) for n in N]
    R = [np.array(n.get("rotation", [0, 0, 0, 1]), np.float64) for n in N]
    S = [np.array(n.get("scale", [1, 1, 1]), np.float64) for n in N]
    Wt = []
    for n in N:
        m = g["meshes"][n["mesh"]] if "mesh" in n else None
        nt = len(m["primitives"][0].get("targets", [])) if m else 0
        Wt.append(np.array(n["weights"] if "weights" in n else m.get("weights", [0.0] * nt) if nt else [], np.float64))
    if animation >= 0:
        A = g["animations"][animation]
        for ch in A["channels"]:
            nd, path = ch["target"]["node"], ch["target"]["path"]
            v = sample(g, blobs, A["samplers"][ch["sampler"]], float(np.float32(t)), path == "rotation")
            {"translation": T, "rotation": R, "scale": S, "weights": Wt}[path][nd] = np.asarray(v, np.float64).reshape(-1)
    parent = {c: i for i, n in enumerate(N) for c in n.get("children", [])}
    world = [None] * len(N); wabs = [None] * len(N)
    def wm(i):
        if world[i] is None:
            if "matrix" in N[i]: loc = np.array(N[i]["matrix"], np.float64).reshape(4, 4).T; la = np.abs(loc)
            else:
                loc = trs(T[i], R[i], S[i]); rm = np.eye(4); rm[:3, :3] = qmat(R[i])
                la = np.abs(trs(T[i], (0, 0, 0, 1), (1, 1, 1))) @ np.abs(rm) @ np.diag([*np.abs(S[i]), 1.0])
            world[i] = (wm(parent[i]) if i in parent else np.eye(4)) @ loc
            wabs[i] = (wabs[parent[i]] if i in parent else np.eye(4)) @ la
        return world[i]
    out = np.stack([wm(i) for i in range(len(N))])
    return (out, Wt, np.stack(wabs)) if with_abs else (out, Wt)


# ---------------------------------------------------------------- CPU: the loader returns what it returned, the hook matches the model
def _same_load(a, b):
    assert len(a["meshes"]) == len(b["meshes"])
    for (va, ia), (vb, ib_) in zip(a["meshes"], b["meshes"]):
        assert va.tobytes() == vb.tobytes() and ia.tobytes() == ib_.tobytes()
    assert a["materials_bytes"].tobytes() == b["materials_bytes"].tobytes()
    assert [t.tobytes() for t in a["textures"]] == [t.tobytes() for t in b["textures"]]
    assert [(x.tobytes(), m, k) for x, m, k in a["instances"]] == [(x.tobytes(), m, k) for x, m, k in b["instances"]]
    assert a["camera_view"].tobytes() == b["camera_view"].tobytes() and a["aspect"] == b["aspect"]


def test_load_is_byte_identical_without_the_animation_blocks(scene, tmp_path):
    import vpt_b200 as pt
    path, g, blobs, _ = scene
    full = pt.load_gltf(path)
    _same_load(full, pt.load_gltf(write(tmp_path, stripped(g), blobs, "plain")))
    assert len(full["meshes"]) == 9 and len(full["instances"]) == 11      # the chain's cube is instanced by three nodes
    v7 = full["meshes"][7][0]                                              # generated normals; the vertex no face uses is NaN
    assert np.isnan(v7["nrm"][-1]).all() and np.isfinite(v7["nrm"][:-1]).all()


def test_animations_are_listed(scene):
    import vpt_b200 as pt
    path = scene[0]
    assert pt.gltf_animations(path) == [("chain", 0.0, 2.0), ("bend", np.float32(0.2), np.float32(1.7)), ("empty", 0.0, 0.0)]
    L = pt.lib(); n = C.c_uint32()
    assert L.b200pt_gltf_animation_info(path.encode(), 3, C.byref(n), None, 0, None, None) == pt.ERR_WRONG_ARGUMENTS
    assert L.b200pt_gltf_animation_info(None, 0, C.byref(n), None, 0, None, None) == pt.ERR_WRONG_ARGUMENTS
    for f in ("b200pt_animation_count", "b200pt_get_animation", "b200pt_pose", "b200pt_gltf_animation_info", "b200pt_gltf_pose_nodes"):
        assert f in pt.declared_symbols()
    assert L.b200pt_pose(None, 0, C.c_float(0.0), 0) == pt.ERR_WRONG_ARGUMENTS
    assert L.b200pt_animation_count(None, C.byref(n)) == pt.ERR_WRONG_ARGUMENTS


TIMES = {0: [-1.0, 0.0, 0.25, 0.5, 0.8, 1.2, 1.6, 2.0, 3.5], 1: [0.0, 0.2, 0.45, 1.0, 1.3, 1.7, 9.0], 2: [0.0, 1.0], -1: [0.0]}


def test_hook_matches_the_float64_model(scene):
    import vpt_b200 as pt
    path, g, blobs, _ = scene
    for a, times in TIMES.items():
        for t in times:
            world, weights = pt.gltf_pose_nodes(path, a, t)
            ref_w, ref_wt = model_pose(g, blobs, a, t)
            got = world.reshape(-1, 4, 4).transpose(0, 2, 1).astype(np.float64)
            scale = np.abs(ref_w).max(axis=(1, 2), keepdims=True)
            assert (np.abs(got - ref_w) <= 64 * EPS * 4 * np.maximum(scale, 1)).all(), (a, t, np.abs(got - ref_w).max())
            assert len(weights) == len(ref_wt)
            for x, y in zip(weights, ref_wt):
                assert x.shape == y.shape and np.allclose(x, y, rtol=0, atol=1e-6), (a, t, x, y)
    # a node no channel of the chain animation touches keeps its loaded world matrix; an untouched node under an animated one does not
    w0, _ = pt.gltf_pose_nodes(path, -1, 0.0); w1, _ = pt.gltf_pose_nodes(path, 0, 0.8)
    untouched = [0, 1, 5, 6, 7, 8, 9, 18]
    assert w0[untouched].tobytes() == w1[untouched].tobytes() and not np.array_equal(w0[3], w1[3])


def _mutate(rng, g, model):
    """one random corruption of the animation blocks (never of what the geometry reads)"""
    g = copy.deepcopy(g)
    bad = [-1, 10 ** 9, 2.5, "x", None, len(g["nodes"]), len(g["accessors"]), 0, 1, 3]
    kind = rng.integers(0, 9)
    pick = lambda seq: seq[int(rng.integers(0, len(seq)))]
    if kind == 0:
        s = pick(g["skins"]); s["joints"][int(rng.integers(0, len(s["joints"])))] = pick(bad)
    elif kind == 1:
        s = pick(g["skins"]); s["inverseBindMatrices"] = pick(bad)
    elif kind == 2:
        a = pick(g["animations"][:2]); ch = pick(a["channels"]); ch["target"][pick(["node", "path"])] = pick(bad + ["weights", "rotation", "pointer"])
    elif kind == 3:
        a = pick(g["animations"][:2]); s = pick(a["samplers"]); s[pick(["input", "output", "interpolation"])] = pick(bad + ["CUBICSPLINE", "STEP"])
    elif kind == 4:
        i = pick(model["anim_accessors"]); g["accessors"][i][pick(["count", "componentType", "type", "bufferView", "byteOffset"])] = pick(bad + ["VEC2", "MAT4", 5121, 2 ** 31])
    elif kind == 5:
        m = g["meshes"][5]; m["primitives"][0]["targets"][int(rng.integers(0, 2))][pick(["POSITION", "NORMAL", "TEXCOORD_0"])] = pick(bad)
    elif kind == 6:
        m = pick(g["meshes"][3:9]); m["primitives"][0]["attributes"][pick(["JOINTS_0", "WEIGHTS_0", "JOINTS_1"])] = pick(bad)
    elif kind == 7:
        n = pick(g["nodes"]); n[pick(["skin", "weights"])] = pick(bad + [[0.5], [1.0, 2.0], [float("nan"), 0.0]])
    else:
        i = pick(model["anim_accessors"]); a = g["accessors"][i]
        if "sparse" in a: a["sparse"]["count"] = pick(bad)
        else: g["meshes"][5]["weights"] = pick(bad + [[0.1], [1, 2, 3]])
    return g


def test_corrupt_animation_data_never_fails_a_load(scene, tmp_path):
    import vpt_b200 as pt
    path, g, blobs, model = scene
    ref = pt.load_gltf(path)
    rng = np.random.default_rng(7)
    outcomes = {"posed": 0, "rejected": 0}
    for it in range(160):
        gi, bi = g, list(blobs)
        if it % 4 == 3:                                                     # byte flips or truncation of the animation buffer
            b = bytearray(blobs[1])
            if it % 8 == 3: b = b[:int(rng.integers(0, len(b)))]
            else:
                for k in rng.integers(0, len(b), 24): b[k] ^= int(rng.integers(1, 256))
            bi[1] = bytes(b)
        else:
            gi = _mutate(rng, g, model)
        p = write(tmp_path, gi, bi, f"c{it}")
        _same_load(ref, pt.load_gltf(p))
        pt.gltf_animations(p)
        for a in (-1, 0, 1):
            try:
                pt.gltf_pose_nodes(p, a, 0.7); outcomes["posed"] += 1
            except pt.B200ptError as e:
                assert e.code == pt.ERR_WRONG_ARGUMENTS, e; outcomes["rejected"] += 1
    assert outcomes["posed"] and outcomes["rejected"]


def test_malformed_data_is_named_by_the_pose(scene, tmp_path):
    import vpt_b200 as pt
    path, g, blobs, _ = scene
    cases = {"joint index out of range": lambda g: g["skins"][0]["joints"].__setitem__(1, 99),
             "input times do not increase": None,
             "two ways": lambda g: g["nodes"].append({"mesh": 3, "skin": 1}) or g["scenes"][0]["nodes"].append(len(g["nodes"]) - 1),
             "different morph weights": lambda g: g["nodes"].append({"mesh": 5, "weights": [0.5, 0.5]}) or g["scenes"][0]["nodes"].append(len(g["nodes"]) - 1)}
    for what, edit in cases.items():
        gi = copy.deepcopy(g); bi = list(blobs)
        if edit: edit(gi)
        else:                                                               # keys of the chain's first sampler: 0, 0.5, 0.5, 2
            a = gi["accessors"][gi["animations"][0]["samplers"][0]["input"]]; bv = gi["bufferViews"][a["bufferView"]]
            b = bytearray(bi[1]); b[bv["byteOffset"] + 8:bv["byteOffset"] + 12] = np.float32(0.5).tobytes(); bi[1] = bytes(b)
        p = write(tmp_path, gi, bi, what.replace(" ", "_"))
        pt.load_gltf(p)
        anim = 0 if edit is None else -1
        with pytest.raises(pt.B200ptError) as e: pt.gltf_pose_nodes(p, anim, 0.3)
        assert e.value.code == pt.ERR_WRONG_ARGUMENTS and what in pt.lib().b200pt_last_error(None).decode(), (what, str(e.value))
    for bad in ((3, 0.0), (-2, 0.0), (0, float("nan")), (0, float("inf"))):
        with pytest.raises(pt.B200ptError) as e: pt.gltf_pose_nodes(path, *bad)
        assert e.value.code == pt.ERR_WRONG_ARGUMENTS


# ---------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def pt():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import vpt_b200
    return vpt_b200


def _configure(T):
    import vpt_b200 as P
    raw, _, _ = util.env_small()
    T.set_env_map(raw); T.set_luts(*util.luts())
    T.set_config(P.default_config(MaxDepth=DEPTH)); T.resize(W, H)
    return T


def _file_tracer(pt, path):
    T = pt.PathTracer(0); T.set_scene_file(path)
    return _configure(T)


def _array_scene(pt, path, T):
    """the load of `path` with T's current vertices and instance transforms"""
    d = pt.load_gltf(path)
    meshes = [(T.get_mesh_vertices(m), idx) for m, (_, idx) in enumerate(d["meshes"])]
    xf = T.get_instance_transforms()
    return dict(meshes=meshes, materials=d["materials_bytes"].view(np.dtype((np.void, 112))), textures=d["textures"],
                instances=[(xf[i], m, k) for i, (_, m, k) in enumerate(d["instances"])], camera_view=d["camera_view"], aspect=d["aspect"])


def _rows(v):
    return np.ascontiguousarray(v).view(np.float32).reshape(-1, 8)


DEFORMED = {3: "tube", 4: "tube8", 5: "morphbox", 6: "morphskin", 7: "nonormals", 8: "emissive"}   # mesh index: model key


def _model_vertices(g, blobs, M, mesh, prim, world, weights, wabs):
    """float64 posed (positions, raw normals, uvs, abs-term sums for position / uv, cofactor abs-term sums) of primitive `prim` of glTF
    mesh `mesh`, in the space its vertices are stored in.  M: that primitive's influences (joints / weights [vertex, 4 * sets]) and morph
    deltas per target (dpos / dnrm / duv, None where the target lacks the attribute)"""
    prim = g["meshes"][mesh]["primitives"][prim]; at = prim["attributes"]
    p = _acc(g, blobs, at["POSITION"]); uv = _acc(g, blobs, at["TEXCOORD_0"])
    n = _acc(g, blobs, at["NORMAL"]) if "NORMAL" in at else np.zeros_like(p)
    pa, ua, na = np.abs(p), np.abs(uv), np.abs(n)
    node = next(i for i, nd in enumerate(g["nodes"]) if nd.get("mesh") == mesh)
    for t, w in enumerate(weights[node] if "targets" in prim else []):
        if w == 0: continue
        for arr, absarr, d in ((p, pa, M["dpos"][t]), (n, na, M["dnrm"][t]), (uv, ua, M["duv"][t])):
            if d is not None: arr += w * d; absarr += abs(w) * np.abs(d)
    cof_abs = np.ones_like(p)
    if "skin" in g["nodes"][node]:
        sk = g["skins"][g["nodes"][node]["skin"]]
        ibm = _acc(g, blobs, sk["inverseBindMatrices"]).reshape(-1, 4, 4).transpose(0, 2, 1) if "inverseBindMatrices" in sk else np.tile(np.eye(4), (len(sk["joints"]), 1, 1))
        J = np.stack([world[j] @ ibm[k] for k, j in enumerate(sk["joints"])])
        Jabs = np.stack([wabs[j] @ np.abs(ibm[k]) for k, j in enumerate(sk["joints"])])   # the terms of world(joint) x inverseBind
        Mv = np.einsum("vi,vijk->vjk", M["weights"], J[M["joints"]])
        Ma = np.einsum("vi,vijk->vjk", np.abs(M["weights"]), Jabs[M["joints"]])
        ph = np.concatenate([p, np.ones((len(p), 1))], 1); pah = np.concatenate([pa, np.ones((len(p), 1))], 1)
        p = np.einsum("vjk,vk->vj", Mv, ph)[:, :3]; pa = np.einsum("vjk,vk->vj", Ma, pah)[:, :3]
        m3 = Mv[:, :3, :3]                                              # cofactor() of every vertex's matrix at once
        cof = np.stack([np.cross(m3[:, :, 1], m3[:, :, 2]), np.cross(m3[:, :, 2], m3[:, :, 0]), np.cross(m3[:, :, 0], m3[:, :, 1])], axis=2)
        cof_abs = np.einsum("vjk,vk->vj", np.abs(cof), na) / np.maximum(np.linalg.norm(np.einsum("vjk,vk->vj", cof, n), axis=1, keepdims=True), 1e-300)
        n = np.einsum("vjk,vk->vj", cof, n)
    else:
        cof_abs = na / np.maximum(np.linalg.norm(n, axis=1, keepdims=True), 1e-300)
    return p, n, uv, pa, ua, cof_abs


def _check_pose(pt, T, path, g, blobs, model, a, t):
    world, weights, wabs = model_pose(g, blobs, a, t, with_abs=True)
    d = pt.load_gltf(path); xf = T.get_instance_transforms()
    for mesh in DEFORMED:
        got = _rows(T.get_mesh_vertices(mesh)).astype(np.float64)
        p, n, uv, pa, ua, na = _model_vertices(g, blobs, model[DEFORMED[mesh]], mesh, 0, world, weights, wabs)   # one primitive per mesh
        inst = next(i for i, (_, m, _) in enumerate(d["instances"]) if m == mesh)
        X = xf[inst].reshape(4, 4).T.astype(np.float64)
        skinned = "skin" in g["nodes"][next(i for i, nd in enumerate(g["nodes"]) if nd.get("mesh") == mesh)]
        flip = np.diag([1.0, -1.0, 1.0, 1.0])
        Xm = flip if skinned else flip @ world[next(i for i, nd in enumerate(g["nodes"]) if nd.get("mesh") == mesh)]
        assert np.abs(X - Xm).max() <= 64 * EPS * 4 * max(1.0, np.abs(Xm).max()), mesh
        gp = got[:, :3] @ X[:3, :3].T + X[:3, 3]; rp = p @ Xm[:3, :3].T + Xm[:3, 3]
        Xa = np.diag([1.0, 1.0, 1.0, 1.0]) if skinned else wabs[next(i for i, nd in enumerate(g["nodes"]) if nd.get("mesh") == mesh)]
        tol = 64 * EPS * (pa @ Xa[:3, :3].T + Xa[:3, 3])
        assert (np.abs(gp - rp) <= tol).all(), (mesh, a, t, np.abs(gp - rp).max(), tol.min())
        assert (np.abs(got[:, 6:8] - uv) <= 64 * EPS * ua).all(), (mesh, a, t)
        if mesh == 7:                                                       # generated: the last face's normal of the posed positions
            idx = np.asarray(d["meshes"][7][1], np.int64).reshape(-1, 3); P = got[:, :3]
            last = np.full(len(P), -1); last[idx.reshape(-1)] = np.repeat(np.arange(len(idx)), 3)
            fn = np.cross(P[idx[:, 1]] - P[idx[:, 0]], P[idx[:, 2]] - P[idx[:, 0]]); fn /= np.linalg.norm(fn, axis=1, keepdims=True)
            assert np.isnan(got[last < 0, 3:6]).all() and (last < 0).sum() == 1
            assert np.allclose(got[last >= 0, 3:6], fn[last[last >= 0]], rtol=0, atol=1e-5), (a, t)
            continue
        nrm = n / np.linalg.norm(n, axis=1, keepdims=True)
        gn = got[:, 3:6] @ cofactor(X[:3, :3]).T; rn = nrm @ cofactor(Xm[:3, :3]).T
        gn /= np.linalg.norm(gn, axis=1, keepdims=True); rn /= np.linalg.norm(rn, axis=1, keepdims=True)
        assert (np.abs(gn - rn) <= 64 * EPS * 4 * (na.max(1, keepdims=True) + 1)).all(), (mesh, a, t, np.abs(gn - rn).max())


@pytest.mark.gpu
def test_posed_vertices_match_the_float64_model(pt, tmp_path):
    g, blobs, model = build_scene(); path = write(tmp_path, g, blobs)
    T = _file_tracer(pt, path)
    assert T.animations() == pt.gltf_animations(path)
    for a in (-1, 0, 1):
        for t in TIMES[a]:
            T.pose(a, t)
            _check_pose(pt, T, path, g, blobs, model, a, t)


@pytest.mark.gpu
def test_rest_pose_keeps_what_the_load_gave(pt, tmp_path):
    g, blobs, model = build_scene(); path = write(tmp_path, g, blobs)
    T = _file_tracer(pt, path); d = pt.load_gltf(path)
    xf0 = T.get_instance_transforms()
    for a, t in ((-1, 0.0), (0, 0.8), (1, 1.3)):
        T.pose(a, t, rebuild="gpu")
        xf = T.get_instance_transforms()
        for i, (x, m, _) in enumerate(d["instances"]):
            if m in (0, 1): assert xf[i].tobytes() == x.tobytes() == xf0[i].tobytes()      # room and light: untouched nodes
        for m in (0, 1, 2): assert _rows(T.get_mesh_vertices(m)).tobytes() == _rows(d["meshes"][m][0]).tobytes()
    T.pose(-1, 0.0)                                  # the morph-only box at rest: the loaded vertices bit for bit
    assert _rows(T.get_mesh_vertices(5)).tobytes() != _rows(d["meshes"][5][0]).tobytes()       # mesh.weights = [0.25, 0]
    gz = copy.deepcopy(g); gz["meshes"][5]["weights"] = [0.0, 0.0]; pz = write(tmp_path, gz, blobs, "zero")
    Z = _file_tracer(pt, pz); Z.pose(-1, 0.0)
    assert _rows(Z.get_mesh_vertices(5)).tobytes() == _rows(pt.load_gltf(pz)["meshes"][5][0]).tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("rebuild", list(REBUILDS))
def test_pose_equals_a_fresh_handle(pt, tmp_path, rebuild):
    g, blobs, model = build_scene(); path = write(tmp_path, g, blobs)
    A = _file_tracer(pt, path)
    A.path_trace(F, SEED)                            # in flight while the pose runs
    A.pose(1, 1.3, rebuild=REBUILDS[rebuild])
    assert A.samples_accumulated() == 0
    A.path_trace(F, SEED)
    B = pt.PathTracer(0); B.set_scene(_array_scene(pt, path, A)); _configure(B)
    B.path_trace(F, SEED)
    C0 = _file_tracer(pt, path); C0.path_trace(F, SEED)
    a, b = A.get_hdr(), B.get_hdr()
    assert np.array_equal(ti._bits(a), ti._bits(b)), int((ti._bits(a) != ti._bits(b)).any(-1).sum())
    assert np.isfinite(a).all() and a[..., :3].max() > 0
    ca, cb, c0 = A.counters(), B.counters(), C0.counters()
    assert {k: ca[k] for k in ti.WORK} == {k: cb[k] + c0[k] for k in ti.WORK}


@pytest.mark.gpu
def test_pose_depends_only_on_file_animation_and_time(pt, tmp_path):
    g, blobs, model = build_scene(); path = write(tmp_path, g, blobs)
    A = _file_tracer(pt, path); B = _file_tracer(pt, path)
    A.update_mesh_vertices({3: _rows(A.get_mesh_vertices(3)) * 1.5})        # replaced by the pose
    A.pose(0, 0.3); A.pose(1, 0.6); A.pose(1, 1.45)
    B.pose(1, 1.45)
    for m in range(9): assert _rows(A.get_mesh_vertices(m)).tobytes() == _rows(B.get_mesh_vertices(m)).tobytes(), m
    assert A.get_instance_transforms().tobytes() == B.get_instance_transforms().tobytes()
    A.path_trace(F, SEED); B.path_trace(F, SEED)
    assert np.array_equal(ti._bits(A.get_hdr()), ti._bits(B.get_hdr()))


@pytest.mark.gpu
def test_rejected_poses_change_nothing(pt, tmp_path):
    g, blobs, model = build_scene(); path = write(tmp_path, g, blobs)
    E = pt.PathTracer(0)
    with pytest.raises(pt.B200ptError) as e: E.pose(0, 0.0)
    assert e.value.code == pt.ERR_NO_SCENE
    arr = pt.PathTracer(0); arr.set_scene(util.scene_dict("cornell_box")); _configure(arr)
    for call in (lambda: arr.pose(-1, 0.0), arr.animations):
        with pytest.raises(pt.B200ptError) as e: call()
        assert e.value.code == pt.ERR_NO_SCENE
    gw = copy.deepcopy(g); gw["nodes"].append({"mesh": 3, "skin": 1}); gw["scenes"][0]["nodes"].append(len(gw["nodes"]) - 1)
    gb = copy.deepcopy(g); gb["animations"][0]["channels"][0]["target"]["node"] = 999
    for p, bad in ((path, [(3, 0.0), (-2, 0.0), (0, float("nan")), (1, float("inf"))]),
                   (write(tmp_path, gw, blobs, "twoways"), [(-1, 0.0), (1, 0.5)]),
                   (write(tmp_path, gb, blobs, "badnode"), [(0, 0.5)])):
        A = _file_tracer(pt, p)
        if p == path: A.pose(1, 0.9)
        A.path_trace(2, SEED)
        before = [_rows(A.get_mesh_vertices(m)).tobytes() for m in range(9)] + [A.get_instance_transforms().tobytes()]
        img = A.get_hdr(); acc = A.samples_accumulated()
        for a, t in bad:
            for rebuild in REBUILDS.values():
                with pytest.raises(pt.B200ptError) as e: A.pose(a, t, rebuild=rebuild)
                assert e.value.code == pt.ERR_WRONG_ARGUMENTS, (p, a, t)
        assert [_rows(A.get_mesh_vertices(m)).tobytes() for m in range(9)] + [A.get_instance_transforms().tobytes()] == before
        assert A.samples_accumulated() == acc and np.array_equal(ti._bits(A.get_hdr()), ti._bits(img))


@pytest.mark.gpu
def test_cli_pose_equals_python_pose(pt, tmp_path):
    g, blobs, model = build_scene(); path = write(tmp_path, g, blobs)
    exe = os.path.join(os.path.dirname(pt.LIB_PATH), "b200pt_render")
    hdr = str(tmp_path / "env.hdr"); util.write_rgbe(hdr, util.gltf_ref.synthetic_env(64, 32, 5)[..., :3])
    luts = util.write_luts_dir(tmp_path / "luts")
    out = str(tmp_path / "cli.png")
    r = subprocess.run([exe, "--scene", path, "--env", hdr, "--luts", luts, "--size", str(W), str(H), "--depth", str(DEPTH), "--spp", "4",
                        "--batch", "4", "--quiet", "--animation", "1", "--time", "1.1", "--out", out], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    T = pt.PathTracer(0); T.set_luts_dir(luts); T.set_env_map_file(hdr); T.set_scene_file(path)
    T.pose(1, 1.1, rebuild=True); T.resize(W, H)
    cfg = T.get_config(); cfg.MaxDepth = DEPTH; cfg.MaxSamplesAccumulated = 4; T.set_config(cfg)
    T.path_trace(4, 0x1234ABCD); T.synchronize(); T.post_process()
    assert np.array_equal(pt.decode_image(out), T.get_ldr())
