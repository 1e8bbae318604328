"""One bounce of the renderer, path by path (b200pt_bounce_query): the extension ray, the mesh-medium branch at the head of k_shade_hit,
the NEE join, the path epilogue (path_roulette / path_radiance, finish_missed_path), the fold into the sample slot (finish_path_slot) and
the warp-ballot compaction of the survivors, in the launch sequence Engine::path_trace runs (fused k_shade_hit, k_shade_hit + k_connect, or
k_shadow_dyn + k_connect<TRACE=false>), on caller-given paths: Depths 0, 1, 2 and MaxDepth - 1, throughputs of 0, > 1, 3e38, +Inf and NaN,
subnormal and zero pdfs, radiance that is already NaN or Inf, channel-split paths, paths inside a medium with densities from negative to
large and anisotropies -0.9, 0, 0.9 and 1 (the Beer-law case), sampler states whose first draw is exactly 1 (a miss's roulette draw; inside
a medium, sd = -0: a scatter at the origin).

Model (numpy), record by record, on the steps the other query suites do not cover:
  extension ray: the float64 brute force and tie rule of test_traversal_queries (tmin 0.01, tmax 1e5);
  mesh medium (SH/ClosestHit.slang:80-116, Q6): sd = -ln(u) / density from the exact draw against the distance to the shading position; a
      scatter keeps Depth, InMedium and the stale pdf, moves the origin to o + d sd, takes BxDF = medium colour and draws the
      Henyey-Greenstein direction (float64 restatement); the Beer case (anisotropy 1) draws nothing;
  surface: the shading step of b200pt_shade_query at the hit (test_shading_queries / test_nee_queries check it against the oracle and a
      float64 model) at the record's sampler state -- after the free-flight draw inside a medium -- for Depth >= 1, and for Depth 0 on
      surfaces that emit nothing (shade_query evaluates the emission MIS term at Depth 1); the sky and light shadow rays by float64 brute
      force: any hit in (1e-4, 1e6) from POS + 1e-5 N occludes the sky ray, the light ray from POS + 1e-2 l must reach the sampled triangle
      first (ties to the lower id); the successor's medium: the material's on entry (colour 1 in furnace mode), none on exit, else carried;
  miss: b200pt_miss_query's radiance (checked against its own model in test_nee_queries);
  epilogue (SH/RayGen.slang:92-128): payload.Emitted = (emitted + sky) + light, contribution x throughput, the luminance clamp unless the
      new Depth is 1 (always on a miss), throughput *= BxDF / PDF, roulette p = min(max(thr), 1) against the next draw, alive iff p >= u and
      the new Depth < MaxDepth, an invalid sample at PT_MAX_DEPTH + Depth; a finished path adds its radiance to its slot (stores it under
      STORE) unless a component is NaN or Inf, and leaves its sampler state under CARRY.  A miss ends the path after one roulette draw.
The epilogue is restated in fp32 (numpy float32 operations round as the GPU's __fadd_rn / __fmul_rn do); the three divisions are the
2-ulp approximate division of the build, so values are compared with VALUE_ULPS ulps of slack and the roulette is decided only when p and u
are further apart than that.  Geometric outputs (origins, directions) take the margins of the brute force.

The surface and miss terms come from the implementation's own shade_query / miss_query (and, for orc_bounce_query, the oracle's), not from
the float64 models of test_shading_queries / test_nee_queries: those hooks run the device functions k_shade_hit runs (surface_init,
hit_emission, the samplers), so a defect in that shared code is caught there, where the hooks are checked against the oracle and the float64
models, not here.  Depth 0 emission on an emitter (no MIS) is shade_query's EMITTED at a BSDF pdf of 1e18, where the MIS weight rounds to 1.
Some records get a roulette draw of exactly 1.0 with a clamped p (roulette_ones), the one input on which `!(p < u)` and `p > u` differ.
The oracle (orc_bounce_query: the loop body of trace_one_sample and the fold of render_thread, factored into path_segment and fold_sample)
runs the same records through the same model on its own shading; GPU and oracle may differ only where one of them is undecided.

A record is undecided when the hit, a shadow ray, the free-flight comparison or the roulette is within its margin; its outputs are skipped,
counted and bounded per case (UNDECIDED_MAX).  Decided records must match with alive, Depth, flags, hit ids, sampler states and slot ids
exact.  A value the model makes non-finite must be non-finite on the GPU.

Invariants with no model (no undecided records): each slot is either exactly one survivor or dead and the survivor count equals the number
alive; an alive path's slot is unchanged bit for bit; batches of 1, 31, 32, 33, 1000 and more paths than any persistent grid give the same
records; B200PT_FUSE=0 and the default, B200PT_CLASSES=0, big mode and the dynamic-fetch kernels give bit-identical records; a bounce_query
between two path_trace calls leaves the image unchanged; the work counters move by the counts the model derives.
"""
import math
import re
import zlib

import numpy as np
import pytest

import util
from util import orc
from test_shading_queries import REL, SQ, VALUE_ULPS, draw, pcg, state_for_draw
from test_traversal_queries import Ref

BQ_IN = dict(ORG=0, PDF=3, DIR=4, RNG=7, THR=8, DFLAGS=11, RAD=12, SLOT=15, MEDIUM=16, MEDIUM_G=20, SAMPLE=21, STRIDE=25)
BQ_OUT = dict(T=0, U=1, V=2, INST=3, PRIM=4, ALIVE=5, NEXT=6, SAMPLE=27, CARRY=31, STRIDE=32)
BQ_FLAGS = dict(STORE=2, CARRY=4)
PT_MAX_DEPTH = 1000000
UNDECIDED_MAX = 0.05
LUM = (np.float32(0.212671), np.float32(0.715160), np.float32(0.072169))
F32 = np.float32
ULP_REL = VALUE_ULPS * 2.0 ** -23                    # value slack of the fp32 epilogue (test_margin_is_tight)
ROULETTE_REL = 2 * VALUE_ULPS * 2.0 ** -23           # |p - u| / p below this: the roulette is undecided


def test_bounce_layout_matches_header():
    import vpt_b200
    hdr = open(f"{util.ROOT}/include/b200pt.h").read()
    d = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define B200PT_BQ_(\w+)\s+(\d+)", hdr)}
    assert {k[3:]: v for k, v in d.items() if k.startswith("IN_")} == BQ_IN == vpt_b200.BQ_IN
    assert {k[4:]: v for k, v in d.items() if k.startswith("OUT_")} == BQ_OUT == vpt_b200.BQ_OUT
    assert {k: d[k] for k in BQ_FLAGS} == BQ_FLAGS == dict(STORE=vpt_b200.BQ_STORE, CARRY=vpt_b200.BQ_CARRY)
    assert BQ_OUT["SAMPLE"] - BQ_OUT["NEXT"] == BQ_IN["SAMPLE"]
    ohdr = open(f"{util.ROOT}/oracle/pt_oracle.h").read()
    assert {m.group(1): int(m.group(2)) for m in re.finditer(r"#define ORC_BQ_(\w+)\s+(\d+)", ohdr)} == d


def test_oracle_max_luminance_edges():
    """What an infinite, NaN or zero MaxLuminance does (b200pt_set_config refuses them): MaxLuminance / max(lum, MaxLuminance) is inf / inf
    = NaN on every segment at Depth != 1 and 0 / 0 on every zero contribution, and the sample rejection then drops the whole path."""
    S = util.oracle_scene("cornell_box")
    img = {ml: S.render(util.oracle_config("cornell_box", MaxDepth=6, MaxLuminance=ml), 24, 16, 2, util.BASE_SEED)[0][..., :3]
           for ml in (1e30, math.inf, math.nan, 0.0, 0.01)}
    big, inf, nan, zero, small = (img[k] for k in (1e30, math.inf, math.nan, 0.0, 0.01))
    assert all(np.isfinite(v).all() for v in img.values())
    assert np.array_equal(inf, nan) and np.all(inf <= big) and inf.mean() < 0.05 * big.mean()   # only paths that end at Depth 1 remain
    assert (inf.max(-1) == 0).mean() > 0.5
    assert (small.max(-1) > 0).all() and (zero.max(-1) == 0).mean() > 0.3                      # zero-contribution segments discard paths


# ---------------------------------------------------------------- scenes and records
def _edit(sc, mats):
    sc = dict(sc); m = sc["materials"].copy()
    for i, kw in mats.items():
        for k, v in kw.items(): m[k][i % len(m)] = v
    sc["materials"] = m
    return sc


MEDIUM_MATS = {1: dict(Metallic=1.0, Roughness=0.3),
               2: dict(Metallic=0.0, Transmission=1.0, IOR=1.5, Roughness=0.05, MediumDensity=2.0, MediumAnisotropy=0.3, MediumColor=(0.9, 0.5, 0.3)),
               3: dict(Metallic=0.4, Transmission=0.3, Roughness=0.4)}
# name: (fixture, material edits, environment, config)
CASES = {
    "cornell": ("cornell_box", {}, {}, dict(MaxDepth=6)),
    "cornell_fuse0": ("cornell_box", {}, {"B200PT_FUSE": "0"}, dict(MaxDepth=6)),
    "classes": ("cornell_box", MEDIUM_MATS, {}, dict(MaxDepth=5, MaxLuminance=0.01)),
    "classes_general": ("cornell_box", MEDIUM_MATS, {"B200PT_CLASSES": "0"}, dict(MaxDepth=5, MaxLuminance=0.01)),
    "furnace_nonee": ("cornell_box", MEDIUM_MATS, {}, dict(MaxDepth=8, FurnaceTestMode=1, EnableSkyMIS=0, EnableMeshMIS=0)),
    "glass": ("cornell_box_glass", {}, {}, dict(MaxDepth=6, ShowEnvMapDirectly=1)),
    "glass_big": ("cornell_box_glass", {}, {"B200PT_SMEM_BIG": "1"}, dict(MaxDepth=6, ShowEnvMapDirectly=1)),
    "breakfast": ("breakfast_room", {}, {}, dict(MaxDepth=4, ShowEnvMapDirectly=0)),
}
PAIRS = [("cornell", "cornell_fuse0"), ("classes", "classes_general"), ("glass", "glass_big")]


def case_scene(name):
    fx, mats, _, _ = CASES[name]
    return _edit(util.scene_dict(fx), mats)


def _u(x):
    return np.asarray(x, np.uint32).view(np.float32)


def make_records(sc, n, seed, max_depth, cfg=None):
    """n live paths: origins in the scene's box, unit directions, the edge values of the module docstring; with cfg, some states whose
    roulette draw is exactly 1 (roulette_ones)"""
    rng = np.random.default_rng(seed)
    P = np.concatenate([sc["meshes"][m][0]["pos"] for _, m, _ in sc["instances"]])   # (object space is enough for a box around the scene)
    lo, hi = np.percentile(P, 2, 0), np.percentile(P, 98, 0)
    R = np.zeros((n, BQ_IN["STRIDE"]), np.float32)
    o = lo + (hi - lo) * (0.05 + 0.9 * rng.random((n, 3)))
    d = rng.normal(size=(n, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    R[:, 0:3] = o; R[:, 4:7] = d
    R[:, BQ_IN["PDF"]] = rng.choice([0.3, 1.0, 7.5, 1e-40, 0.0], n, p=[0.4, 0.3, 0.2, 0.05, 0.05])
    states = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32)
    R[:, BQ_IN["RNG"]] = _u(states)
    thr = rng.uniform(0.05, 1.0, (n, 3)).astype(np.float32)
    edge = rng.random(n)
    specials = [0.0, 3.0, 3e38, np.inf, np.nan]
    for j, s in enumerate(specials):
        sel = (edge > 0.80 + 0.03 * j) & (edge <= 0.83 + 0.03 * j)
        thr[sel, rng.integers(0, 3)] = s
    R[:, 8:11] = thr
    depth = np.array([0, 1, 2, max_depth - 1], np.uint32)[rng.integers(0, 4, n)]
    chan = rng.choice(4, n, p=[0.7, 0.1, 0.1, 0.1]).astype(np.uint32)
    inmed = rng.random(n) < 0.3
    R[:, BQ_IN["DFLAGS"]] = _u(depth | (chan << 27) | (inmed.astype(np.uint32) << 31))
    rad = rng.uniform(0, 2, (n, 3)).astype(np.float32)
    rad[rng.random(n) < 0.03, 0] = np.nan; rad[rng.random(n) < 0.03, 1] = np.inf
    R[:, 12:15] = rad
    R[:, 16:19] = rng.uniform(0.2, 1.0, (n, 3))
    R[:, 19] = rng.choice([0.05, 0.5, 3.0, -0.5], n, p=[0.3, 0.4, 0.2, 0.1])
    R[:, 20] = rng.choice([0.0, 0.9, -0.9, 1.0], n)
    R[:, 21:25] = rng.uniform(0, 1, (n, 4))
    # sampler states whose first draw is exactly 1 (a miss's roulette draw; inside a medium: u = 1 gives sd = -0, a scatter at the origin)
    k = np.nonzero(rng.random(n) < 0.05)[0]
    R[k, BQ_IN["RNG"]] = _u(np.full(len(k), state_for_draw(1.0, 0), np.uint32))
    if cfg is not None: roulette_ones(sc, R, cfg, rng)
    return R


def _oracle(sc, cfg):
    raw, env_pdf, alias = util.env_small()
    return orc.Scene(sc, env_pdf, alias, util.luts()), orc.default_config(**cfg)


def _draw_count(s0, s1, limit=64):
    for k in range(limit + 1):
        if s0 == s1: return k
        s0 = pcg(s0)
    return None


def roulette_ones(sc, R, cfg, rng, frac=0.1):
    """Give a share of the records a roulette draw of exactly 1.0 and a throughput of 8 (p clamps to 1, so `!(p < u)` keeps the path where
    `p > u` would end it).  A mesh-medium scatter makes three draws before the roulette; a surface hit makes as many as its shading step,
    counted on the oracle's shade_query at the hit and kept only when the new state's shading step makes the same number."""
    S, oc = _oracle(sc, cfg)
    pick = np.nonzero(rng.random(len(R)) < frac)[0]
    d = R[pick, 4:7] / np.linalg.norm(R[pick, 4:7], axis=1, keepdims=True)
    t, prim, inst, uv = S.trace_closest(R[pick, 0:3], d.astype(np.float32), 0.01, 1e5)
    df = R[pick, BQ_IN["DFLAGS"]].view(np.uint32)
    scatter = (df >> 31 != 0) & (R[pick, BQ_IN["MEDIUM_G"]] != 1.0)
    for i in pick[scatter & (t > 0)]:
        R[i, BQ_IN["RNG"]] = _u(state_for_draw(1.0, 3)); R[i, 8:11] = 8.0
    sel = ~scatter & (t > 0)
    rows, s0 = pick[sel], R[pick[sel], BQ_IN["RNG"]].view(np.uint32).copy()
    if not len(rows): return
    args = (inst[sel], prim[sel], uv[sel], R[rows, 4:7], R[rows, 0:3], R[rows, BQ_IN["PDF"]])
    k0 = [_draw_count(int(a), int(b)) for a, b in zip(s0, S.shade_query(oc, *args, s0, None)[:, SQ["RNG"]].view(np.uint32))]
    s1 = np.array([state_for_draw(1.0, k) if k else 0 for k in k0], np.uint32)
    k1 = [_draw_count(int(a), int(b)) for a, b in zip(s1, S.shade_query(oc, *args, s1, None)[:, SQ["RNG"]].view(np.uint32))]
    for i, a, b, st in zip(rows, k0, k1, s1):
        if a and a == b: R[i, BQ_IN["RNG"]] = _u(st); R[i, 8:11] = 8.0


# ---------------------------------------------------------------- model
def _draws_from(state, k):
    out = []
    for _ in range(k):
        state, x = draw(state)
        out.append(x)
    return state, out


def _f(x):
    return F32(x)


def hg_dir(d, g, rx, ry):
    """sample_henyey_greenstein (SH/Sampler.slang) in float64"""
    if abs(g) < 1e-5: c = 2 * rx - 1
    else:
        sq = (1 - g * g) / (1 - g + 2 * g * rx); c = (1 + g * g - sq * sq) / (2 * g)
    phi = 2 * float(np.float32(3.1415926535897)) * ry
    s = math.sqrt(max(0.0, 1 - c * c))
    nd = np.array([s * math.cos(phi), s * math.sin(phi), c])
    up = np.array([0, 1.0, 0]) if abs(d[1]) < 0.9999999 else np.array([0, 0, 1.0])
    t = np.cross(up, d); t /= np.linalg.norm(t)
    b = np.cross(d, t)
    r = t * nd[0] + b * nd[1] + d * nd[2]
    return r / np.linalg.norm(r)


def epilogue(cfg, emitted, thr3, r3, b4, new_dflags, state, miss):
    """SH/RayGen.slang:92-113 in fp32: (alive, throughput, radiance, state after the roulette draw, roulette margin |p - u| / p)"""
    emitted = np.asarray(emitted, np.float32); thr3 = np.asarray(thr3, np.float32)[:3]; r3 = np.asarray(r3, np.float32)[:3]
    new_depth = new_dflags & 0x07FFFFFF
    ML = F32(cfg["MaxLuminance"])
    with np.errstate(all="ignore"):
        c = emitted * thr3
        if miss or new_depth != 1:
            lum = F32(F32(c[2] * LUM[2]) + F32(F32(c[0] * LUM[0]) + F32(c[1] * LUM[1])))   # (the GPU's two FMAs: within the value slack)
            c = c * F32(ML / np.fmax(lum, ML))
        rad = r3 + c
        state, (u,) = _draws_from(state, 1)
        if miss: return False, None, rad, state, math.inf
        b4 = np.asarray(b4, np.float32)
        thr = thr3 * (b4[:3] / b4[3])
        pmax = F32(np.fmax(thr[0], np.fmax(thr[1], thr[2])))
        p = float(np.fmin(pmax, F32(1.0)))
        alive = not (p < u)
        if alive: thr = thr / F32(p)
        margin = math.inf if not (pmax < 1.0) else abs(p - u) / max(p, 1e-30)    # a clamped p (or NaN max: p = 1) is exact
    return alive and new_depth < cfg["MaxDepth"], thr, rad, state, margin


class Model:
    def __init__(self, name, T):
        self.name, self.T = name, T
        self.sc = case_scene(name)
        fx, mats, env, cfg = CASES[name]
        self.cfg = dict(EnableSkyMIS=1, EnableMeshMIS=1, FurnaceTestMode=0, MaxLuminance=500.0); self.cfg.update(cfg)
        self.ref = Ref(self.sc)
        self.mat_of = np.array([m for _, _, m in self.sc["instances"]])

    def closest(self, o, d, tmin, tmax):
        return self.ref.classify(o[None], d[None], np.array([tmin]), np.array([tmax]))[0]

    def occluded_sky(self, o, d):
        """True / False, None when an occluder lies within the margin of (1e-4, 1e6)"""
        cand, t, et, req, adm, *_ = self.closest(o, d, 1e-4, 1e6)
        return True if req.any() else (None if adm.any() else False)

    def visible_light(self, o, d, target):
        cand, t, et, req, adm, *_ = self.closest(o, d, 1e-4, 1e6)
        j = np.nonzero(cand == target)[0]
        if not len(j): return False
        j = j[0]
        if not req[j]: return None if adm[j] else False
        other = cand != target
        if (req & other & (t + et < t[j] - et[j])).any(): return False
        if (adm & other & (t <= t[j] + et[j] + et)).any(): return None
        return True

    def run(self, R, got, store, carry):
        """per record: None (undecided) or the list of failures; and the counts of the decided records (misses, surface hits, mesh-medium
        scatters, NEE requests)"""
        T, cfg, n = self.T, self.cfg, len(R)
        o, d = R[:, 0:3].astype(np.float64), R[:, 4:7].astype(np.float64)
        dflags = R[:, BQ_IN["DFLAGS"]].view(np.uint32)
        states = R[:, BQ_IN["RNG"]].view(np.uint32)
        inst, prim = got[:, BQ_OUT["INST"]].view(np.uint32), got[:, BQ_OUT["PRIM"]].view(np.uint32)
        gid = self.ref.gid(prim, inst)
        # the extension ray, against the brute force
        dn = d / np.linalg.norm(d, axis=1, keepdims=True)
        cls = self.ref.classify(o, dn, np.full(n, 0.01), np.full(n, 1e5))
        verdict, ctr = [None] * n, dict(misses=0, surface_hits=0, medium_events=0, shadow_rays=0)
        misses = np.nonzero(gid < 0)[0]
        miss_rgb = T.miss_query(R[misses, 4:7], dflags[misses] & 0x07FFFFFF, R[misses, BQ_IN["PDF"]])[:, :3] if len(misses) else None
        miss_row = {int(i): k for k, i in enumerate(misses)}
        # surface records: the shading step at the hit, at the state after the free-flight draw inside a medium
        hits = np.nonzero(gid >= 0)[0]
        sq_state = states.copy()
        ff = {}
        for i in hits:
            if dflags[i] >> 31 and R[i, BQ_IN["MEDIUM_G"]] != 1.0:
                s, (u0,) = _draws_from(int(states[i]), 1)
                ff[int(i)] = (s, u0); sq_state[i] = s
        S = T.shade_query(inst[hits], prim[hits], got[hits, 1:3], R[hits, 4:7], R[hits, 0:3], R[hits, BQ_IN["PDF"]], sq_state[hits]) if len(hits) else None
        hit_row = {int(i): k for k, i in enumerate(hits)}
        # Depth 0 on an emitter: emission without MIS.  shade_query weights it for Depth 1; at a BSDF pdf of 1e18 that weight rounds to 1.
        em_mat = np.array([max(self.sc["materials"][self.mat_of[j]]["EmissiveColor"]) > 0 for j in inst[hits]], bool) if len(hits) else np.zeros(0, bool)
        z = hits[em_mat & ((dflags[hits] & 0x07FFFFFF) == 0)]
        E0 = {int(i): r[SQ["EMITTED"]:SQ["EMITTED"] + 3] for i, r in zip(z, T.shade_query(inst[z], prim[z], got[z, 1:3], R[z, 4:7], R[z, 0:3], 1e18, sq_state[z]))} if len(z) else {}
        for i in range(n):
            cand, t, et, req, adm, u_, v_, eu, ev = cls[i]
            fails = []
            g = gid[i]
            best = t[req].min() if req.any() else np.inf
            if (adm & ~req & (t <= best + et)).any(): continue                     # the hit itself is undecided
            if g < 0:
                if req.any(): verdict[i] = ["hit missed"]; continue
            else:
                j = np.nonzero(cand == g)[0]
                if not len(j) or not req[j[0]] or (t[req] + et[req] < t[j[0]] - et[j[0]]).any(): verdict[i] = [f"wrong hit {g}"]; continue
            r4 = R[i, 12:16].copy(); r4[3] = R[i, BQ_IN["SLOT"]]
            thr4 = R[i, 8:12]
            depth = int(dflags[i] & 0x07FFFFFF); chan_bits = int(dflags[i] & (3 << 27)); inmed = bool(dflags[i] >> 31)
            slot0 = R[i, 21:25]
            if g < 0:
                ctr["misses"] += 1
                alive, thr, rad, st, _ = epilogue(cfg, miss_rgb[miss_row[i]], thr4, r4, None, int(dflags[i]), int(states[i]), True)
                verdict[i] = self._fold(got[i], fails, False, rad, chan_bits, st, slot0, store, carry)
                continue
            ctr["surface_hits"] += 1
            k = hit_row[i]; q = S[k]
            pos = q[SQ["POS"]:SQ["POS"] + 3].astype(np.float64)
            if inmed and i in ff:
                s_after, u0 = ff[i]
                dens = float(R[i, 19])
                with np.errstate(all="ignore"):
                    sd = -math.log(u0) / dens if u0 > 0 else math.inf
                dist = float(np.linalg.norm(o[i] - pos))
                if abs(sd - dist) <= 16 * REL * max(dist, 1e-30) + 1e-6: continue             # free flight within the margin
                if sd < dist:
                    ctr["medium_events"] += 1
                    s2, (rx, ry) = _draws_from(s_after, 2)
                    med = R[i, 16:20]
                    b4 = np.array([med[0], med[1], med[2], R[i, BQ_IN["PDF"]]], np.float32)
                    alive, thr, rad, st, rm = epilogue(cfg, np.zeros(3, np.float32), thr4, r4, b4, int(dflags[i]), s2, False)
                    if rm <= ROULETTE_REL: continue
                    nd = hg_dir(R[i, 4:7].astype(np.float64), float(R[i, 20]), rx, ry)
                    no = o[i] + d[i] * sd
                    verdict[i] = self._fold(got[i], fails, alive, rad, chan_bits, st, slot0, store, carry)
                    if alive:
                        self._next(got[i], fails, no, float(R[i, BQ_IN["PDF"]]), nd, st, thr, int(dflags[i]), rad, i, med=R[i, 16:21],
                                   geo_tol=1e-4 * (1 + abs(sd)))
                    continue
            # surface
            m = self.sc["materials"][self.mat_of[inst[i]]]
            emissive = max(m["EmissiveColor"]) > 0
            e = (E0[i] if i in E0 else q[SQ["EMITTED"]:SQ["EMITTED"] + 3]).astype(np.float32)
            N = q[SQ["N"]:SQ["N"] + 3].astype(np.float32)
            und = False
            if cfg["EnableSkyMIS"] and q[SQ["SKY_LV"] + 3] > 0 and q[SQ["SKY_EVAL"] + 3] > 0:
                ctr["shadow_rays"] += 1
                so = (q[SQ["POS"]:SQ["POS"] + 3] + N * F32(1e-5)).astype(np.float32)
                occ = self.occluded_sky(so.astype(np.float64), q[SQ["SKY_W"]:SQ["SKY_W"] + 3].astype(np.float64))
                if occ is None: und = True
                elif not occ: e = e + q[SQ["SKY_C"]:SQ["SKY_C"] + 3]
            if cfg["EnableMeshMIS"] and not emissive and q[SQ["LIGHT_LV"] + 3] > 0 and q[SQ["LIGHT_EVAL"] + 3] > 0:
                ctr["shadow_rays"] += 1
                lw = q[SQ["LIGHT_W"]:SQ["LIGHT_W"] + 3]
                lo_ = (q[SQ["POS"]:SQ["POS"] + 3] + lw * F32(1e-2)).astype(np.float32)
                vis = self.visible_light(lo_.astype(np.float64), lw.astype(np.float64), int(q[SQ["LIGHT_GID"]:SQ["LIGHT_GID"] + 1].view(np.uint32)[0]))
                if vis is None: und = True
                elif vis: e = e + q[SQ["LIGHT_C"]:SQ["LIGHT_C"] + 3]
            if und: continue
            b4 = q[SQ["SAMPLE"]:SQ["SAMPLE"] + 4]
            invalid = not (b4[3] > 0)
            new_depth = PT_MAX_DEPTH + depth if invalid else depth + 1
            refr, entered, inside = q[SQ["REFRACTED"]] != 0, q[SQ["ENTERED"]] != 0, q[SQ["INSIDE"]] != 0
            new_in = False if (refr and inside) else (True if refr else inmed)
            nf = new_depth | chan_bits | (int(new_in) << 31)
            st0 = int(q[SQ["RNG"]:SQ["RNG"] + 1].view(np.uint32)[0])
            alive, thr, rad, st, rm = epilogue(cfg, e, thr4, r4, b4, nf, st0, False)
            if rm <= ROULETTE_REL: continue
            verdict[i] = self._fold(got[i], fails, alive, rad, chan_bits, st, slot0, store, carry)
            if alive:
                off = -1e-3 if refr else 1e-3
                no = pos + N.astype(np.float64) * off
                if entered:
                    mc = (1.0, 1.0, 1.0) if cfg.get("FurnaceTestMode") else tuple(m["MediumColor"])
                    med = np.array(list(mc) + [m["MediumDensity"], m["MediumAnisotropy"]], np.float32)
                else: med = R[i, 16:21]
                self._next(got[i], fails, no, float(b4[3]), q[SQ["SCATTER"]:SQ["SCATTER"] + 3].astype(np.float64), st, thr, nf, rad, i,
                           med=med if new_in else None, geo_tol=1e-5 * (1 + np.abs(pos).max()))
        return verdict, ctr

    @staticmethod
    def _close(a, b, tol_rel, tol_abs=0.0):
        a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
        fin = np.isfinite(b)
        if not np.array_equal(np.isfinite(a)[fin], fin[fin]): return False
        if not (~np.isfinite(a[~fin])).all(): return False                               # model non-finite -> GPU non-finite
        return bool(np.all(np.abs(a[fin] - b[fin]) <= tol_rel * np.abs(b[fin]) + tol_abs + 1e-37))

    def _fold(self, g, fails, alive, rad, chan_bits, st, slot0, store, carry):
        if bool(g[BQ_OUT["ALIVE"]]) != alive: fails.append(f"alive {g[BQ_OUT['ALIVE']]} != {alive}"); return fails
        slot = g[BQ_OUT["SAMPLE"]:BQ_OUT["SAMPLE"] + 4]
        c = g[BQ_OUT["CARRY"]:BQ_OUT["CARRY"] + 1].view(np.uint32)[0]
        if alive:
            if not np.array_equal(slot.view(np.uint32), slot0.view(np.uint32)): fails.append("alive path's slot changed")
            if c != 0: fails.append("alive path carried a state")
            return fails
        base = np.zeros(4, np.float32) if store else slot0.copy()
        want = base.copy()
        if np.isfinite(rad).all():
            ch = (chan_bits >> 27) - 1
            with np.errstate(all="ignore"):
                if ch < 0: want[:3] = base[:3] + rad
                else: want[ch] = base[ch] + rad[ch]
        if not self._close(slot, want, ULP_REL, ULP_REL * float(np.abs(base).max())): fails.append(f"slot {slot} != {want}")
        if c != (st if carry else 0): fails.append(f"carry {c} != {st if carry else 0}")
        return fails

    def _next(self, g, fails, no, pdf, nd, st, thr, nf, rad, slot, med, geo_tol):
        s = g[BQ_OUT["NEXT"]:BQ_OUT["NEXT"] + BQ_IN["SAMPLE"]]
        u = s.view(np.uint32)
        if not self._close(s[0:3], no, 0.0, geo_tol): fails.append(f"origin {s[0:3]} != {no}")
        if not np.array_equal(np.float32(pdf).view(np.uint32), u[3]): fails.append(f"pdf {s[3]} != {pdf}")
        if not self._close(s[4:7], nd, 0.0, 2e-4): fails.append(f"direction {s[4:7]} != {nd}")
        if u[7] != st: fails.append(f"state {u[7]} != {st}")
        if not self._close(s[8:11], thr, ULP_REL): fails.append(f"throughput {s[8:11]} != {thr}")
        if u[11] != nf: fails.append(f"dflags {u[11]:#x} != {nf:#x}")
        if not self._close(s[12:15], rad, ULP_REL, 1e-30): fails.append(f"radiance {s[12:15]} != {rad}")
        if u[15] != slot: fails.append(f"slot id {u[15]} != {slot}")
        if med is not None and not np.array_equal(s[16:21].view(np.uint32), np.asarray(med, np.float32).view(np.uint32)):
            fails.append(f"medium {s[16:21]} != {med}")


# ---------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def pt():
    import torch
    if not torch.cuda.is_available(): pytest.skip("no CUDA device")
    import vpt_b200
    return vpt_b200


def tracer(name, monkeypatch, **over):
    fx, mats, env, cfg = CASES[name]
    for k in ("B200PT_FUSE", "B200PT_CLASSES", "B200PT_SMEM_BIG"): monkeypatch.delenv(k, raising=False)
    for k, v in env.items(): monkeypatch.setenv(k, v)
    return util.product_tracer(fx, 8, 8, scene=case_scene(name), **dict(cfg, **over))


def _records(name, n=400, seed=0, ones=True):
    cfg = CASES[name][3]
    return make_records(case_scene(name), n, seed, cfg["MaxDepth"], _model_cfg(cfg) if ones else None)


def _model_cfg(cfg):
    c = dict(EnableSkyMIS=1, EnableMeshMIS=1, FurnaceTestMode=0, MaxLuminance=500.0); c.update(cfg)
    return c


class OracleShading:
    """the oracle's shade_query / miss_query under the case's config, in the product's call signature"""
    def __init__(self, S, oc): self.S, self.oc = S, oc
    def shade_query(self, *a): return self.S.shade_query(self.oc, *a, None)
    def miss_query(self, *a): return self.S.miss_query(self.oc, *a)


def check(name, T, R, got, store, carry):
    verdict, ctr = Model(name, T).run(R, got, store, carry)
    und = np.array([v is None for v in verdict])
    return verdict, ctr, und, [(i, v) for i, v in enumerate(verdict) if v]


@pytest.mark.parametrize("name", [c for c in CASES if not CASES[c][2]])
def test_oracle_matches_float64_model(name):
    """CPU only: orc_bounce_query against the model, on the oracle's own shading; validates the model and the margins"""
    S, oc = _oracle(case_scene(name), _model_cfg(CASES[name][3]))
    for store in (False, True):
        R = _records(name, seed=zlib.crc32(f"{name} {store}".encode()))
        got, m = S.bounce_query(oc, R, store=store, carry=store)
        invariants(R, got, m)
        verdict, ctr, und, fails = check(name, OracleShading(S, oc), R, got, store, store)
        print(f"oracle {name} store={store}: alive {m}, undecided share {und.mean():.3f}, counts {ctr}")
        assert not fails, fails[:8]
        assert und.mean() <= UNDECIDED_MAX, und.mean()


def invariants(R, got, m):
    alive = got[:, BQ_OUT["ALIVE"]]
    assert set(np.unique(alive)) <= {0.0, 1.0}, "a slot was written by two survivors"
    assert int(alive.sum()) == m
    a = alive == 1
    assert np.array_equal(got[a, BQ_OUT["SAMPLE"]:BQ_OUT["SAMPLE"] + 4].view(np.uint32), R[a, 21:25].view(np.uint32))
    assert np.array_equal(got[a, BQ_OUT["NEXT"] + BQ_IN["SLOT"]].view(np.uint32), np.nonzero(a)[0].astype(np.uint32))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("store,carry", [(False, False), (True, True)])
def test_gpu_bounce_matches_model(pt, name, store, carry, monkeypatch):
    T = tracer(name, monkeypatch)
    R = _records(name, seed=zlib.crc32(f"{name} {store}".encode()))
    c0 = T.counters()
    got, m = T.bounce_query(R, store=store, carry=carry)
    c1 = T.counters()
    invariants(R, got, m)
    verdict, ctr, und, fails = check(name, T, R, got, store, carry)
    # the oracle on the same records, checked by the same model on its own shading; GPU and oracle may differ only where one is undecided
    S, oc = _oracle(case_scene(name), _model_cfg(CASES[name][3]))
    ref, _ = S.bounce_query(oc, R, store=store, carry=carry)
    _, _, und_o, fails_o = check(name, OracleShading(S, oc), R, ref, store, carry)
    both = ~und & ~und_o
    agree = np.array_equal(got[both, BQ_OUT["ALIVE"]], ref[both, BQ_OUT["ALIVE"]]) and all(
        np.array_equal(got[both, BQ_OUT[f]:BQ_OUT[f] + 1].view(np.uint32), ref[both, BQ_OUT[f]:BQ_OUT[f] + 1].view(np.uint32)) for f in ("INST", "PRIM", "CARRY")) and all(
        np.array_equal(got[both, BQ_OUT["NEXT"] + BQ_IN[f]].view(np.uint32), ref[both, BQ_OUT["NEXT"] + BQ_IN[f]].view(np.uint32)) for f in ("RNG", "DFLAGS", "SLOT"))
    print(f"{name} store={store}: {len(R)} records, alive {m}, undecided share {und.mean():.3f} (oracle {und_o.mean():.3f}), counters {ctr}")
    assert not fails, fails[:8]
    assert not fails_o, fails_o[:8]
    assert agree
    assert und.mean() <= UNDECIDED_MAX, und.mean()
    assert c1["extend_rays"] - c0["extend_rays"] == len(R)
    assert c1["shade_invocations"] - c0["shade_invocations"] == len(R)
    assert c1["paths"] == c0["paths"]
    # the decided records bound the counts (an undecided record adds at most one miss, hit or scatter and two NEE requests); mesh-medium
    # scatters count as surface hits as well as medium events
    nu = int(und.sum())
    for k, per in (("misses", 1), ("surface_hits", 1), ("medium_events", 1), ("shadow_rays", 2)):
        assert ctr[k] <= c1[k] - c0[k] <= ctr[k] + per * nu, (k, c1[k] - c0[k], ctr[k], nu)
    assert c1["surface_hits"] - c0["surface_hits"] == len(R) - (c1["misses"] - c0["misses"])


@pytest.mark.gpu
@pytest.mark.parametrize("a,b", PAIRS)
def test_gpu_pipelines_give_identical_records(pt, a, b, monkeypatch):
    R = _records(a, n=1000, seed=7)
    got = [tracer(x, monkeypatch).bounce_query(R, store=True, carry=True) for x in (a, b)]
    assert got[0][1] == got[1][1]
    assert np.array_equal(got[0][0].view(np.uint32), got[1][0].view(np.uint32)), np.nonzero((got[0][0] != got[1][0]).any(1))[0][:10]


@pytest.mark.gpu
def test_gpu_batches_give_identical_records(pt, monkeypatch):
    """1, 31, 32, 33, 1000 and more paths than any persistent grid holds: the records do not depend on the batch"""
    T = tracer("classes", monkeypatch)
    big = 300_000
    R = _records("classes", n=big, seed=11)
    ref, m = T.bounce_query(R, carry=True)
    invariants(R, ref, m)
    for n in (1, 31, 32, 33, 1000):
        got, mm = T.bounce_query(R[:n], carry=True)
        invariants(R[:n], got, mm)
        assert np.array_equal(got.view(np.uint32), ref[:n].view(np.uint32)), n
    assert T.bounce_query(R[:0])[1] == 0


@pytest.mark.gpu
def test_gpu_bounce_query_leaves_the_image(pt, monkeypatch):
    T = tracer("classes", monkeypatch); U = tracer("classes", monkeypatch)
    T.resize(32, 24); U.resize(32, 24)
    T.path_trace(2, util.BASE_SEED); U.path_trace(2, util.BASE_SEED)
    U.bounce_query(_records("classes", n=5000, seed=3), store=True, carry=True)
    T.path_trace(2, util.BASE_SEED + 9); U.path_trace(2, util.BASE_SEED + 9)
    a, b = T.get_hdr(), U.get_hdr()
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert T.samples_accumulated() == U.samples_accumulated()


@pytest.mark.gpu
def test_gpu_bounce_query_refusals(pt, monkeypatch):
    T = tracer("cornell", monkeypatch)
    R = _records("cornell", n=8)
    def refused(X, **kw):
        with pytest.raises(pt.B200ptError, match=str(pt.ERR_WRONG_ARGUMENTS)): T.bounce_query(X, **kw)
    for field, val in ((0, np.nan), (1, np.inf), (4, np.nan), (5, -np.inf)):
        X = R.copy(); X[3, field] = val; refused(X)
    X = R.copy(); X[2, 4:7] = 0; refused(X)
    X = R.copy(); X[1, BQ_IN["DFLAGS"]] = _u(CASES["cornell"][3]["MaxDepth"]); refused(X)
    for bit in (29, 30):
        X = R.copy(); X[0, BQ_IN["DFLAGS"]] = _u(1 | (1 << bit)); refused(X)
    L, C = pt.lib(), __import__("ctypes")
    out = np.zeros((8, BQ_OUT["STRIDE"]), np.float32); m = C.c_uint32()
    assert L.b200pt_bounce_query(T.h, 8, R.ctypes.data, 1, out.ctypes.data, C.byref(m)) == pt.ERR_WRONG_ARGUMENTS   # WAVE_IMPLIED is not a hook flag
    assert L.b200pt_bounce_query(T.h, 8, R.ctypes.data, 8, out.ctypes.data, C.byref(m)) == pt.ERR_WRONG_ARGUMENTS
    assert L.b200pt_bounce_query(T.h, 0, None, 0, None, C.byref(m)) == 0 and m.value == 0
    V = tracer("cornell", monkeypatch)
    V.add_volume(CornerMin=(-1.0, -1.0, -1.0), CornerMax=(1.0, 1.0, 1.0), Density=0.5)
    with pytest.raises(pt.B200ptError, match=str(pt.ERR_WRONG_ARGUMENTS)): V.bounce_query(R)
    E = pt.PathTracer(0)
    with pytest.raises(pt.B200ptError, match=str(pt.ERR_NO_SCENE)): E.bounce_query(R)


@pytest.mark.gpu
def test_gpu_counters_before_the_first_render(pt, monkeypatch):
    """counters() on a fresh handle reads the timing events before any render recorded them; that failed query must not fail the next call"""
    T = tracer("cornell", monkeypatch)
    assert T.counters()["ms_total"] == 0.0
    T.path_trace(1, util.BASE_SEED)
    T.bounce_query(_records("cornell", n=4))


@pytest.mark.gpu
def test_config_refuses_bad_max_luminance(pt, monkeypatch):
    T = tracer("cornell", monkeypatch)
    for ml in (math.nan, math.inf, -math.inf, 0.0, -1.0):
        c = pt.default_config(); c.MaxLuminance = ml
        with pytest.raises(pt.B200ptError, match=str(pt.ERR_WRONG_ARGUMENTS)): T.set_config(c)
    for ml in (1e-30, 0.01, 3e38):
        c = pt.default_config(); c.MaxLuminance = ml; T.set_config(c)


@pytest.mark.gpu
def test_margin_is_tight(pt, monkeypatch):
    """K / 10 (VALUE_ULPS / 10 here): the fp32 epilogue's value slack is needed by some GPU answer.  Only the value slack shrinks (the
    roulette margin is ROULETTE_REL), and the rejection must be of a value, not of alive, a state or an id."""
    global ULP_REL
    T = tracer("classes", monkeypatch)
    R = _records("classes", seed=5)
    got, _ = T.bounce_query(R)
    keep = ULP_REL
    try:
        ULP_REL = keep / 10
        verdict, _ = Model("classes", T).run(R, got, False, False)
    finally:
        ULP_REL = keep
    values = ("slot ", "throughput ", "radiance ", "origin ", "direction ")
    assert any(f.startswith(values) for v in verdict if v for f in v), "K / 10 rejects no value"
