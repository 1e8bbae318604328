"""Next-event estimation record by record: the sky and light draws of b200pt_shade_query, their NEE terms c, the emission MIS term of a hit
on a light, and the miss shading of b200pt_miss_query, against the CPU oracle (orc_shade_query, orc_miss_query) and a float64 model, on inputs
no shipped scene has: odd-sized, one-row, one-column, black, half-black, constant and 4096 x 2048 environment maps under five sky rotations,
several emissive meshes (1 to 300 triangles, scaled, mirrored and sheared instances, textured, with a zero channel, with a zero-area
triangle), shading points on a light's plane, behind it, 1e-3 from it and 1e4 away, and sampler states on every draw threshold.

Model (numpy float64, restating the Slang with its quirks):
  sky NEE (SH/Sampler.slang:287-346): the alias pick on the same table the renderer builds (test_host_api checks it bit for bit), the texel
      jitter with (xy - imp) / (1 - imp) in the alias branch, cos(theta0) and cos(theta0 + stepTheta) at the fp32 theta0 the renderer takes,
      acos / sin, the azimuth-then-altitude rotation, the bilinear REPEAT lookup with its alpha (the pdf), the intensity applied twice (Q7);
  light NEE (:349-422): uniform mesh then uniform triangle (Q16), the sqrt barycentric warp on the fp32 instance transform, the emissive
      texel at the interpolated uv, d2 / (count * tc * area * |n_geo . l|);
  the emission MIS term of a hit (SH/ClosestHit.slang:265-317, shading normal, bias max), the power heuristic and c;
  miss shading (SH/Miss.slang:8-76): inverse rotation, direction_to_uv, ShowEnvMapDirectly at depth 0, furnace mode, the MIS weight.
The surface frame, the material and the BSDF come from test_shading_queries.model_hit, whose draws follow the NEE draws.

Margins follow test_shading_queries: every input (and every draw) moved by a relative 2^-23 in +/- pairs, margin = K * spread + VALUE_ULPS
ulps.  A record is undecided when a perturbation flips the texel pick (xx * size), xy < imp, the mesh or triangle pick, lv.w > 0, e.PDF > 0,
any branch of the surface model, or the finiteness of an output; undecided records are counted and bounded per case.  An output the model
computes as inf / NaN must be non-finite in the implementation too.

Pair invariants (GPU): a sky draw seen from the BSDF side (miss_query along the drawn direction) must return the pdf of the draw and its
radiance without Q7's second intensity, and the two MIS weights of that path must sum to one; a light draw traced to its triangle and shaded
there (shade_query at the hit, pay_pdf = the BSDF pdf of the draw) must give the light pdf lv.w * |NG . l| / |N . l| (the reference's NEE
takes the geometric normal, its emission term the shading normal), floored by the bias.
"""
import functools
import itertools
import math

import numpy as np
import pytest

import util
from util import gltf_ref, orc
from test_shading_queries import (K, NPERT, REL, SQ, TEX, TEX_NAMES, VALUE_ULPS, _draws, _gpu_vs_oracle, _mat, _n, _perturbations, _quad_mesh,
                                  M32, model_hit, model_inputs, pcg, pcg_inv, records, scene_for, state_for_draw, tex_u8)

MQ = dict(RGB=0, PDF=3, STRIDE=4)
UNDECIDED_MAX = 0.35
PT_PI = float(np.float32(3.1415926535897))
PT_1_OVER_PI = float(np.float32(0.3183098861837))
NEE_FIELDS = dict(POS=3, EMITTED=3, SKY_W=3, SKY_LV=4, SKY_L=3, SKY_EVAL=4, SKY_C=3, LIGHT_W=3, LIGHT_LV=4, LIGHT_L=3, LIGHT_EVAL=4, LIGHT_C=3)
ORACLE_FIELDS = tuple(NEE_FIELDS)


# ---------------------------------------------------------------- environment maps
def _env_raw(name):
    if name == "synthetic": return gltf_ref.synthetic_env(512, 256, 3)
    if name == "bench": return gltf_ref.synthetic_env(4096, 2048, seed=3, sun=150000.0)     # the map bench.py renders with
    if name in ("37x19", "37x1", "1x19"):
        w, h = map(int, name.split("x"))
        return gltf_ref.synthetic_env(w, h, 5 + w + h)
    out = np.ones((19, 37, 4), np.float32)
    if name == "hot00":                                                     # one hot texel on the u seam, in the pole row
        out[..., :3] = 0.0; out[0, 0, :3] = (50.0, 40.0, 30.0)
    elif name == "halfblack":
        out[..., :3] = gltf_ref.synthetic_env(37, 19, 9)[..., :3]; out[19 // 2:, :, :3] = 0.0
    elif name == "constant": out[..., :3] = 0.7
    return out


ENV_NAMES = ("synthetic", "37x19", "37x1", "1x19", "hot00", "halfblack", "constant", "bench")


@functools.lru_cache(maxsize=None)
def env(name):
    """(raw rgba given to the renderer, rgba with the pdf in alpha, alias table), the last two built by the oracle"""
    raw = _env_raw(name)
    env_pdf, alias, _ = orc.build_env_alias(raw)
    return raw, env_pdf, alias


# ---------------------------------------------------------------- float64 model
def _f(x):
    return np.asarray(x, np.float64)


def ph(a, b):
    with np.errstate(all="ignore"): return _f(a) * a / (_f(a) * a + _f(b) * b)


def rot(v, axis, c, s):                                                     # SH/RTCommon.slang:37-45
    n = np.array(axis, np.float64)
    return (v * c + np.cross(n, v) * s) + n * (n @ v) * (1 - c)


def env_lookup(t, u, v, jit):
    """bilinear REPEAT of an rgba32f map [H, W, 4] (pdf in alpha); u, v and the texel coordinates are fp32 in the implementations"""
    H, W = t.shape[:2]
    with np.errstate(all="ignore"):
        u, v = jit("u", u), jit("v", v)
        x, y = jit("x", u * W - 0.5), jit("y", v * H - 0.5)
    if not (np.isfinite(x) and np.isfinite(y)): return np.full(4, np.nan)
    fx, fy = math.floor(x), math.floor(y); ax, ay = x - fx, y - fy
    x0, x1, y0, y1 = fx % W, (fx + 1) % W, fy % H, (fy + 1) % H
    p = lambda yy, xx: t[yy, xx].astype(np.float64)
    a = p(y0, x0) + ax * (p(y0, x1) - p(y0, x0)); b = p(y1, x0) + ax * (p(y1, x1) - p(y1, x0))
    return a + ay * (b - a)


def _angles(cfg, jit):
    az = jit("az", cfg["SkyRotationAzimuth"] / 180.0 * math.pi); al = jit("al", cfg["SkyRotationAltitude"] / 180.0 * math.pi)
    return math.cos(az), math.sin(az), math.cos(al), math.sin(al)


def model_sky(draws, ex, envd, cfg, br, jit):
    """sample_env (SH/Sampler.slang:287-346): world direction and (radiance * intensity, pdf); the hit applies the intensity once more (Q7).
    ex(): the exact fp32 value of the draw just made.  The picks compare exact fp32 values (the texel index is one correctly rounded product),
    so they are emulated exactly; the perturbed draws only feed the arithmetic after them."""
    _, tex, alias = envd
    H, W = tex.shape[:2]
    size = W * H
    _ = next(draws); idx = min(int(np.float32(ex()) * np.float32(size)), size - 1)
    br.append(("texel", idx))
    imp = alias["Importance"][idx]
    xy = next(draws); pick = bool(np.float32(ex()) < imp)
    imp = float(imp)
    br.append(("imp", pick))
    xz = next(draws)
    with np.errstate(all="ignore"):
        e, xy = (idx, np.float64(xy) / imp) if pick else (int(alias["Alias"][idx]), (np.float64(xy) - imp) / (np.float64(1.0) - imp))
    px, py = e % W, e // W
    u = jit("u", (px + xy) / W)
    phi = jit("phi", u * (2 * PT_PI) - PT_PI)
    step = np.float32(np.float32(PT_PI) / np.float32(H))                    # the host's env_row_cos: cos of the fp32 angles
    t0 = np.float32(np.float32(py) * step); t1 = np.float32(t0 + step)
    c0, c1 = jit("rc0", math.cos(float(t0))), jit("rc1", math.cos(float(t1)))
    cosT = float(c0 * (1 - xz) + c1 * xz)
    theta = math.acos(min(max(cosT, -1.0), 1.0))
    sinT = math.sin(theta)
    v = theta * PT_1_OVER_PI
    with np.errstate(all="ignore"):
        d = jit("dir:d0", np.array([np.sin(phi) * sinT, -cosT, -np.cos(phi) * sinT]))
    cz, sz, cl, sl = _angles(cfg, jit)
    d = jit("dir:sky", rot(rot(d, (0, 1, 0), cz, sz), (1, 0, 0), cl, sl))
    val = env_lookup(tex, u, v, jit)
    val[:3] *= cfg["EnvironmentIntensity"]
    return d, val


def model_miss(d, depth, pdf, envd, cfg, jit):
    """SH/Miss.slang:8-76: [emitted rgb, env pdf]"""
    if cfg["ShowEnvMapDirectly"] or depth > 0:
        cz, sz, cl, sl = _angles(cfg, jit)
        r = jit("dir:r", rot(rot(_f(d), (1, 0, 0), cl, -sl), (0, 1, 0), cz, -sz))
        if math.hypot(r[0], r[2]) < 1e-5: return np.full(4, np.nan)        # a pole: u is made of the rounding of r (undecided)
        gamma, theta = math.asin(min(max(r[1], -1.0), 1.0)), math.atan2(r[0], -r[2])
        c = env_lookup(envd[1], theta * PT_1_OVER_PI * 0.5 + 0.5, gamma * PT_1_OVER_PI + 0.5, jit)
    else: c = np.array([0, 0, 0, 1.0])
    em = c[:3] * cfg["EnvironmentIntensity"]
    if cfg["FurnaceTestMode"]: em = np.ones(3)
    if cfg["EnableSkyMIS"] and depth > 0: em = em * ph(pdf, c[3])
    return np.concatenate([em, c[3:]])


def model_light(draws, ex, pos, sc, emit, br, jit):
    """sample_emissive (SH/Sampler.slang:349-422): (world direction, [colour, pdf], global triangle id); the picks are emulated exactly"""
    count = len(emit)
    if count == 0: return np.zeros(3), np.zeros(4), M32
    _ = next(draws); mi = min(int(np.floor(np.float32(ex()) * np.float32(count))), count - 1)
    br.append(("mesh", mi))
    em = emit[mi]
    tc = em["tc"]
    _ = next(draws); ti = min(int(np.floor(np.float32(ex()) * np.float32(tc))), tc - 1)
    br.append(("tri", ti))
    v, idx = sc["meshes"][em["mesh"]]
    tri = idx[3 * ti: 3 * ti + 3]
    M = em["M"]
    p = [jit(f"c{k}", M[:3, :3] @ v["pos"][tri[k]].astype(np.float64) + M[:3, 3]) for k in range(3)]
    uv = v["uv"][tri].astype(np.float64)
    x0, x1 = next(draws), next(draws)
    su1 = math.sqrt(x0)
    b0 = 1 - su1; b1 = x1 * su1; b2 = 1 - b0 - b1
    tp = p[0] * b0 + p[1] * b1 + p[2] * b2
    uu, vv = b0 * uv[0] + b1 * uv[1] + b2 * uv[2]
    with np.errstate(all="ignore"):
        dl = tp - pos
        toL = dl / np.sqrt(dl @ dl)
        nrm = np.cross(p[2] - p[0], p[1] - p[0]); nrm = nrm / np.sqrt(nrm @ nrm)
        area = np.sqrt(np.cross(p[1] - p[0], p[2] - p[0]) @ np.cross(p[1] - p[0], p[2] - p[0])) * 0.5
        cosT = abs(nrm @ toL)
        mat = sc["materials"][em["material"]]
        te = tex_u8(sc["textures"][mat["EmissiveTextureIndex"]], uu, vv)
        lv = np.concatenate([_f(mat["EmissiveColor"]) * te[:3], [(dl @ dl) / (np.float64(count) * tc * area * cosT)]])
    return toL, lv, em["gid0"] + ti


def emitters(sc):
    """the renderer's emissive list (constant EmissiveColor != 0, Q16) in instance order, with each instance's first global triangle id"""
    out, base = [], 0
    for xf, mi, mat in sc["instances"]:
        tc = len(sc["meshes"][mi][1]) // 3
        if np.any(np.asarray(sc["materials"][mat]["EmissiveColor"]) != 0):
            out.append(dict(mesh=mi, material=mat, tc=tc, gid0=base, M=np.asarray(xf, np.float32).reshape(4, 4).T.astype(np.float64)))
        base += tc
    return out


def tri_bases(sc):
    return np.cumsum([0] + [len(sc["meshes"][mi][1]) // 3 for _, mi, _ in sc["instances"]])[:-1]


class _Counted:
    def __init__(self, it): self.it, self.n = it, 0
    def __iter__(self): return self
    def __next__(self): self.n += 1; return next(self.it)


def model_record(sc, R, i, inp, cfg, envd, emit, luts, draws, jit):
    """one shade_query record: (outputs by B200PT_SQ_* name, branches, draws made)"""
    br, out = [], {f: np.zeros(w) for f, w in NEE_FIELDS.items()}
    draws = _Counted(draws)
    exact = list(itertools.islice(_draws(int(R["rng"][i])), 8))
    ex = lambda: exact[draws.n - 1]
    xf, mi, mat = sc["instances"][R["inst"][i]]
    M = np.asarray(xf, np.float32).reshape(4, 4).T.astype(np.float64)
    b = np.array([1 - inp["u"] - inp["v"], inp["u"], inp["v"]])
    pos = jit("pos", M[:3, :3] @ (inp["P"][0] * b[0] + inp["P"][1] * b[1] + inp["P"][2] * b[2]) + M[:3, 3])
    out["POS"] = pos
    m = sc["materials"][mat]
    uv = inp["UV"][0] * b[0] + inp["UV"][1] * b[1] + inp["UV"][2] * b[2]
    Em = _f(m["EmissiveColor"]) * tex_u8(sc["textures"][m["EmissiveTextureIndex"]], *uv)[:3]
    isLight = bool(np.any(Em > 0))
    br.append(("isLight", isLight))
    sky = None
    if cfg["EnableSkyMIS"]:
        d, lv = model_sky(draws, ex, envd, cfg, br, jit)
        lv[:3] *= cfg["EnvironmentIntensity"]                               # Q7
        out["SKY_W"], out["SKY_LV"] = d, lv
        sky = lv
    light = None
    if cfg["EnableMeshMIS"] and not isLight:
        d, lv, gid = model_light(draws, ex, pos, sc, emit, br, jit)
        out["LIGHT_W"], out["LIGHT_LV"], out["LIGHT_GID"] = d, lv, gid
        light = lv
    ref, hb = model_hit(inp, dict(geo=False, ec=bool(cfg["UseEnergyCompensation"])), luts, draws)
    br += hb
    T, B, N = ref["T"], ref["B"], ref["N"]
    tan = lambda w: _n(np.array([w @ T, w @ B, w @ N]))
    with np.errstate(all="ignore"):
        for name, lv in (("SKY", sky), ("LIGHT", light)):
            if lv is None: continue
            need = bool(lv[3] > 0)
            br.append((name, "need", need))
            if name == "SKY" or need: out[name + "_L"] = tan(out[name + "_W"])
            if not need: continue
            e = ref["eval"](jit(name + "_Limpl", inp[name + "_Limpl"]), br)
            out[name + "_EVAL"] = e
            br.append((name, "pdf", bool(e[3] > 0)))
            if e[3] > 0: out[name + "_C"] = e[:3] * lv[:3] / lv[3] * ph(lv[3], e[3])
        if cfg["EnableMeshMIS"]:
            if isLight:
                P = [M[:3, :3] @ inp["P"][k] + M[:3, 3] for k in range(3)]
                area = np.sqrt(np.cross(P[1] - P[0], P[2] - P[0]) @ np.cross(P[1] - P[0], P[2] - P[0])) * 0.5
                org = jit("org", inp["org"])
                dl = pos - org
                cosT = abs(N @ _n(org - pos))
                tc = next(e["tc"] for e in emit if e["gid0"] == tri_bases(sc)[R["inst"][i]])
                lp = (1.0 / len(emit)) * (1.0 / tc) * (1.0 / area) * ((dl @ dl) / cosT)
                out["EMITTED"] = Em * ph(inp["pay_pdf"], max(lp, cfg["EmissiveMeshSamplingPDFBias"]))
        else: out["EMITTED"] = Em
    br.append(("finite", tuple(bool(np.all(np.isfinite(v))) for v in out.values() if not np.isscalar(v))))
    return out, br, draws.n


def _jit_exact(key, x):
    return _f(x)


def _jits(rng):
    """NPERT perturbation functions paired like _perturbations: a pair moves each quantity both ways"""
    out = []
    for _ in range(NPERT // 2):
        sg = {}
        for pm in (1.0, -1.0):
            def jit(key, x, sg=sg, pm=pm):
                x = _f(x)
                if key not in sg: sg[key] = rng.choice([-1.0, 1.0], np.shape(x))
                if key.startswith("dir:"): return x + pm * REL * sg[key] * np.abs(x).max()   # a direction's rounding is relative to its length
                return x * (1 + pm * REL * sg[key])
            out.append(jit)
    return out


def check_nee(sc, R, got, cfg, envd, k=K, label=""):
    """returns (records checked in full, undecided mask, failures, per-record margins by field); got: [n, STRIDE] records"""
    luts = util.luts(); emit = emitters(sc)
    rng = np.random.default_rng(7)
    n = len(R["inst"])
    checked = 0; undecided = np.zeros(n, bool); fails = []
    margins = {f: np.full(n, np.nan) for f in NEE_FIELDS}
    for i in range(n):
        inp = model_inputs(sc, R, i)
        inp["Ls"] = got[i, SQ["BSDF_L"]: SQ["BSDF_L"] + 3].astype(np.float64)
        inp["V"] = got[i, SQ["V"]: SQ["V"] + 3].astype(np.float64)
        inp["org"] = R["org"][i].astype(np.float64); inp["pay_pdf"] = float(R["pdf"][i])
        for f in ("SKY", "LIGHT"): inp[f + "_Limpl"] = got[i, SQ[f + "_L"]: SQ[f + "_L"] + 3].astype(np.float64)
        ref, br, nd = model_record(sc, R, i, inp, cfg, envd, emit, luts, _draws(int(R["rng"][i])), _jit_exact)
        runs = [model_record(sc, R, i, q, cfg, envd, emit, luts, _draws(int(R["rng"][i]), rng), j) for q, j in zip(_perturbations(inp, rng), _jits(rng))]
        if any(b != br for _, b, _ in runs) or ("cancel", True) in br or ref_v_below(got, i):
            undecided[i] = True; continue
        checked += 1
        g = got[i]
        s = int(R["rng"][i])
        for _ in range(nd): s = pcg(s)
        if g[SQ["RNG"]: SQ["RNG"] + 1].view(np.uint32)[0] != s: fails.append((label, i, "RNG"))
        gid = ref.get("LIGHT_GID", M32)
        if g[SQ["LIGHT_GID"]: SQ["LIGHT_GID"] + 1].view(np.uint32)[0] != gid: fails.append((label, i, "LIGHT_GID", gid))
        for f, w in NEE_FIELDS.items():
            val = _f(ref[f]); gv = g[SQ[f]: SQ[f] + w].astype(np.float64)
            fin = np.isfinite(val)
            if not np.array_equal(np.isfinite(gv), fin):
                fails.append((label, i, f, "finiteness", gv.tolist(), val.tolist())); continue
            if not fin.any(): continue
            spread = max(np.abs(_f(o[f])[fin] - val[fin]).max() for o, _, _ in runs)
            margin = k * spread + VALUE_ULPS * np.spacing(np.float32(np.abs(val[fin]).max()))
            margins[f][i] = margin
            if not np.abs(gv[fin] - val[fin]).max() <= margin:
                fails.append((label, i, f, gv.tolist(), val.tolist(), float(margin)))
    return checked, undecided, fails, margins


def ref_v_below(got, i):
    return not got[i, SQ["V"] + 2] > 0                                      # a view below the bent frame (the shading model skips it too)


def check_miss(dirs, depth, pdf, got, cfg, envd, k=K, label=""):
    """miss_query records against model_miss; returns (failures, per-record margins [n, 4], undecided mask).  A direction at a pole is
    undecided: its u is made of the rounding of the rotated direction."""
    rng = np.random.default_rng(9)
    fails = []; margins = np.full((len(dirs), 4), np.nan); undecided = np.zeros(len(dirs), bool)
    for i in range(len(dirs)):
        d = dirs[i].astype(np.float64)
        ref = model_miss(d, int(depth[i]), float(pdf[i]), envd, cfg, _jit_exact)
        runs = [model_miss(j("dir:d", d), int(depth[i]), float(pdf[i]), envd, cfg, j) for j in _jits(rng)]
        if any(np.isnan(r).all() for r in [ref] + runs):
            undecided[i] = True; continue
        fin = np.isfinite(ref)
        gv = got[i].astype(np.float64)
        if not np.array_equal(np.isfinite(gv), fin): fails.append((label, i, "finiteness", gv.tolist(), ref.tolist())); continue
        rf = [r for r in runs if np.array_equal(np.isfinite(r), fin)]
        spread = np.max([np.abs(r - ref)[fin] for r in rf], axis=0) if rf else np.full(fin.sum(), np.inf)
        for f, sl in (("RGB", slice(0, 3)), ("PDF", slice(3, 4))):
            m = fin[sl]
            if not m.any(): continue
            sp = np.zeros(4); sp[fin] = spread
            margin = k * sp[sl][m].max() + VALUE_ULPS * np.spacing(np.float32(np.abs(ref[sl][m]).max()))
            margins[i, sl] = margin
            if not np.abs(gv[sl][m] - ref[sl][m]).max() <= margin: fails.append((label, i, f, gv[sl].tolist(), ref[sl].tolist(), float(margin)))
    assert undecided.mean() <= 0.1, undecided.mean()
    return fails, margins, undecided


# ---------------------------------------------------------------- scenes, records and draw thresholds
def _xf(X):
    return np.asarray(X, np.float32).T.reshape(-1)


def _T(x, y, z):
    X = np.eye(4); X[:3, 3] = (x, y, z); return X


def _mesh(P, tris, uv=None):
    P = np.asarray(P, np.float32)
    idx = np.asarray(tris, np.uint32).reshape(-1)
    v = np.zeros(len(P), gltf_ref.VERTEX_DTYPE)
    v["pos"] = P
    v["nrm"] = (0, 0, 1)
    v["uv"] = P[:, :2] * 0.37 + 0.5 if uv is None else uv
    return v, idx


def _grid(nx, ny):
    xs, ys = np.meshgrid(np.linspace(-1, 1, nx + 1), np.linspace(-1, 1, ny + 1))
    P = np.stack([xs.ravel(), ys.ravel(), 0.05 * np.sin(3 * xs.ravel())], 1)
    t = []
    for j in range(ny):
        for i in range(nx):
            a = j * (nx + 1) + i
            t += [a, a + 1, a + nx + 2, a, a + nx + 2, a + nx + 1]
    return _mesh(P, t)


EM_TEX = {"em2x2": np.array([[[255, 40, 90, 255], [30, 200, 255, 255]], [[128, 255, 0, 255], [200, 90, 160, 255]]], np.uint8),
          # columns 0-1 black: a hit with u in [1/8, 3/8] samples black texels only and is not a light there (Q16)
          "emhalf": np.concatenate([np.zeros((4, 2, 4), np.uint8), np.array([[[255, 128, 64, 255], [90, 255, 30, 255]]] * 4, np.uint8)], 1)}


def light_scene():
    """receivers around five emissive instances: a scaled quad, a mirrored triangle, a sheared 7-triangle fan, a 300-triangle grid with a
    half-black texture, a mesh with a zero-area triangle; the quad's mesh is instanced once more without emission"""
    tex_names = TEX_NAMES + list(EM_TEX)
    def emat(color, tex="white", **kw):
        m = _mat(**kw); m["EmissiveColor"] = color; m["EmissiveTextureIndex"] = tex_names.index(tex); return m
    mats = [_mat(Roughness=0.5), _mat(Roughness=0.3, Metallic=1.0), emat((4, 3, 2)), emat((3, 0, 1.5)), emat((2, 2, 2), "em2x2"), emat((5, 5, 5), "emhalf")]
    fan = [[0, 0, 0]] + [[math.cos(a), math.sin(a), 0] for a in np.linspace(0, 1.75 * math.pi, 8)]
    meshes = [_quad_mesh(0.25), _mesh([[0, 0, 0], [1.2, 0, 0], [0.3, 0.9, 0]], [0, 1, 2]), _mesh(fan, [[0, k, k + 1] for k in range(1, 8)]),
              _grid(10, 15), _mesh([[0, 0, 0], [1, 0, 0], [0, 1, 0], [2, 2, 0], [3, 3, 0]], [0, 1, 2, 1, 3, 4])]
    shear = np.eye(4); shear[0, 1] = 0.6; shear[1, 2] = 0.3
    inst = [(_xf(_T(0, 0, 3) @ np.diag([1.5, 0.7, 1, 1])), 0, 2),                 # 0  E0 scaled quad
            (_xf(_T(-2.5, 0, 2.5) @ np.diag([-1.0, 1, 1, 1])), 1, 3),            # 1  E1 mirrored triangle, zero green
            (_xf(_T(3, 0.5, 2.5) @ shear), 2, 4),                                 # 2  E2 sheared fan, 2x2 texture
            (_xf(_T(-1, 3, 2.0) @ np.diag([0.8, 0.8, 1, 1])), 3, 5),             # 3  E3 300-triangle grid, half black
            (_xf(_T(1, -3, 2.5)), 4, 2),                                          # 4  E4 with a zero-area triangle
            (_xf(_T(0, -4, 2.5)), 0, 0),                                          # 5  the quad mesh again, not emissive
            (_xf(np.eye(4)), 0, 0),                                               # 6  receiver facing the lights
            (_xf(_T(3.2, 0, 3)), 0, 1),                                           # 7  in E0's plane
            (_xf(_T(0, 0, 3.6)), 0, 0),                                           # 8  behind E0
            (_xf(_T(0, 0, 3 - 1e-3) @ np.diag([0.5, 0.3, 1, 1])), 0, 1),         # 9  1e-3 under E0
            (_xf(_T(0, 0, -1e4)), 0, 0)]                                          # 10 1e4 away
    return {"meshes": meshes, "materials": np.array(mats), "textures": [TEX[n] for n in TEX_NAMES] + list(EM_TEX.values()), "instances": inst,
            "camera_view": np.eye(4, dtype=np.float32).reshape(-1), "aspect": 1.0}


def light_records(sc, seed, n_recv=24, n_emit=10):
    """hits on the receivers (n_recv each) and on the emitters (n_emit each): random triangles and barycentrics, views from either side"""
    rng = np.random.default_rng(seed)
    R = dict(inst=[], prim=[], uv=[], dir=[], org=[], pdf=[], rng=[], L=[])
    for i, (xf, mi, mat) in enumerate(sc["instances"]):
        M = np.asarray(xf, np.float64).reshape(4, 4).T
        v, idx = sc["meshes"][mi]
        for j in range(n_recv if i >= 5 else n_emit):
            p = int(rng.integers(0, len(idx) // 3))
            u, w = rng.random(2) * 0.5
            P = v["pos"][idx[3 * p: 3 * p + 3]].astype(np.float64)
            gn = np.linalg.inv(M[:3, :3]).T @ np.cross(P[1] - P[0], P[2] - P[0])
            gn = gn / np.linalg.norm(gn) if np.linalg.norm(gn) > 0 else np.array([0, 0, 1.0])
            pos = M[:3, :3] @ (P[0] * (1 - u - w) + P[1] * u + P[2] * w) + M[:3, 3]
            cos = [1.0, 0.7, 0.3, 0.05][j % 4] * (1 if j % 3 else -1)
            a = rng.normal(size=3); a -= (a @ gn) * gn; a /= np.linalg.norm(a)
            d = -(cos * gn + math.sqrt(1 - cos * cos) * a)
            R["inst"].append(i); R["prim"].append(p); R["uv"].append((u, w)); R["dir"].append(d); R["org"].append(pos - d * rng.uniform(0.3, 3))
            R["pdf"].append(rng.uniform(0.05, 4)); R["rng"].append(int(rng.integers(0, 2 ** 32))); R["L"].append(-d)
    return {k: np.array(v, np.float32 if k not in ("inst", "prim", "rng") else np.uint32) for k, v in R.items()}


def states_for(value, before, want=lambda d: True, limit=1):
    """sampler states whose draw number `before` (from 0) is exactly the fp32 `value` and whose earlier draws satisfy want(list)"""
    v = float(np.float32(value))
    half = float(np.spacing(np.float32(v))) / 2
    lo, hi = int(math.ceil((v - half) * 2.0 ** 32)), min(int(math.floor((v + half) * 2.0 ** 32)), M32)
    out = []
    for s in range(max(lo, 0), hi + 1):
        if float(np.float32(s)) / 2.0 ** 32 != v: continue
        st, earlier = s, []
        for _ in range(before):
            st = pcg_inv(st); earlier.insert(0, float(np.float32(st)) / 2.0 ** 32)
        if want(earlier):
            out.append(pcg_inv(st))
            if len(out) >= limit: break
    return out


def _texel(xx, size):
    return min(int(np.float32(xx) * np.float32(size)), size - 1)


def sky_thresholds(envd, seed):
    """states whose xx sits on texel-index boundaries, whose xy sits on its texel's imp and one ulp either side, and whose draws are 1.0"""
    _, tex, alias = envd
    size = tex.shape[0] * tex.shape[1]
    rng = np.random.default_rng(seed)
    out = []
    for k in rng.choice(np.arange(max(1, size // 512), size), min(6, size - 1), replace=False):
        x = np.float32(k / size)
        for v in (np.nextafter(x, np.float32(0)), x, np.nextafter(x, np.float32(2))):
            if 2.0 ** -9 <= v <= 1: out.append(state_for_draw(float(v), 0))
    imp = alias["Importance"]
    cand = np.flatnonzero((imp >= 2.0 ** -8) & (imp < 1))
    found = 0
    for t in rng.permutation(cand)[:400]:
        for v in (np.nextafter(imp[t], np.float32(0)), imp[t], np.nextafter(imp[t], np.float32(2))):
            out += states_for(float(v), 1, lambda d, t=t: _texel(d[0], size) == t)
        found = len(out)
        if found > 40: break
    out += [state_for_draw(1.0, b) for b in range(3)]
    return out


def light_thresholds(sc, before):
    """states whose mesh and triangle picks sit on their k / count boundaries and at 1.0, and whose x0, x1 are 1.0 (a sample on an edge)"""
    emit = emitters(sc); count = len(emit)
    out = []
    for k in range(1, count + 1):
        x = np.float32(k / count)
        for v in (np.nextafter(x, np.float32(0)), x):
            out += states_for(float(v), before)
    for e in emit:
        if e["tc"] < 2: continue
        for k in (1, e["tc"] // 2, e["tc"]):
            x = np.float32(k / e["tc"])
            pick = lambda d, e=e: min(int(math.floor(np.float32(d[-1]) * np.float32(count))), count - 1) == emit.index(e)
            out += states_for(float(x), before + 1, pick, limit=2)
    out += [state_for_draw(1.0, before + b) for b in range(4)]
    return out


def with_states(R, states, seed):
    """R plus one record per state, each a copy of a random record of R"""
    pick = np.random.default_rng(seed).integers(0, len(R["inst"]), len(states))
    out = {k: np.concatenate([R[k], R[k][pick]]) for k in R}
    out["rng"][len(R["inst"]):] = np.array(states, np.uint32)
    return out


# ---------------------------------------------------------------- cases
ROT = {(0, 0), (70, 20), (180, -90), (-45, 90), (360, 0.001)}
SKY_CASES = {"synthetic-0": ("synthetic", (0, 0), 1.0), "synthetic-70": ("synthetic", (70, 20), 2.5), "37x19": ("37x19", (180, -90), 1.0),
             "37x1": ("37x1", (-45, 90), 2.5), "1x19": ("1x19", (360, 0.001), 1.0), "hot00": ("hot00", (0, 0), 1.0), "hot00-180": ("hot00", (180, -90), 2.5),
             "halfblack": ("halfblack", (70, 20), 1.0), "constant": ("constant", (-45, 90), 1.0), "bench": ("bench", (360, 0.001), 1.0)}
LIGHT_CASES = {"light": dict(EmissiveMeshSamplingPDFBias=0.0, EnableSkyMIS=0), "light-bias": dict(EmissiveMeshSamplingPDFBias=2.0, EnableSkyMIS=0),
               "light-sky": dict(EmissiveMeshSamplingPDFBias=0.0, EnableSkyMIS=1, env="37x19", rot=(70, 20), I=2.5)}
CASES = sorted(SKY_CASES) + sorted(LIGHT_CASES)
SKY_MATS = [_mat(Roughness=0.5), _mat(Roughness=0.3, Metallic=1.0), _mat(Roughness=0.35, Metallic=0.5, Transmission=0.5)]


def _cfg(**kw):
    c = dict(EnableSkyMIS=1, EnableMeshMIS=1, ShowEnvMapDirectly=1, FurnaceTestMode=0, EnvironmentIntensity=1.0, SkyRotationAzimuth=0.0,
             SkyRotationAltitude=0.0, EmissiveMeshSamplingPDFBias=0.0, UseEnergyCompensation=1)
    c.update(kw); return c


@functools.lru_cache(maxsize=None)
def case(name):
    """(scene, env name, config dict, records, number of records before the draw-threshold ones)"""
    if name in SKY_CASES:
        en, (az, al), I = SKY_CASES[name]
        sc = scene_for(SKY_MATS)
        R = records(sc, 30, 21)
        n = len(R["inst"])
        R = with_states(R, sky_thresholds(env(en), 5), 6)
        return sc, en, _cfg(EnableMeshMIS=0, EnvironmentIntensity=I, SkyRotationAzimuth=float(az), SkyRotationAltitude=float(al)), R, n
    kw = dict(LIGHT_CASES[name])
    en, (az, al), I = kw.pop("env", "synthetic"), kw.pop("rot", (0, 0)), kw.pop("I", 1.0)
    sc = light_scene()
    R = light_records(sc, 31)
    n = len(R["inst"])
    R = with_states(R, light_thresholds(sc, 3 * kw["EnableSkyMIS"]), 7)
    return sc, en, _cfg(EnvironmentIntensity=I, SkyRotationAzimuth=float(az), SkyRotationAltitude=float(al), **kw), R, n


def _oracle(sc, en, cfg):
    _, env_pdf, alias = env(en)
    return orc.Scene(sc, env_pdf, alias, util.luts()), orc.default_config(**cfg)


def _shade(X, cfg_or_none, R):
    args = (R["inst"], R["prim"], R["uv"], R["dir"], R["org"], R["pdf"], R["rng"], R["L"])
    return X.shade_query(cfg_or_none, *args) if cfg_or_none is not None else X.shade_query(*args)


def _report(label, R, und, n_base):
    return f"{label}: {len(und)} records ({len(und) - n_base} on draw thresholds), undecided share {und[:n_base].mean():.3f} (thresholds {und[n_base:].mean():.3f})"


def test_rotations_cover_the_issue_list():
    assert {v[1] for v in SKY_CASES.values()} == ROT and set(ENV_NAMES) == {v[0] for v in SKY_CASES.values()}


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_float64_model(name):
    """CPU only: the oracle's NEE draws, terms and emission against the model, on every case.  Validates the model and the margins."""
    sc, en, cfg, R, n_base = case(name)
    S, oc = _oracle(sc, en, cfg)
    got = _shade(S, oc, R)
    checked, und, fails, _ = check_nee(sc, R, got, cfg, env(en), label=name)
    print(_report(f"oracle vs model {name}", R, und, n_base), f"checked {checked}")
    assert not fails, fails[:5]
    assert und[:n_base].mean() <= UNDECIDED_MAX, und[:n_base].mean()
    if cfg["EnableSkyMIS"]: assert np.any(got[~und, SQ["SKY_LV"] + 3] > 0)
    if cfg["EnableMeshMIS"]: assert np.any(got[~und, SQ["LIGHT_LV"] + 3] > 0) and np.any(got[~und, SQ["EMITTED"]] > 0)


MISS_CFGS = [dict(), dict(ShowEnvMapDirectly=0), dict(EnableSkyMIS=0), dict(FurnaceTestMode=1)]


def miss_inputs(seed, cfg):
    """random directions, the poles and the u seam (before and after the sky rotation), at depths 0 and 1, pdfs from 0 to 10"""
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(150, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    special = np.array([[0, 1, 0], [0, -1, 0], [0, 0, 1], [1e-7, 0, 1], [-1e-7, 0, 1], [0, 0, -1], [1, 0, 0], [0.6, 0.8, 0]], np.float64)
    cz, sz, cl, sl = _angles(cfg, _jit_exact)
    rotated = np.array([rot(rot(s, (0, 1, 0), cz, sz), (1, 0, 0), cl, sl) for s in special])
    d = np.concatenate([d, special, rotated]).astype(np.float32)
    depth = np.arange(len(d)) % 2
    pdf = rng.uniform(0, 10, len(d)).astype(np.float32); pdf[::7] = 0
    return d, depth.astype(np.uint32), pdf


@pytest.mark.parametrize("en", ENV_NAMES)
def test_oracle_miss_matches_float64_model(en):
    for j, mk in enumerate(MISS_CFGS):
        az, al = sorted(ROT)[j % len(ROT)]
        cfg = _cfg(SkyRotationAzimuth=float(az), SkyRotationAltitude=float(al), EnvironmentIntensity=(1.0, 2.5)[j % 2], **mk)
        S, oc = _oracle(scene_for(SKY_MATS[:1]), en, cfg)
        d, depth, pdf = miss_inputs(j, cfg)
        fails, _, _ = check_miss(d, depth, pdf, S.miss_query(oc, d, depth, pdf), cfg, env(en), label=f"{en} {mk}")
        assert not fails, fails[:5]


# ---------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def pt():
    import torch
    if not torch.cuda.is_available(): pytest.skip("no CUDA device")
    import vpt_b200
    return vpt_b200


def _tracer(sc, en, cfg):
    return util.product_tracer("cornell_box", 8, 8, env=env(en), scene=sc, **cfg)


def test_miss_record_layout_matches_header():
    import re
    import vpt_b200
    hdr = open(f"{util.ROOT}/include/b200pt.h").read()
    assert {m.group(1): int(m.group(2)) for m in re.finditer(r"#define B200PT_MQ_(\w+)\s+(\d+)", hdr)} == MQ == vpt_b200.MQ


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_gpu_matches_oracle_and_model(pt, name):
    sc, en, cfg, R, n_base = case(name)
    S, oc = _oracle(sc, en, cfg)
    ref = _shade(S, oc, R)
    got = _shade(_tracer(sc, en, cfg), None, R)
    checked, und, fails, _ = check_nee(sc, R, got, cfg, env(en), label=name)
    agree, bad = _gpu_vs_oracle(got[~und], ref[~und], fields=ORACLE_FIELDS)     # an undecided record may take either side of a rounding
    print(_report(f"GPU vs model {name}", R, und, n_base), f"checked {checked}; GPU vs oracle: same path {agree:.4f}")
    assert not fails, fails[:5]
    assert und[:n_base].mean() <= UNDECIDED_MAX, und[:n_base].mean()
    assert agree >= 0.97 and not bad, (agree, bad[:5])


@pytest.mark.gpu
@pytest.mark.parametrize("en", ENV_NAMES)
def test_gpu_miss_matches_oracle_and_model(pt, en):
    T = None
    for j, mk in enumerate(MISS_CFGS):
        az, al = sorted(ROT)[j % len(ROT)]
        cfg = _cfg(SkyRotationAzimuth=float(az), SkyRotationAltitude=float(al), EnvironmentIntensity=(1.0, 2.5)[j % 2], **mk)
        sc = scene_for(SKY_MATS[:1])
        S, oc = _oracle(sc, en, cfg)
        T = _tracer(sc, en, cfg)
        d, depth, pdf = miss_inputs(j, cfg)
        got, ref = T.miss_query(d, depth, pdf), S.miss_query(oc, d, depth, pdf)
        fails, _, und = check_miss(d, depth, pdf, got, cfg, env(en), label=f"{en} {mk}")
        assert not fails, fails[:5]
        got, ref = got[~und], ref[~und]
        assert np.array_equal(np.isfinite(got), np.isfinite(ref))
        scale = np.maximum(np.abs(ref).max(1, keepdims=True), 1e-6)
        fin = np.isfinite(ref).all(1)
        assert np.all(np.abs(got - ref)[fin] / scale[fin] <= 2e-3), np.max(np.abs(got - ref)[fin] / scale[fin])


def sky_pairs(T, R, got, cfg, envd, margins, und):
    """decided sky draws with lv.w > 0, seen from the BSDF side: returns the failures and the number of pairs checked"""
    sel = np.flatnonzero(~und & (got[:, SQ["SKY_LV"] + 3] > 0))
    w = got[sel, SQ["SKY_W"]: SQ["SKY_W"] + 3]
    lv = got[sel, SQ["SKY_LV"]: SQ["SKY_LV"] + 4].astype(np.float64)
    bp = got[sel, SQ["SKY_EVAL"] + 3].astype(np.float64)
    pay = np.where(bp > 0, bp, 1.0).astype(np.float32)
    mq = T.miss_query(w, 1, pay).astype(np.float64)
    mf, mm, mu = check_miss(w, np.ones(len(sel)), pay, mq, cfg, envd)
    I = cfg["EnvironmentIntensity"]
    fails = list(mf)
    for k, i in enumerate(sel):
        if mu[k]: continue                                                  # a draw at a pole (xz on 0 or 1 in the first or last row)
        tol = margins["SKY_LV"][i] + mm[k].max()
        if not abs(mq[k, 3] - lv[k, 3]) <= tol: fails.append(("pdf", int(i), mq[k, 3], lv[k, 3], tol))
        want = lv[k, :3] / I * ph(pay[k], lv[k, 3])                        # the miss side's radiance, weighted at the BSDF pdf
        if not np.abs(mq[k, :3] - want).max() <= tol + 2 * VALUE_ULPS * np.spacing(np.float32(np.abs(want).max())): fails.append(("rgb", int(i), mq[k, :3].tolist(), want.tolist(), tol))
        wsum = ph(lv[k, 3], pay[k]) + ph(pay[k], mq[k, 3])
        if not abs(wsum - 1) <= 4 * tol / max(lv[k, 3], 1e-30) + 1e-6: fails.append(("weights", int(i), wsum))
    return fails, int((~mu).sum())


def light_pairs(T, sc, R, got, cfg):
    """each light draw traced from the shading point with the renderer's light-ray offset; where the closest hit is the sampled triangle,
    shade_query there must give the BSDF-side weight power_heuristic(pdf, max(lv.w |NG.l| / |N.l|, bias)).  Returns (failures, pairs, draws)."""
    sel = np.flatnonzero((got[:, SQ["LIGHT_LV"] + 3] > 0) & np.isfinite(got[:, SQ["LIGHT_LV"] + 3]) & (got[:, SQ["LIGHT_EVAL"] + 3] > 0))
    pos = got[sel, SQ["POS"]: SQ["POS"] + 3]; l = got[sel, SQ["LIGHT_W"]: SQ["LIGHT_W"] + 3]
    ro = pos + l * np.float32(1e-2)                                         # :171, both roundings in fp32 as the renderer makes them
    h = T.trace_query("global", "closest", ro, l, 1e-4, 1e6, stats=False)
    gid = tri_bases(sc)[h["inst"]] + h["prim"]
    hit = (h["t"] > 0) & (gid == got[sel, SQ["LIGHT_GID"]].view(np.uint32))
    s = sel[hit]
    e_pdf = got[s, SQ["LIGHT_EVAL"] + 3]
    r2 = T.shade_query(h["inst"][hit], h["prim"][hit], h["uv"][hit], l[hit], pos[hit], e_pdf, 0, None)
    lv = got[s, SQ["LIGHT_LV"]: SQ["LIGHT_LV"] + 4].astype(np.float64)
    fails = []
    for k, i in enumerate(s):
        L = l[hit][k].astype(np.float64); N = r2[k, SQ["N"]: SQ["N"] + 3].astype(np.float64); NG = r2[k, SQ["NG"]: SQ["NG"] + 3].astype(np.float64)
        cg, cs = abs(NG @ L), abs(N @ L)
        lp = max(lv[k, 3] * cg / cs, cfg["EmissiveMeshSamplingPDFBias"])
        want = ph(float(e_pdf[k]), lp)
        c = int(np.argmax(lv[k, :3]))
        if not lv[k, c] > 0: continue                                       # a black texel: no radiance on either side
        wgot = r2[k, SQ["EMITTED"] + c] / lv[k, c]
        d = math.sqrt(float(np.sum((pos[hit][k].astype(np.float64) - ro[hit][k]) ** 2))) + float(h["t"][hit][k])
        rel = K * REL * (4 + np.abs(pos[hit][k]).max() / d + 1 / cg + 1 / cs)
        tol = 2 * want * (1 - want) * rel + 16 * 2.0 ** -24                # and a few ulps of the fp32 weight and of the division above
        if not abs(wgot - want) <= tol: fails.append((int(i), wgot, want, tol, cg, cs, lv[k].tolist(), float(e_pdf[k]), r2[k, SQ["EMITTED"]: SQ["EMITTED"] + 3].tolist()))
    return fails, len(s), len(sel)


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_nee_pairs(pt, name):
    """the sky pair holds in the reference exactly, the light pair up to its geometric-versus-shading-normal ratio (Q10 tilt included)"""
    sc, en, cfg, R, _ = case(name)
    T = _tracer(sc, en, cfg)
    got = _shade(T, None, R)
    _, und, fails, margins = check_nee(sc, R, got, cfg, env(en), label=name)
    assert not fails, fails[:5]
    if cfg["EnableSkyMIS"]:
        f, n = sky_pairs(T, R, got, cfg, env(en), margins, und)
        print(f"sky pairs {name}: {n}")
        assert n > 10 and not f, f[:5]
    if cfg["EnableMeshMIS"]:
        f, n, m = light_pairs(T, sc, R, got, cfg)
        print(f"light pairs {name}: {n} of {m} draws reach their triangle")
        assert n > 20 and not f, f[:5]


@pytest.mark.gpu
def test_margin_is_tight(pt):
    """K / 10 rejects some GPU answer, so K is not loose by an order of magnitude"""
    fails = 0
    for name in CASES:
        sc, en, cfg, R, _ = case(name)
        fails += len(check_nee(sc, R, _shade(_tracer(sc, en, cfg), None, R), cfg, env(en), k=K / 10)[2])
    assert fails > 0


@pytest.mark.gpu
def test_miss_query_refuses_bad_input(pt):
    T = pt.PathTracer(0)
    d = np.zeros((2, 3), np.float32)
    with pytest.raises(pt.B200ptError): T.miss_query(d, 1, 0.5)             # no scene
    T.set_scene(scene_for(SKY_MATS[:1]))
    with pytest.raises(pt.B200ptError): T.miss_query(d, 1, 0.5)             # no environment map
