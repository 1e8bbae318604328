"""One shading step of the renderer's hit kernel, checked hit by hit (b200pt_shade_query) against the CPU oracle (orc_shade_query) and a
float64 model, on materials no shipped scene has: anisotropic GGX with rotation, mixed lobes, rough glass at real IORs seen from both
sides, LUT layer ties, textured metallic, tilted normal maps, mirrored instances, grazing views.

Model: the Slang functions the oracle restates (surface frame and normal-map bends, material set-up with bilinear u8 texels and
pow(., 2.2), the LUT bilinear with its nearest-even layer, anisotropic GGX D / G1 / VNDF, dielectric and Schlick Fresnel, EvaluateBSDF and
the direction part of SampleBSDF) in numpy float64.  The draws are exact: they come from the record's sampler state through pcg_hash.

Margins: the model runs at the exact fp32 inputs and again at NPERT random relative perturbations of size 2^-23 of every input (vertices,
normals, uvs, barycentrics, ray direction, the caller's L, the material scalars, and the draws, which stand in for the rounding of 2 pi u
and its kin), in +/- pairs.  The sampled direction is evaluated at
the fp32 L the implementation returned, and every stage after V runs on the implementation's fp32 V (both perturbed too); that L and that V
are compared with the model's own.  Each stage is thus checked on the inputs it was given, so the margins need not absorb the rounding of
earlier stages.  For each output,

    margin = K * (largest deviation of a perturbed run from the exact one) + VALUE_ULPS * ulp32(largest component of that output)

A record is undecided when a perturbation flips any branch the model takes: the lobe pick (x1 < pm, x1 < pm + pd), u < F, sinT2 > 1,
L.z < 0, L.z <= 1e-5, validRefraction, H.z < 0, glassEC > 0.01, |V Eta + L| < 1e-3 (the refraction half vector is then made of rounding), |n.z| < 0.9999999, the two dot < 0 bends of the surface frame, the
geometry-normal rejection and the LUT layer (a half-integer layer rounds to even).  The outputs of undecided records are skipped and counted, except
the surface frame and material (N, T, B, V, Ax, Ay, Eta, pm, pd, pg), which are still checked when only branches after the frame flip; the
undecided share must stay under UNDECIDED_MAX per group.  The LUT texels are taken as exact (they are fp32 data).  Flags (validDir, refracted, entered,
rejected) must be equal on decided records.  test_margin_is_tight shows that K / 10 rejects some GPU answer.

Sky and light NEE, their terms c and the emission term are compared GPU against oracle here; test_nee_queries.py checks them, and miss
shading, against a float64 model of the samplers.  A value the oracle computes as inf / NaN must be inf / NaN on the GPU too.  The class kernels are compared with the all-lobes kernel
(a class kernel must never be finite where the all-lobes one is not), and the per-material precompute with the per-hit texel path bit for bit.
"""
import math

import numpy as np
import pytest

import util
from util import gltf_ref, orc

K = 64.0
VALUE_ULPS = 8
NPERT = 4
UNDECIDED_MAX = 0.35
REL = 2.0 ** -23

SQ = dict(N=0, T=3, B=6, NG=9, INSIDE=12, AX=13, AY=14, ETA=15, PM=16, PD=17, PG=18, BASECOLOR=19, ROUGHNESS=22, V=23, H=26, EMITTED=29,
          SKY_L=32, SKY_LV=35, SKY_EVAL=39, SKY_C=43, LIGHT_L=46, LIGHT_LV=49, LIGHT_EVAL=53, LIGHT_C=57, LIGHT_GID=60, BSDF_L=61, BSDF_EVAL=64,
          VALID=68, SCATTER=69, SAMPLE=72, REFRACTED=76, ENTERED=77, REJECTED=78, USER_L=79, USER_EVAL=82, RNG=86, CLASS=87, POS=88, SKY_W=91,
          LIGHT_W=94, STRIDE=97)


# ---------------------------------------------------------------- pcg_hash and its inverse (a bijection on 32-bit words)
M32 = 0xFFFFFFFF


def pcg(s):
    state = (s * 747796405 + 2891336453) & M32
    word = (((state >> ((state >> 28) + 4)) ^ state) * 277803737) & M32
    return ((word >> 22) ^ word) & M32


def pcg_inv(h):
    word = (h ^ (h >> 22)) & M32
    x = (word * pow(277803737, -1, 1 << 32)) & M32
    r = (x >> 28) + 4
    state = x
    for _ in range(32 // r + 1): state = x ^ (state >> r)
    return ((state - 2891336453) * pow(747796405, -1, 1 << 32)) & M32


def draw(s):
    """the next state and the draw Rng::next() makes from it: (float)s / 2^32, with the u32 -> fp32 conversion rounded to nearest"""
    s = pcg(s)
    return s, float(np.float32(s)) / 4294967296.0


def state_for_draw(value, before):
    """a sampler state whose `before + 1`-th draw is exactly the fp32 `value` (in [2^-9, 1])"""
    s = int(round(float(np.float32(value)) * 4294967296.0))
    s = min(s, M32) if value < 1.0 else M32
    assert float(np.float32(s)) / 4294967296.0 == float(np.float32(value))
    for _ in range(before + 1): s = pcg_inv(s)
    return s


def test_pcg_inverse():
    rng = np.random.default_rng(0)
    for s in rng.integers(0, 2 ** 32, 2000, dtype=np.uint64).tolist():
        assert pcg_inv(pcg(s)) == s and pcg(pcg_inv(s)) == s
        assert pcg(s) == orc.pcg_hash(s)


# ---------------------------------------------------------------- float64 model
def _n(a):
    return a / math.sqrt(float(a @ a))


def tex_u8(t, u, v):
    t = np.asarray(t, np.float64) / 255.0
    H, W, C = t.shape
    if W == 1 and H == 1: c = t[0, 0]
    else:
        x, y = u * W - 0.5, v * H - 0.5
        fx, fy = math.floor(x), math.floor(y); ax, ay = x - fx, y - fy
        x0, x1, y0, y1 = fx % W, (fx + 1) % W, fy % H, (fy + 1) % H
        c = (t[y0, x0] + ax * (t[y0, x1] - t[y0, x0])) + ay * ((t[y1, x0] + ax * (t[y1, x1] - t[y1, x0])) - (t[y0, x0] + ax * (t[y0, x1] - t[y0, x0])))
    return np.array([c[0], 0.0, 0.0, 1.0]) if C == 1 else c


def lut(tab, u, v, layer, br):
    Lc, H, W = tab.shape
    li = min(max(int(np.rint(layer)), 0), Lc - 1)                         # round half to even, as __float2int_rn
    br.append(("layer", li))
    x, y = u * W - 0.5, v * H - 0.5
    fx, fy = math.floor(x), math.floor(y); ax, ay = x - fx, y - fy
    c = lambda i, n: min(max(i, 0), n - 1)
    p = tab[li].astype(np.float64)
    a = p[c(fy, H), c(fx, W)] + ax * (p[c(fy, H), c(fx + 1, W)] - p[c(fy, H), c(fx, W)])
    b = p[c(fy + 1, H), c(fx, W)] + ax * (p[c(fy + 1, H), c(fx + 1, W)] - p[c(fy + 1, H), c(fx, W)])
    return a + ay * (b - a)


def fresnel(cosI, eta, br):
    sinT2 = eta * eta * (1 - cosI * cosI)
    br.append(("tir", sinT2 > 1))
    if sinT2 > 1: return 1.0
    cosT = math.sqrt(max(1 - sinT2, 0.0))
    rs = (eta * cosT - cosI) / (eta * cosT + cosI); rp = (eta * cosI - cosT) / (eta * cosI + cosT)
    return 0.5 * (rs * rs + rp * rp)


def g1(m, V):
    return 1.0 / (1.0 + (-1.0 + math.sqrt(1.0 + (m["Ax"] ** 2 * V[0] ** 2 + m["Ay"] ** 2 * V[1] ** 2) / (V[2] * V[2]))) / 2.0)


def ggx_d(m, H):
    e = H[0] ** 2 / m["Ax"] ** 2 + H[1] ** 2 / m["Ay"] ** 2 + H[2] ** 2
    return 1.0 / (math.pi * m["Ax"] * m["Ay"] * e * e)


def vndf(u1, u2, Ve, Ax, Ay):
    Vh = _n(np.array([Ax * Ve[0], Ay * Ve[1], abs(Ve[2])]))
    lensq = Vh[0] ** 2 + Vh[1] ** 2
    T1 = np.array([-Vh[1], Vh[0], 0.0]) / math.sqrt(lensq) if lensq > 0 else np.array([1.0, 0, 0])
    T2 = np.cross(Vh, T1)
    r, phi = math.sqrt(u1), 2 * math.pi * u2
    t1, t2 = r * math.cos(phi), r * math.sin(phi)
    s = 0.5 * (1 + Vh[2])
    t2 = (1 - s) * math.sqrt(1 - t1 * t1) + s * t2
    Nh = T1 * t1 + T2 * t2 + Vh * math.sqrt(max(0.0, 1 - t1 * t1 - t2 * t2))
    return _n(np.array([Ax * Nh[0], Ay * Nh[1], max(0.0, Nh[2])]))


def reflect(i, n):
    return i - n * (2 * (n @ i))


def refract(i, n, eta):
    d = n @ i; k = 1 - eta * eta * (1 - d * d)
    return np.zeros(3) if k < 0 else i * eta - n * (eta * d + math.sqrt(k))


def eval_bsdf(m, c, V, L, ec, br):
    out, pdf = np.zeros(3), 0.0
    br.append(("refr", L[2] < 0))
    if not L[2] < 0:
        H = _n(V + L); VdotH = V @ H
        F = fresnel(abs(VdotH), m["Eta"], br)
        refl = not L[2] <= 1e-5
        br.append(("lz", refl))
        D = GL = rpdf = 0.0
        if refl:
            D = ggx_d(m, H); GL = g1(m, L)
            rpdf = (c["GV"] * max(VdotH, 0.0) * D / V[2]) / (4 * VdotH)
        sch = min(max(1 - VdotH, 0.0), 1.0) ** 5
        Fm = m["Base"] * (1 - sch) + m["Spec"] * sch
        b = Fm * D * c["GV"] * GL / (4 * V[2]) if refl else np.zeros(3)
        if ec: b = c["metalEC"] * b
        out += b * m["pm"]; pdf += rpdf * m["pm"]
        pd_ = L[2] / math.pi * (1.0 if L[2] > 0 else 0.0)
        out += m["Base"] / math.pi * L[2] * m["pd"] * (1 - F); pdf += pd_ * m["pd"] * (1 - F)
        spec = m["Spec"] * D * c["GV"] * GL / (4 * V[2]) if refl else np.zeros(3)
        out += (spec / c["reflEC"] if ec else spec) * m["pd"] * F; pdf += rpdf * m["pd"] * F
        gl = ec and c["glassEC"] > 0.01
        out += (spec / c["glassEC"] if gl else spec) * m["pg"] * F; pdf += rpdf * m["pg"] * F
    else:
        Hr = V * m["Eta"] + L
        br.append(("cancel", math.sqrt(float(Hr @ Hr)) < 1e-3))           # |V Eta + L| this small is set by the fp32 rounding of V and L
        Hr = _n(Hr)
        br.append(("hz", Hr[2] < 0))
        if Hr[2] < 0: Hr = -Hr
        VdotH, LdotH = V @ Hr, L @ Hr
        valid = (VdotH > 0 and LdotH < 0) or (VdotH < 0 and LdotH > 0)
        br.append(("validRefraction", valid))
        F = fresnel(abs(VdotH), m["Eta"], br)
        if valid:
            b, p = np.zeros(3), 0.0
            if not L[2] >= 1e-5:
                D = ggx_d(m, Hr); GL = g1(m, L); G = c["GV"] * GL
                den = LdotH + m["Eta"] * VdotH; eta2 = m["Eta"] ** 2
                p = (c["GV"] * abs(VdotH) * D / V[2]) * (eta2 * abs(LdotH) / den ** 2)
                b = m["Base"] * D * G * eta2 / den ** 2 * (abs(VdotH) * abs(LdotH) / abs(V[2]))
            if ec and c["glassEC"] > 0.01: b = b / c["glassEC"]
            out += b * m["pg"] * (1 - F); pdf += p * m["pg"] * (1 - F)
    return np.concatenate([out, [pdf]])


def model_hit(inp, cfg, luts, draws):
    """inp: float64 inputs of one record (possibly perturbed); draws: iterator of exact draws.  Returns (outputs dict, branch list)."""
    br = []
    b0, b1, b2 = 1 - inp["u"] - inp["v"], inp["u"], inp["v"]
    P, Nv, UV, W = inp["P"], inp["Nv"], inp["UV"], inp["W"]
    lp = P[0] * b0 + P[1] * b1 + P[2] * b2
    uv = UV[0] * b0 + UV[1] * b1 + UV[2] * b2
    gn = _n(_n(np.cross(P[1] - P[0], P[2] - P[0])) @ W)
    n = gn if cfg["geo"] else _n(_n(Nv[0] * b0 + Nv[1] * b1 + Nv[2] * b2) @ W)
    d = _n(inp["dir"]); view = -d
    inside = gn @ view < 0
    br.append(("inside", inside))
    if inside: n, gn = -n, -gn
    upz = abs(n[2]) < 0.9999999
    br.append(("up", upz))
    up = np.array([0, 0, 1.0]) if upz else np.array([1.0, 0, 0])
    T = _n(np.cross(up, n)); B = _n(np.cross(n, T)); N = n
    if not cfg["geo"]:
        t = tex_u8(inp["tex_normal"], *uv)
        N = _n(T * (t[0] * 2 - 1) + B * (t[1] * 2 - 1) + n * (t[2] * 2 - 1))
    bend1 = N @ view < 0
    br.append(("bend1", bend1))
    if bend1: N = _n(N - view * ((N @ view) - 0.01))
    bend2 = _n(reflect(-view, N)) @ gn < 0
    br.append(("bend2", bend2))
    if bend2: N = _n(N + gn * (0.1 + N @ gn))
    T = _n(np.cross(N, up)); B = _n(np.cross(N, T))
    mt = inp["mat"]
    rot = mt["AnisotropyRotation"] * math.pi / 180
    c_, s_ = math.cos(rot), math.sin(rot)
    T = T * c_ + np.cross(N, T) * s_ + N * (N @ T) * (1 - c_); B = np.cross(T, N)
    tb = tex_u8(inp["tex_base"], *uv)
    IOR = max(mt["IOR"], 1.000001)
    m = dict(Base=mt["BaseColor"] * tb[:3] ** 2.2, Spec=mt["SpecularColor"], Roughness=mt["Roughness"] * tex_u8(inp["tex_rough"], *uv)[0],
             Metallic=mt["Metallic"] * tex_u8(inp["tex_metal"], *uv)[0], IOR=IOR)
    aspect = math.sqrt(1 - math.sqrt(mt["Anisotropy"]) * 0.9)
    m["Ax"] = max(1e-5, m["Roughness"] / aspect); m["Ay"] = max(1e-5, m["Roughness"] * aspect)
    pm, pd, pg = m["Metallic"], (1 - m["Metallic"]) * (1 - mt["Transmission"]), (1 - m["Metallic"]) * mt["Transmission"]
    sm = pm + pd + pg
    m.update(pm=pm / sm, pd=pd / sm, pg=pg / sm, Eta=IOR if inside else 1 / IOR)
    V = Vm = _n(np.array([view @ T, view @ B, view @ N]))
    if inp.get("V") is not None: V = inp["V"]                              # the stages after V run on the implementation's fp32 V
    ec = cfg["ec"]
    c = dict(GV=g1(m, V), reflEC=1.0, glassEC=0.0, metalEC=np.ones(3))
    if ec:
        c["glassEC"] = lut(luts[2] if m["Eta"] > 1 else luts[1], math.sqrt(max(V[2], 0.0)), m["Roughness"], (min(max(IOR, 1.0001), 2.0) - 1) * 32, br)
        br.append(("glassEC", c["glassEC"] > 0.01))
        c["reflEC"] = lut(luts[0], V[2], m["Roughness"], mt["Anisotropy"] * 32, br)
        c["metalEC"] = 1 + m["Base"] * ((1 - c["reflEC"]) / c["reflEC"])
    u1, u2, x1 = next(draws), next(draws), next(draws)
    H = vndf(u1, u2, V, m["Ax"], m["Ay"])
    F = fresnel(V @ H, m["Eta"], br)
    refracted = False
    lobe = 0 if x1 < m["pm"] else (1 if x1 < m["pm"] + m["pd"] else 2)
    br.append(("lobe", lobe))
    if lobe == 0: L = _n(reflect(-V, H))
    else:
        uF = next(draws)
        br.append(("uF", uF < F))
        if uF < F: L = _n(reflect(-V, H))
        elif lobe == 1:
            a, bb = next(draws), next(draws)
            z = 1 - 2 * bb; rad = math.sqrt(1 - z * z)
            L = _n(np.array([rad * math.cos(2 * math.pi * a), rad * math.sin(2 * math.pi * a), z]) + [0, 0, 1.0])
        else: L = _n(refract(-V, H, m["Eta"])); refracted = True
    valid = not ((L[2] < 0 and not refracted) or (refracted and L[2] >= 0))
    br.append(("valid", valid))
    Lv = L if valid else np.zeros(3)
    # the sampled direction is evaluated where the implementation put it: an fp32 L next to a sharp lobe moves D by far more than the
    # inputs' rounding would, and that L is checked against the model's on its own
    ev = eval_bsdf(m, c, V, inp["Ls"] if inp.get("Ls") is not None else Lv, ec, br) if valid else np.zeros(4)
    wr = Lv[2] < 0
    sw = _n(T * Lv[0] + B * Lv[1] + N * Lv[2]) if valid else np.zeros(3)
    rej = (not wr) and sw @ gn < 0
    br.append(("rejected", rej))
    user = np.zeros(4)
    if inp.get("L") is not None:
        Lu = _n(np.array([inp["L"] @ T, inp["L"] @ B, inp["L"] @ N]))
        user = eval_bsdf(m, c, V, Lu, ec, br)
    out = dict(N=N, T=T, B=B, AX=m["Ax"], AY=m["Ay"], ETA=m["Eta"], PM=m["pm"], PD=m["pd"], PG=m["pg"], V=Vm, H=H, BSDF_L=Lv, BSDF_EVAL=ev,
               USER_EVAL=user, VALID=float(valid), REFRACTED=float(wr), ENTERED=float(wr and not inside), REJECTED=float(rej and valid), INSIDE=float(inside))
    out["eval"] = lambda Lt, b: eval_bsdf(m, c, V, Lt, ec, b)             # the BSDF of this hit at a tangent-space direction (NEE draws)
    out["GN"] = gn
    return out, br


FIELDS = dict(N=3, T=3, B=3, AX=1, AY=1, ETA=1, PM=1, PD=1, PG=1, V=3, H=3, BSDF_L=3, BSDF_EVAL=4, USER_EVAL=4)
FLAGS = ("VALID", "REFRACTED", "ENTERED", "REJECTED", "INSIDE")
# the surface frame and the material depend only on these branches: an output of that kind is checked whenever they are decided, the rest
# of a record only when every branch is
FRAME_BRANCHES = ("inside", "up", "bend1", "bend2")
FRAME_FIELDS = ("N", "T", "B", "AX", "AY", "ETA", "PM", "PD", "PG", "V")
PERTURBED = ("P", "Nv", "UV", "dir", "L", "Ls", "V")
MAT_SCALARS = ("BaseColor", "SpecularColor", "Roughness", "Metallic", "IOR", "Transmission", "Anisotropy", "AnisotropyRotation")


# ---------------------------------------------------------------- scenes and records
def _quad_mesh(tilt=0.0):
    v = np.zeros(6, gltf_ref.VERTEX_DTYPE)
    P = np.array([[-1, -1, 0], [1, -1, 0], [1, 1, 0], [-1, -1, 0], [1, 1, 0], [-1, 1, 0]], np.float32)
    v["pos"] = P
    nr = np.array([[tilt, -tilt, 1], [-tilt, 0.5 * tilt, 1], [0.3 * tilt, tilt, 1]] * 2, np.float32)
    v["nrm"] = nr / np.linalg.norm(nr, axis=1, keepdims=True)
    v["uv"] = (P[:, :2] + 1) / 2
    return v, np.arange(6, dtype=np.uint32)


TEX = {"white": np.full((1, 1, 4), 255, np.uint8), "normal": np.array([[[128, 128, 255, 255]]], np.uint8),
       "tilted": np.array([[[200, 90, 180, 255], [60, 170, 200, 255]], [[128, 40, 220, 255], [230, 200, 150, 255]]], np.uint8),
       "metal2x2": np.array([[[0], [255]], [[64], [191]]], np.uint8), "rough2x2": np.array([[[3], [255]], [[128], [40]]], np.uint8),
       "black": np.array([[[0, 0, 0, 255]]], np.uint8), "grey1": np.full((1, 1, 1), 200, np.uint8), "grey2": np.full((2, 2, 1), 200, np.uint8),
       "r1": np.full((1, 1, 1), 255, np.uint8), "base1": np.array([[[230, 120, 40, 255]]], np.uint8), "base2": np.tile(np.array([[[230, 120, 40, 255]]], np.uint8), (2, 2, 1))}
TEX_NAMES = list(TEX)


def _mat(**kw):
    m = np.zeros(1, gltf_ref.MATERIAL_DTYPE)[0]
    m["BaseColor"] = (0.8, 0.6, 0.4); m["SpecularColor"] = (1, 1, 1); m["Roughness"] = 0.5; m["IOR"] = 1.5
    tex = dict(BaseColorTextureIndex="white", NormalTextureIndex="normal", RoughnessTextureIndex="r1", MetallicTextureIndex="r1", EmissiveTextureIndex="white")
    for k, v in kw.items():
        if k in tex: tex[k] = v
        else: m[k] = v
    for k, v in tex.items(): m[k] = TEX_NAMES.index(v)
    return m


def material_groups():
    g = {}
    g["roughness"] = [_mat(Roughness=r, Metallic=mt) for r in (0, 1e-3, 0.05, 0.3, 0.7, 1) for mt in (0.0, 1.0)]
    g["anisotropy"] = [_mat(Roughness=0.4, Metallic=1.0, Anisotropy=a, AnisotropyRotation=d) for a in (0, 0.1, 0.5, 0.9, 1) for d in (0, 30, 90, -45, 360)]
    g["ior"] = [_mat(Roughness=r, Transmission=1.0, IOR=i) for i in (1.0, 1.0001, 1.33, 1.5, 1.515625, 1.53125, 2.0, 2.4, 3.0) for r in (0.05, 0.5)]
    g["lobes"] = [_mat(Roughness=0.35, Metallic=mt, Transmission=t, SpecularColor=(0.9, 0.5, 0.2)) for mt in (0, 0.25, 0.5, 0.999999, 1) for t in (0, 0.5, 1)]
    g["textures"] = [_mat(Roughness=0.6, Metallic=1.0, MetallicTextureIndex="metal2x2", RoughnessTextureIndex="rough2x2"),
                     _mat(Roughness=0.6, Transmission=0.5, MetallicTextureIndex="metal2x2"),
                     _mat(BaseColorTextureIndex="black", Roughness=0.3), _mat(NormalTextureIndex="tilted", Roughness=0.2, Metallic=0.5),
                     _mat(NormalTextureIndex="tilted", Roughness=0.3, Transmission=1.0, IOR=1.33)]
    return g


def scene_for(mats, tilt=0.25):
    """one quad per material, in a row; every third one mirrored, every fourth rotated"""
    inst = []
    for k in range(len(mats)):
        X = np.eye(4)
        if k % 3 == 1: X = np.diag([-1.0, 1, 1, 1])
        if k % 4 == 2: X = np.array([[0.0, 0, 1, 0], [0, 1, 0, 0], [-1, 0, 0, 0], [0, 0, 0, 1]]) @ np.diag([1.0, 2.0, 1, 1])
        X[:3, 3] = (3.0 * k, 0.5 * (k % 5), -0.25 * (k % 7))
        inst.append((np.asarray(X, np.float32).T.reshape(-1), 0, k))
    return {"meshes": [_quad_mesh(tilt)], "materials": np.array(mats), "textures": [TEX[n] for n in TEX_NAMES], "instances": inst,
            "camera_view": np.eye(4, dtype=np.float32).reshape(-1), "aspect": 1.0}


def records(sc, n_per, seed):
    """hits on every instance: random barycentrics, views from head-on to grazing, from both sides, random states, random extra L"""
    rng = np.random.default_rng(seed)
    R = dict(inst=[], prim=[], uv=[], dir=[], org=[], pdf=[], rng=[], L=[])
    for i, (xf, mi, _) in enumerate(sc["instances"]):
        M = np.asarray(xf, np.float64).reshape(4, 4).T
        gn = np.linalg.inv(M[:3, :3]).T @ np.array([0, 0, 1.0]); gn /= np.linalg.norm(gn)
        for j in range(n_per):
            u, v = rng.random(2) * 0.5
            cos = [1.0, 0.7, 0.3, 0.05, 0.003][j % 5] * (1 if j % 3 else -1)
            a = rng.normal(size=3); a -= (a @ gn) * gn; a /= np.linalg.norm(a)
            d = -(cos * gn + math.sqrt(1 - cos * cos) * a)
            L = rng.normal(size=3); L /= np.linalg.norm(L)
            R["inst"].append(i); R["prim"].append(j % 2); R["uv"].append((u, v)); R["dir"].append(d); R["org"].append(-d * 2.0)
            R["pdf"].append(0.5); R["rng"].append(int(rng.integers(0, 2 ** 32))); R["L"].append(L)
    return {k: np.array(v, np.float32 if k not in ("inst", "prim", "rng") else np.uint32) for k, v in R.items()}


def model_inputs(sc, R, i):
    xf, mi, mat = sc["instances"][R["inst"][i]]
    v, idx = sc["meshes"][mi]
    tri = idx[3 * R["prim"][i]: 3 * R["prim"][i] + 3]
    M = np.asarray(xf, np.float32).reshape(4, 4).T.astype(np.float64)
    m = sc["materials"][mat]
    t = sc["textures"]
    return dict(P=v["pos"][tri].astype(np.float64), Nv=v["nrm"][tri].astype(np.float64), UV=v["uv"][tri].astype(np.float64), W=np.linalg.inv(M[:3, :3]),
                u=float(R["uv"][i, 0]), v=float(R["uv"][i, 1]), dir=R["dir"][i].astype(np.float64), L=R["L"][i].astype(np.float64),
                mat={k: np.asarray(m[k], np.float64) for k in MAT_SCALARS}, tex_base=t[m["BaseColorTextureIndex"]], tex_normal=t[m["NormalTextureIndex"]],
                tex_rough=t[m["RoughnessTextureIndex"]], tex_metal=t[m["MetallicTextureIndex"]])


def _draws(state, rng=None):
    """the record's exact draws; with rng, each moved by a relative 2^-23 (the rounding of 2 pi u, sqrt(u) and the like downstream)"""
    while True:
        state, x = draw(state)
        yield x if rng is None else x * (1 + REL * rng.choice([-1.0, 1.0]))


def _perturbations(inp, rng):
    """NPERT perturbed copies of the inputs, in +/- pairs (a pair moves every input both ways, so it flips any branch within reach)"""
    out = []
    for _ in range(NPERT // 2):
        sg = {k: rng.choice([-1.0, 1.0], np.shape(inp[k])) for k in PERTURBED + ("u", "v") if inp.get(k) is not None}
        sm = {k: rng.choice([-1.0, 1.0], np.shape(v)) for k, v in inp["mat"].items()}
        for pm in (1.0, -1.0):
            q = dict(inp)
            for k, g in sg.items(): q[k] = inp[k] * (1 + pm * REL * g)
            q["mat"] = {k: v * (1 + pm * REL * sm[k]) for k, v in inp["mat"].items()}
            out.append(q)
    return out


def check_against_model(sc, R, got, cfg, k=K, label="", luts=None):
    """returns (records checked in full, undecided mask, failures); got: [n, STRIDE] records.  An undecided record still has its frame and
    material outputs checked when the frame branches are decided."""
    luts = luts or util.luts()
    rng = np.random.default_rng(7)
    checked = 0; undecided = np.zeros(len(R["inst"]), bool); fails = []
    for i in range(len(R["inst"])):
        inp = model_inputs(sc, R, i)
        inp["Ls"] = got[i, SQ["BSDF_L"]: SQ["BSDF_L"] + 3].astype(np.float64)
        inp["V"] = got[i, SQ["V"]: SQ["V"] + 3].astype(np.float64)
        ref, br = model_hit(inp, cfg, luts, _draws(int(R["rng"][i])))
        runs = [model_hit(q, cfg, luts, _draws(int(R["rng"][i]), rng)) for q in _perturbations(inp, rng)]
        frame_ok = all([x for x in b if x[0] in FRAME_BRANCHES] == [x for x in br if x[0] in FRAME_BRANCHES] for _, b in runs)
        if any(b != br for _, b in runs) or ref["V"][2] <= 0 or ("cancel", True) in br:
            undecided[i] = True
        else: checked += 1
        if not frame_ok: continue
        g = got[i]
        for f in FLAGS:
            if (not undecided[i] or f == "INSIDE") and g[SQ[f]] != ref[f]: fails.append((label, i, f, g[SQ[f]], ref[f]))
        for f, w in FIELDS.items():
            if undecided[i] and f not in FRAME_FIELDS: continue
            val = np.atleast_1d(ref[f]); gv = g[SQ[f]: SQ[f] + w].astype(np.float64)
            spread = max(np.abs(np.atleast_1d(o[f]) - val).max() for o, _ in runs)
            scale = np.abs(val).max()
            margin = k * spread + VALUE_ULPS * np.spacing(np.float32(scale))
            if not (np.all(np.isfinite(gv)) and np.abs(gv - val).max() <= margin):
                fails.append((label, i, f, gv.tolist(), val.tolist(), float(margin)))
    return checked, undecided, fails


MODEL_CFG = dict(EnableSkyMIS=0, EnableMeshMIS=0)
EC = (1, 0, 2)     # energy compensation on, off, and on with the refraction tables scaled by 0.015: their texels then straddle glassEC > 0.01


def _luts(ec):
    l = util.luts()
    return l if ec != 2 else (l[0], (l[1] * np.float32(0.015)).astype(np.float32), (l[2] * np.float32(0.015)).astype(np.float32))


def _oracle(sc, luts=None, **kw):
    raw, env_pdf, alias = util.env_small()
    S = orc.Scene(sc, env_pdf, alias, luts or util.luts())
    return S, orc.default_config(**kw)


def _threshold_records(sc, R, rec, before=2):
    """extra records whose x1 draw sits on pm, pm + pd (and one fp32 ulp either side) and on exactly 1.0 (Q12); rec: the records' first results;
    before: the draws ahead of x1 (the two VNDF draws, and the three sky draws when sky MIS is on)"""
    extra = {k: [] for k in R}
    for i in range(0, len(R["inst"]), 3):
        pm, pd = float(rec[i, SQ["PM"]]), float(rec[i, SQ["PD"]])
        for t in (pm, pm + pd):
            for x in (np.nextafter(np.float32(t), np.float32(0)), np.float32(t), np.nextafter(np.float32(t), np.float32(2))):
                if 2.0 ** -9 <= x <= 1.0:
                    for k2 in R: extra[k2].append(R[k2][i])
                    extra["rng"][-1] = state_for_draw(float(x), before)
        for k2 in R: extra[k2].append(R[k2][i])
        extra["rng"][-1] = state_for_draw(1.0, before)
    return {k: np.concatenate([R[k], np.array(extra[k], R[k].dtype)]) for k in R}


GROUPS = sorted(material_groups())


@pytest.mark.parametrize("ec", EC)
@pytest.mark.parametrize("group", GROUPS)
def test_oracle_matches_float64_model(group, ec):
    """CPU only: the oracle's shading step against the float64 model, on every material group.  Validates the model and the margins."""
    sc = scene_for(material_groups()[group])
    R = records(sc, 10, 3); nb = len(R["inst"])
    S, cfg = _oracle(sc, _luts(ec), UseEnergyCompensation=int(ec != 0), **MODEL_CFG)
    R = _threshold_records(sc, R, S.shade_query(cfg, R["inst"], R["prim"], R["uv"], R["dir"], R["org"], R["pdf"], R["rng"], R["L"]))
    got = S.shade_query(cfg, R["inst"], R["prim"], R["uv"], R["dir"], R["org"], R["pdf"], R["rng"], R["L"])
    checked, und, fails = check_against_model(sc, R, got, dict(geo=False, ec=bool(ec)), label=group, luts=_luts(ec))
    print(f"oracle vs model {group} ec={ec}: {checked} of {len(und)} checked, undecided share {und[:nb].mean():.3f} (threshold records {und[nb:].mean():.3f})")
    assert not fails, fails[:5]
    assert und[:nb].mean() <= UNDECIDED_MAX, und[:nb].mean()


# ---------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def pt():
    import torch
    if not torch.cuda.is_available(): pytest.skip("no CUDA device")
    import vpt_b200
    return vpt_b200


def _tracer(pt, sc, luts=None, **kw):
    raw, env_pdf, alias = util.env_small()
    T = pt.PathTracer(0)
    T.set_scene(sc); T.set_env_map(raw); T.set_luts(*(luts or util.luts()))
    c = pt.default_config()
    for k, v in kw.items(): setattr(c, k, v)
    T.set_config(c)
    return T


def _q(T, R, **kw):
    return T.shade_query(R["inst"], R["prim"], R["uv"], R["dir"], R["org"], R["pdf"], R["rng"], R["L"], **kw)


def test_shade_record_layout_matches_headers():
    """the offsets the binding and this module use are the B200PT_SQ_* of the C header and the ORC_SQ_* of the oracle, with the world-space
    NEE fields (shading position, sky and light directions) after the class"""
    import re
    import vpt_b200
    hdr = open(f"{util.ROOT}/include/b200pt.h").read()
    assert {m.group(1): int(m.group(2)) for m in re.finditer(r"#define B200PT_SQ_(\w+)\s+(\d+)", hdr)} == SQ == vpt_b200.SQ
    ohdr = open(f"{util.ROOT}/oracle/pt_oracle.h").read()
    assert {m.group(1): int(m.group(2)) for m in re.finditer(r"#define ORC_SQ_(\w+)\s+(\d+)", ohdr)} == SQ
    assert (SQ["POS"], SQ["SKY_W"], SQ["LIGHT_W"], SQ["STRIDE"]) == (SQ["CLASS"] + 1, SQ["CLASS"] + 4, SQ["CLASS"] + 7, SQ["CLASS"] + 10)


BITS = (SQ["LIGHT_GID"], SQ["RNG"], SQ["CLASS"])                          # u32 fields of the record
FLAG_FIELDS = ("VALID", "REFRACTED", "ENTERED", "REJECTED", "INSIDE")
# BSDF_EVAL / SAMPLE (the BSDF at the sampled direction) are left to the model, which evaluates them at each implementation's own fp32 L: next
# to a near-specular lobe the rounding of L alone moves D by tens of per cent, so two implementations need not agree there.
VALUE_FIELDS = ("N", "T", "B", "NG", "AX", "AY", "ETA", "PM", "PD", "PG", "BASECOLOR", "ROUGHNESS", "V", "H", "EMITTED", "SKY_L", "SKY_LV", "SKY_EVAL", "SKY_C",
                "LIGHT_L", "LIGHT_LV", "LIGHT_EVAL", "LIGHT_C", "BSDF_L", "SCATTER", "USER_EVAL")
WIDTH = {f: (SQ[n] - SQ[f]) for f, n in zip(sorted(SQ, key=SQ.get), sorted(SQ, key=SQ.get)[1:])}


def _gpu_vs_oracle(got, ref, rtol=2e-3, fields=VALUE_FIELDS):
    """same draws (final states equal), equal flags, the same fields non-finite, and finite values within rtol of the record's scale where
    the record took the same path"""
    same = got[:, SQ["RNG"]].view(np.uint32) == ref[:, SQ["RNG"]].view(np.uint32)
    same &= got[:, SQ["LIGHT_GID"]].view(np.uint32) == ref[:, SQ["LIGHT_GID"]].view(np.uint32)
    for f in FLAG_FIELDS: same &= got[:, SQ[f]] == ref[:, SQ[f]]
    # a value the reference computes as inf / NaN must be inf / NaN here too (a finite one keeps a path the reference drops), in every field,
    # including those whose finite values are left to the model
    vals = [k for k in range(SQ["STRIDE"]) if k not in BITS]
    bad = [("finiteness", int(j), np.flatnonzero(np.isfinite(got[j, vals]) != np.isfinite(ref[j, vals])).tolist())
           for j in np.flatnonzero(same & np.any(np.isfinite(got[:, vals]) != np.isfinite(ref[:, vals]), axis=1))]
    for f in fields:
        a, b = got[same, SQ[f]: SQ[f] + WIDTH[f]].astype(np.float64), ref[same, SQ[f]: SQ[f] + WIDTH[f]].astype(np.float64)
        fin = np.isfinite(b).all(1)
        scale = np.maximum(np.abs(b).max(1, keepdims=True), 1e-6)
        err = (np.abs(a - b) / scale).max(1)
        bad += [(f, int(np.flatnonzero(same)[j]), a[j].tolist(), b[j].tolist()) for j in np.flatnonzero(fin & ~(err <= rtol))]
    return same.mean(), bad


@pytest.mark.gpu
@pytest.mark.parametrize("ec", EC)
@pytest.mark.parametrize("group", GROUPS)
def test_gpu_matches_oracle_and_model(pt, group, ec):
    sc = scene_for(material_groups()[group])
    R = records(sc, 10, 3); nb = len(R["inst"])
    S, cfg = _oracle(sc, _luts(ec), UseEnergyCompensation=int(ec != 0), **MODEL_CFG)
    R = _threshold_records(sc, R, S.shade_query(cfg, R["inst"], R["prim"], R["uv"], R["dir"], R["org"], R["pdf"], R["rng"], R["L"]))
    ref = S.shade_query(cfg, R["inst"], R["prim"], R["uv"], R["dir"], R["org"], R["pdf"], R["rng"], R["L"])
    T = _tracer(pt, sc, _luts(ec), UseEnergyCompensation=int(ec != 0), **MODEL_CFG)
    got = _q(T, R)
    checked, und, fails = check_against_model(sc, R, got, dict(geo=False, ec=bool(ec)), label=group, luts=_luts(ec))
    agree, bad = _gpu_vs_oracle(got, ref, fields=tuple(f for f in VALUE_FIELDS if f != "USER_EVAL"))   # the model checks it on each side's own V
    print(f"GPU vs model {group} ec={ec}: {checked} of {len(und)} checked, undecided share {und[:nb].mean():.3f}; GPU vs oracle: same path {agree:.4f}")
    assert not fails, fails[:5]
    assert und[:nb].mean() <= UNDECIDED_MAX, und[:nb].mean()
    assert agree >= 0.97 and not bad, (agree, bad[:5])


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(EnableSkyMIS=0), dict(EnableMeshMIS=0), dict(UseOnlyGeometryNormals=1)])
def test_cornell_hits_with_nee_match_oracle(pt, kw):
    """Cornell with its lights, both NEE samplers and the emission MIS term: every hit of random rays, GPU against oracle"""
    name = "cornell_box"
    S = util.oracle_scene(name)
    o, d = (np.random.default_rng(5).normal(size=(4000, 3)) * 0.3).astype(np.float32), np.random.default_rng(6).normal(size=(4000, 3))
    d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    t, prim, inst, uv = S.trace_closest(o, d, 1e-3, 1e5)
    h = t > 0
    R = dict(inst=inst[h], prim=prim[h], uv=uv[h], dir=d[h], org=o[h], pdf=np.full(h.sum(), 0.7, np.float32),
             rng=np.random.default_rng(8).integers(0, 2 ** 32, h.sum(), dtype=np.uint64).astype(np.uint32), L=-d[h])
    cfg = util.oracle_config(name, **kw)
    ref = S.shade_query(cfg, R["inst"], R["prim"], R["uv"], R["dir"], R["org"], R["pdf"], R["rng"], R["L"])
    T = util.product_tracer(name, 8, 8, **kw)
    got = _q(T, R)
    agree, bad = _gpu_vs_oracle(got, ref)
    print(f"cornell NEE {kw}: {h.sum()} hits, same path {agree:.4f}")
    assert h.sum() > 1000 and agree >= 0.99 and not bad, (agree, bad[:5])


def _adversarial(sc, n_per=12):
    """views within a few ulps of the surface after the bend; roughness 0 (Ax = Ay = 1e-5) comes with the materials"""
    R = records(sc, n_per, 11)
    rng = np.random.default_rng(12)
    for i in range(0, len(R["inst"]), 4): R["dir"][i] = R["dir"][i] + np.float32(1e-6) * rng.normal(size=3).astype(np.float32)
    return R


def _adversarial_L(R, rec):
    """each record four more times, its extra L built in the tangent frame the first query returned (rec), for that hit's Eta:
    L = -V (the shortest V Eta + L a unit L allows: |Eta - 1|), (V Eta + L).z = 0 (the half vector's H.z < 0 flip), L just below the surface
    (L.z = -1e-7) and L.z exactly at the 1e-5 reflection cut"""
    out = {k: [] for k in R}
    for i in range(len(R["inst"])):
        T, B, N = (rec[i, SQ[f]: SQ[f] + 3].astype(np.float64) for f in ("T", "B", "N"))
        V, eta = rec[i, SQ["V"]: SQ["V"] + 3].astype(np.float64), float(rec[i, SQ["ETA"]])
        xy = -V[:2] / max(np.linalg.norm(V[:2]), 1e-12)
        cands = [-V]
        z = -eta * V[2]
        if abs(z) < 1: cands.append(np.array([*(xy * math.sqrt(1 - z * z)), z]))
        for z in (-1e-7, 1e-5): cands.append(np.array([*(xy * math.sqrt(1 - z * z)), z]))
        for Lt in cands:
            for k in R: out[k].append(R[k][i])
            out["L"][-1] = (T * Lt[0] + B * Lt[1] + N * Lt[2]).astype(np.float32)
    return {k: np.concatenate([R[k], np.array(out[k], R[k].dtype)]) for k in R}


def _nth_draw(state, n):
    for _ in range(n): state, x = draw(state)
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("sky", [0, 1])
@pytest.mark.parametrize("group", GROUPS)
def test_class_kernels_equal_the_general_kernel(pt, group, sky):
    """k_shade_hit<MC_DIFFUSE / MC_METAL / MC_GLASS> drops lobes whose probability is exactly 0.  The renderer must not keep a path the
    reference drops: wherever a class kernel's answer is finite, the all-lobes kernel's must be too; and where both are finite they agree to
    rounding (two instantiations may contract an a*b+c differently).  x1 == 1.0 records (Q12) send diffuse and metal hits down the glass
    branch; with sky MIS on, the sky draw also evaluates directions below the surface in every class."""
    mats = material_groups()[group] + [_mat(Roughness=0.0, Metallic=1.0), _mat(Roughness=0.0, Transmission=1.0, IOR=1.5), _mat(Roughness=0.0)]
    sc = scene_for(mats)
    T = _tracer(pt, sc, EnableSkyMIS=sky, EnableMeshMIS=0)
    R = _adversarial(sc)
    R = _adversarial_L(R, _q(T, R, force_general=True))
    before = 2 + 3 * sky                                                    # VNDF draws, then the sky draws ahead of them
    R = _threshold_records(sc, R, _q(T, R, force_general=True), before)
    cls, gen = _q(T, R), _q(T, R, force_general=True)
    pure = cls[:, SQ["CLASS"]] != 3
    x1_one = np.array([_nth_draw(int(s), before + 1) == 1.0 for s in R["rng"]])
    glass_branch = pure & x1_one & (cls[:, SQ["CLASS"]] != 2)
    assert glass_branch.any(), "no diffuse or metal class record with x1 == 1.0"
    vals = [k for k in range(SQ["STRIDE"]) if k not in BITS]
    fin_g, fin_c = np.isfinite(gen[:, vals]).all(1), np.isfinite(cls[:, vals]).all(1)
    ident = np.all(cls[:, :SQ["CLASS"]].view(np.uint32) == gen[:, :SQ["CLASS"]].view(np.uint32), axis=1)
    print(f"class vs general {group} sky={sky}: {pure.sum()} class records ({glass_branch.sum()} diffuse / metal with x1 == 1), "
          f"{(pure & ~fin_g).sum()} non-finite in the general kernel, bit-identical {ident[pure & fin_g].mean():.4f}")
    assert not (pure & fin_c & ~fin_g).any(), "the general kernel is non-finite where a class kernel is finite: the renderer keeps a path the reference drops"
    c, g = cls[pure & fin_g], gen[pure & fin_g]
    agree, bad = _gpu_vs_oracle(c, g, rtol=1e-5, fields=tuple(f for f in VALUE_FIELDS if f != "USER_EVAL"))
    # the BSDF at a direction is compared where both kernels evaluated it at the same bits of L: the adversarial directions sit on the
    # L.z <= 1e-5 cut and next to L.z = 0, where a last-bit difference in L (contraction in world_to_tangent) legitimately flips a branch
    for L_f, E_f in (("BSDF_L", "BSDF_EVAL"), ("USER_L", "USER_EVAL")):
        sameL = np.all(c[:, SQ[L_f]: SQ[L_f] + 3].view(np.uint32) == g[:, SQ[L_f]: SQ[L_f] + 3].view(np.uint32), axis=1)
        ev = lambda a: a[sameL, SQ[E_f]: SQ[E_f] + 4].astype(np.float64)
        err = np.abs(ev(c) - ev(g)).max(1) / np.maximum(np.abs(ev(g)).max(1), 1e-6)
        print(f"  {E_f}: same L on {sameL.mean():.4f} of the records, largest relative difference there {err.max() if len(err) else 0:.2e}")
        bad += [(E_f, int(j), ev(c)[k].tolist(), ev(g)[k].tolist()) for k, j in enumerate(np.flatnonzero(sameL)) if not err[k] <= 1e-6]
    assert agree >= 0.99 and not bad, (agree, bad[:5])


@pytest.mark.gpu
def test_per_material_precompute_equals_per_hit_texels(pt):
    """1x1 textures take the per-material results of k_prepare_materials; uniform 2x2 textures of the same texels go through the per-hit path"""
    mats1 = [_mat(Roughness=r, Metallic=mt, Transmission=t, Anisotropy=a, BaseColorTextureIndex="base1", RoughnessTextureIndex="grey1", MetallicTextureIndex="grey1")
             for r, mt, t, a in ((0.3, 1.0, 0, 0.5), (0.5, 0.4, 0.3, 0.1), (0.05, 0, 1, 0), (0.7, 0, 0, 0.9))]
    mats2 = [_mat(**{k: m[k] for k in MAT_SCALARS}, BaseColorTextureIndex="base2", RoughnessTextureIndex="grey2", MetallicTextureIndex="grey2") for m in mats1]
    s1, s2 = scene_for(mats1), scene_for(mats2)
    R = records(s1, 20, 4)
    # the general instantiation in both: a 2x2 metallic texture makes the class MC_GENERAL whatever its texels, and two instantiations may
    # contract an a*b+c differently
    a = _q(_tracer(pt, s1), R, force_general=True); b = _q(_tracer(pt, s2), R, force_general=True)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), np.flatnonzero((a.view(np.uint32) != b.view(np.uint32)).any(0))


@pytest.mark.gpu
def test_margin_is_tight(pt):
    """K / 10 rejects some GPU answer on the adversarial records, so K is not loose by an order of magnitude"""
    fails = 0
    for group in ("anisotropy", "ior"):
        sc = scene_for(material_groups()[group])
        R = _adversarial(sc, 6)
        got = _q(_tracer(pt, sc, **MODEL_CFG), R)
        fails += len(check_against_model(sc, R, got, dict(geo=False, ec=True), k=K / 10)[2])
    assert fails > 0


@pytest.mark.gpu
def test_shade_query_refuses_bad_input(pt):
    sc = scene_for([_mat()])
    T = _tracer(pt, sc)
    R = records(sc, 2, 1)
    with pytest.raises(pt.B200ptError): T.shade_query(R["inst"] + 5, R["prim"], R["uv"], R["dir"], R["org"], R["pdf"], R["rng"])
    with pytest.raises(pt.B200ptError): T.shade_query(R["inst"], R["prim"] + 2, R["uv"], R["dir"], R["org"], R["pdf"], R["rng"])
    T.add_volume()
    with pytest.raises(pt.B200ptError): T.shade_query(R["inst"], R["prim"], R["uv"], R["dir"], R["org"], R["pdf"], R["rng"])
