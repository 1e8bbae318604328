"""The post chain pixel by pixel: HDR accumulate (k_accumulate), bloom (k_bloom_down_first, k_bloom_down, k_bloom_up, k_bloom_final and the
pass-per-pass k_bloom_threshold / k_tonemap) and the RGBA8 tonemap, against the CPU oracle (orc_post_process) and a float64 model, on tiny and
odd images, every MipCount, parameter edges, row blocks and extreme inputs.

Model (numpy float64, restating PostProcessor.cpp:128-246 and BloomDownSample / BloomUpSample / Tonemap.slang):
  mip sizes: halve (odd sizes rounded down first) while both stay >= 2, at most 10 levels; MipCount clamped to [1, levels];
  mip 0 = HDR * smoothstep(T - F, T + F, luminance) with the luminance and the smoothstep's numerator and denominator taken in fp32 (both
      implementations round them alike, so the model knows them exactly: a texel placed on a threshold stays on it);
  down pass i: taps 2xy + (a, b), a, b in [-2, 1], clamped, sum / 25 * strength (Q14);
  up pass i: taps xy / 2 + (a, b) + 1, clamped, sum / 25 * strength, added to mip i-1 in place;
  the bloom fetch: bilinear, CLAMP_TO_EDGE, uv = xy / size, so texels x-1 and x (clamped) at weight 1/2 each (Q15);
  (HDR + bloom) * exposure, pow(., 1 / gamma) with pow(0, y) = 0 and pow(x < 0, y) = NaN, the ACES fit, then the RGBA8 store: saturate
  (NaN -> 0), * 255, round half to even.

Margins are forward error bounds of the fp32 operations the GPU runs, carried with every model value (class E):
  every rounded +, -, *: u = 2^-24 of the result, plus 2^-149 absolute for subnormal results; the sums in the oracle's tap order;
  division (-prec-div=false): 2 ulp = 2^-22 relative;
  pow (exp2f(y * __log2f(x))): __log2f within 2^-22 absolute on [0.5, 2] and 2^-22 relative elsewhere (PTX ISA lg2.approx.f32), the
      product rounded, exp2f within 2 ulp; 1 / gamma is a 2-ulp division; the input error goes through pow as an interval;
  aces_fitted: compiled with free FMA contraction, which only removes roundings, so the unfused bound covers it;
  the bilinear weight: u = x / W (2 ulp), u * W and - 0.5 rounded: |ax - 1/2| <= 7u * x.
The oracle (IEEE division, glibc powf, no contraction) lies inside the same bounds.  A channel passes when |got - model| <= K * bound; an
LDR byte is *decided* when the model's q * 255 +- K * bound (clamped to [0, 255]) holds no rounding boundary k + 1/2, and must then equal
the model's byte exactly; an undecided byte may take either neighbour.  Undecided shares are printed per case and bounded by UNDECIDED_MAX.

Non-finite and overflowing inputs (+-Inf, NaN, 3e38, whose tap sums overflow) are compared with the oracle instead: the finite / Inf / NaN
class of every bloom channel must match, the LDR image must match exactly, and every pixel whose dependency footprint misses the bad texels
must equal the run on the clean image bit for bit.

Dependency model: output row y reads HDR row y and post-up mip-0 rows y-1, y; post-up row y of mip i-1 reads its own down row and post-up
rows y/2 - 1 .. y/2 + 2 of mip i; down row y of mip i reads rows 2y - 2 .. 2y + 1 of mip i-1 (all clamped).  Rows and columns are independent,
so boolean matrices composed pass by pass give the exact HDR rows (and columns) of every output row (column).
"""
import functools

import numpy as np
import pytest

import util
from util import orc

K = 1.0
UNDECIDED_MAX = 0.4
U = 2.0 ** -24
DIV = 2.0 ** -22                 # 2 ulp, relative
TINY = 2.0 ** -149               # absolute rounding error of a subnormal result
F32 = lambda v: float(np.float32(v))
ACES_IN = np.array([[0.59719, 0.35458, 0.04823], [0.07600, 0.90834, 0.01566], [0.02840, 0.13383, 0.83777]], np.float32).astype(np.float64)
ACES_OUT = np.array([[1.60475, -0.53108, -0.07367], [-0.10208, 1.10813, -0.00605], [-0.00327, -0.07276, 1.07602]], np.float32).astype(np.float64)
LUMA = (np.float32(0.2126), np.float32(0.7152), np.float32(0.0722))
DEFAULTS = dict(Exposure=1.0, Gamma=2.2, BloomThreshold=2.0, BloomStrength=1.0, FalloffRange=5.0, MipCount=10)


# ---------------------------------------------------------------- float64 values with a forward error bound
class E:
    __slots__ = ("v", "e")

    def __init__(self, v, e=0.0):
        self.v = np.asarray(v, np.float64); self.e = np.broadcast_to(np.asarray(e, np.float64), self.v.shape).copy()

    @staticmethod
    def _r(v, e, rel=U):         # the result rounded to fp32 (an exact zero stays exact)
        m = np.abs(v) + e
        return E(v, e + rel * m + np.where((m < 2.0 ** -126) & (m > 0), TINY, 0.0))

    def __add__(a, b):
        b = b if isinstance(b, E) else E(b)
        return E._r(a.v + b.v, a.e + b.e)

    def __sub__(a, b):
        b = b if isinstance(b, E) else E(b)
        return E._r(a.v - b.v, a.e + b.e)

    def __mul__(a, b):
        b = b if isinstance(b, E) else E(b)
        return E._r(a.v * b.v, np.abs(a.v) * b.e + np.abs(b.v) * a.e + a.e * b.e)

    def div(a, b):
        b = b if isinstance(b, E) else E(b)
        q = a.v / b.v
        return E._r(q, (a.e + np.abs(q) * b.e) / np.maximum(np.abs(b.v) - b.e, 1e-300), DIV)

    def clamp01(a):
        return E(np.fmin(np.fmax(a.v, 0.0), 1.0), np.where(np.isnan(a.v), 0.0, a.e))     # fminf(fmaxf(NaN, 0), 1) = 0 exactly


def mip_sizes(W, H):
    """PostProcessor.cpp:128-158"""
    out, w, h = [], W, H
    for _ in range(10):
        out.append((w, h))
        w, h = (w - w % 2) // 2, (h - h % 2) // 2
        if w < 2 or h < 2: break
    return out


def mip_count(p, W, H):
    return min(max(int(p["MipCount"]), 1), len(mip_sizes(W, H)))     # PostProcessor.cpp:195


def threshold_factor(rgb32, p):
    """smoothstep(T - F, T + F, luminance): luminance, x - e0 and e1 - e0 in fp32 (exact), the division and the polynomial carried"""
    T, Fr = np.float32(p["BloomThreshold"]), np.float32(p["FalloffRange"])
    e0, e1 = np.float32(T - Fr), np.float32(T + Fr)
    with np.errstate(all="ignore"):
        br = (rgb32[..., 0] * LUMA[0] + rgb32[..., 1] * LUMA[1]) + rgb32[..., 2] * LUMA[2]
        num, den = (br - e0).astype(np.float64), float(np.float32(e1 - e0))
        if den == 0.0:                                                        # x / 0: +-inf, 0 / 0: NaN -> clamp's lower bound (DESIGN Q18)
            t = E(np.where(num > 0, 1.0, 0.0))
        else:
            t = E(num).div(E(den)).clamp01()
    return (t * t) * (E(3.0) - E(2.0) * t)


def _taps(n_src, idx, off):
    return np.clip(idx + off, 0, n_src - 1)


def _tap_sum(src, ys, xs):
    """16 taps, a (x offset) outer, b (y offset) inner, summed in that order; ys / xs: lists of 4 index arrays for b, a = -2..1"""
    acc = None
    for ax in xs:
        for by in ys:
            t = E(src.v[by[:, None], ax[None, :]], src.e[by[:, None], ax[None, :]])
            acc = t if acc is None else acc + t
    return acc


def bloom_scale(acc, strength):
    return acc.div(E(25.0)) * E(F32(strength))


def model_chain(hdr, p):
    """-> (mip 0 after the up passes: E [H, W, 3], LDR bytes [H, W, 3] uint8, decided [H, W, 3] bool) at margin K = 1 (scale .e for others)"""
    H, W = hdr.shape[:2]
    sizes = mip_sizes(W, H); n = mip_count(p, W, H)
    rgb32 = hdr[..., :3].astype(np.float32)
    f = threshold_factor(rgb32, p)
    mips = [E(rgb32.astype(np.float64)) * E(f.v[..., None], f.e[..., None])]
    for i in range(1, n):
        (iw, ih), (ow, oh) = sizes[i - 1], sizes[i]
        ys = [_taps(ih, 2 * np.arange(oh), b) for b in range(-2, 2)]; xs = [_taps(iw, 2 * np.arange(ow), a) for a in range(-2, 2)]
        mips.append(bloom_scale(_tap_sum(mips[-1], ys, xs), p["BloomStrength"]))
    for i in range(n - 1, 0, -1):
        (iw, ih), (ow, oh) = sizes[i], sizes[i - 1]
        ys = [_taps(ih, np.arange(oh) // 2 + 1, b) for b in range(-2, 2)]; xs = [_taps(iw, np.arange(ow) // 2 + 1, a) for a in range(-2, 2)]
        mips[i - 1] = bloom_scale(_tap_sum(mips[i], ys, xs), p["BloomStrength"]) + mips[i - 1]
    b0 = mips[0]
    return b0, tonemap(rgb32.astype(np.float64), b0, p)


def _mix(pv, qv, w_dev):
    """p + w (q - p), w = 1/2 +- w_dev"""
    d = qv - pv
    wd = E._r(0.5 * d.v, 0.5 * d.e + w_dev * (np.abs(d.v) + d.e))
    return pv + wd


def bloom_fetch(b0):
    H, W = b0.v.shape[:2]
    y0, y1 = np.clip(np.arange(H) - 1, 0, H - 1), np.arange(H)
    x0, x1 = np.clip(np.arange(W) - 1, 0, W - 1), np.arange(W)
    g = lambda yy, xx: E(b0.v[yy[:, None], xx[None, :]], b0.e[yy[:, None], xx[None, :]])
    ax = (7 * U * np.arange(W))[None, :, None]; ay = (7 * U * np.arange(H))[:, None, None]
    return _mix(_mix(g(y0, x0), g(y0, x1), ax), _mix(g(y1, x0), g(y1, x1), ax), ay)


def post_pow(c, gamma):
    """exp2(y * __log2f(x)), y = 1 / gamma (2-ulp division); x < 0 -> NaN, x == 0 -> 0; the input error as an interval"""
    y = 1.0 / F32(gamma); ey = DIV * abs(y)
    with np.errstate(all="ignore"):
        pos = c.v > 0
        lo, hi = np.maximum(c.v - c.e, 0.0), c.v + c.e
        pv = np.where(pos, np.abs(c.v) ** y, np.where(c.v == 0, 0.0, np.nan))
        e_in = np.maximum(np.abs(hi ** y - pv), np.abs(pv - lo ** y))
        lg = np.log2(np.where(pos, c.v, 1.0))
        e_lg = 2.0 ** -22 * np.where((c.v >= 0.5) & (c.v <= 2.0), 1.0, np.abs(lg))
        z = y * lg
        ez = ey * np.abs(lg) + abs(y) * e_lg + U * np.abs(z)
        e = e_in + (pv + e_in) * (np.expm1(ez * np.log(2.0)) + DIV) + TINY
    e = np.where(pos, e, np.where(c.v == 0, 0.0, 0.0))
    return E(pv, e), (np.abs(c.v) <= c.e) & (c.e > 0)      # second: the sign of x is not decided


def aces(c):
    """Tonemap.slang:20-55 on E [..., 3]"""
    ch = [E(c.v[..., k], c.e[..., k]) for k in range(3)]
    dot = lambda M, k, x: (x[0] * E(M[k, 0]) + x[1] * E(M[k, 1])) + x[2] * E(M[k, 2])
    v = [dot(ACES_IN, k, ch) for k in range(3)]
    r = []
    for vk in v:
        a = vk * (vk + E(F32(0.0245786))) - E(F32(0.000090537))
        b = vk * (E(F32(0.983729)) * vk + E(F32(0.4329510))) + E(F32(0.238081))
        r.append(a.div(b))
    out = [dot(ACES_OUT, k, r).clamp01() for k in range(3)]
    return E(np.stack([o.v for o in out], -1), np.stack([o.e for o in out], -1))


def tonemap(h, b0, p):
    """-> (q E [H, W, 3] in [0, 1] or NaN, sign_undecided [H, W])"""
    bl = bloom_fetch(b0)
    c = (E(h) + bl) * E(F32(p["Exposure"]))
    pw, undec = post_pow(c, p["Gamma"])
    with np.errstate(all="ignore"):
        q = aces(pw)
    return q, undec.any(-1)


def ldr_of(q, undec, k=K):
    """model bytes and decided mask: q * 255 (rounded), the margin k * bound, boundaries at k + 1/2"""
    v = np.nan_to_num(q.v, nan=0.0) * 255.0
    e = k * q.e * 255.0 + U * 255.0
    nanpix = np.isnan(q.v).any(-1)                       # a NaN channel reaches all three through the ACES matrices: bytes 0
    e = np.where(nanpix[..., None], 0.0, e)
    byte = np.rint(np.clip(v, 0, 255)).astype(np.uint8)
    lo, hi = np.clip(v - e, 0, 255), np.clip(v + e, 0, 255)
    decided = (np.floor(lo + 0.5) == np.floor(hi + 0.5)) & ~undec[..., None]
    byte[nanpix] = 0
    return byte, decided


def check(hdr, p, bloom, ldr, k=K):
    """-> (bad bloom channels, bad decided bytes, undecided share, pixels where the byte is off by more than one)"""
    b0, (q, undec) = model_chain(hdr, p)
    bad_b = ~(np.abs(bloom[..., :3].astype(np.float64) - b0.v) <= k * b0.e)
    mb, dec = ldr_of(q, undec, k)
    got = ldr[..., :3]
    bad_l = dec & (got != mb)
    far = np.abs(got.astype(int) - mb.astype(int)) > 1
    return bad_b, bad_l, 1.0 - dec.mean(), far


# ---------------------------------------------------------------- cases
def _lognormal(W, H, seed):
    rng = np.random.default_rng(seed)
    hdr = np.ones((H, W, 4), np.float32); hdr[..., :3] = (np.exp(rng.normal(0, 1.5, (H, W, 3))) * 0.5).astype(np.float32)
    return hdr


def _hot(W, H, seed):
    """log-normal noise with hot blocks on the corners, the edges and the tile seams (columns 31 / 32 / 33, rows 7 / 8 / 9 and doubles)"""
    hdr = _lognormal(W, H, seed)
    for y in {0, H - 1, 7, 8, 9, 16, 17, 18, H // 2}:
        for x in {0, W - 1, 31, 32, 33, 64, 65, 66, W // 2}:
            if y < H and x < W: hdr[y, x, :3] = (400.0, 300.0, 500.0)
    return hdr


def _input(kind, W, H, p):
    if kind == "lognormal": return _lognormal(W, H, W * 131 + H)
    if kind == "hot": return _hot(W, H, W * 7 + H)
    if kind == "zero": return np.zeros((H, W, 4), np.float32)
    if kind == "constant": hdr = np.ones((H, W, 4), np.float32); hdr[..., :3] = 3.25; return hdr
    if kind == "denormal":
        hdr = _lognormal(W, H, 5); hdr[::3, :, :3] = np.float32(1e-40); hdr[1::5, ::2, 1] = np.float32(-3e-42); return hdr
    if kind == "negative":
        hdr = _lognormal(W, H, 6); hdr[..., :3] -= np.float32(0.8); return hdr
    if kind in ("on_threshold", "on_start_end"):
        # texels whose fp32 luminance equals the threshold (or start / end) exactly: luminance is computed as the implementations do
        hdr = _hot(W, H, 8)
        T, Fr = np.float32(p["BloomThreshold"]), np.float32(p["FalloffRange"])
        targets = [T] if kind == "on_threshold" else [np.float32(T - Fr), np.float32(T + Fr)]
        rng = np.random.default_rng(9)
        for y in range(H):
            for x in range(W):
                if (x + y) % 2: continue
                tgt = targets[(x // 2 + y) % len(targets)]
                g = np.float32(tgt)                                 # grey: search the fp32 neighbourhood for a luminance exactly on target
                for cand in (g + np.float32(d) * np.spacing(g) for d in rng.permutation(np.arange(-8, 9))):
                    rgb = np.full(3, cand, np.float32)
                    if (rgb[0] * LUMA[0] + rgb[1] * LUMA[1]) + rgb[2] * LUMA[2] == tgt:
                        hdr[y, x, :3] = rgb; break
        return hdr
    raise KeyError(kind)


SIZES = [(1, 1), (1, 37), (37, 1), (2, 2), (3, 3), (4, 4), (5, 3), (31, 7), (32, 8), (33, 9), (63, 17), (65, 15), (8, 8), (1023, 767), (317, 203)]


def _cases():
    out = {}
    for W, H in SIZES:
        out[f"{W}x{H}"] = (W, H, "hot", {})
    for W, H in ((63, 17), (317, 203)):
        L = len(mip_sizes(W, H))
        for m in sorted({0, 1, 2, 3, L - 1, L, 11}):
            out[f"{W}x{H}-mips{m}"] = (W, H, "hot", dict(MipCount=m))
    params = {"falloff0": dict(FalloffRange=0.0), "strength0": dict(BloomStrength=0.0), "thr0": dict(BloomThreshold=0.0),
              "thr-1": dict(BloomThreshold=-1.0), "exposure0": dict(Exposure=0.0), "gamma1": dict(Gamma=1.0), "gamma0.5": dict(Gamma=0.5),
              "gamma4": dict(Gamma=4.0)}
    for name, kw in params.items():
        out[f"65x15-{name}"] = (65, 15, "hot", kw)
    out["65x15-falloff0-on-threshold"] = (65, 15, "on_threshold", dict(FalloffRange=0.0, MipCount=3))
    out["65x15-falloff0-on-threshold-fused"] = (65, 15, "on_threshold", dict(FalloffRange=0.0))
    out["65x15-on-threshold"] = (65, 15, "on_threshold", dict(BloomThreshold=3.0, FalloffRange=0.5))
    out["65x15-on-start-end"] = (65, 15, "on_start_end", dict(BloomThreshold=3.0, FalloffRange=1.5))
    for kind in ("lognormal", "zero", "constant", "denormal", "negative"):
        out[f"63x17-{kind}"] = (63, 17, kind, {})
    out["63x17-negative-gamma1"] = (63, 17, "negative", dict(Gamma=1.0))
    out["63x17-negative-gamma0.5"] = (63, 17, "negative", dict(Gamma=0.5, MipCount=1))
    return out


CASES = _cases()


@functools.lru_cache(maxsize=None)
def case(name):
    W, H, kind, kw = CASES[name]
    p = dict(DEFAULTS, **kw)
    return _input(kind, W, H, p), p


def oracle_run(hdr, p):
    pc = orc.default_post_config(**p)
    return orc.post_process(hdr, pc, want_bloom=True)


def _report(tag, name, bad_b, bad_l, und, far):
    print(f"{tag} {name}: undecided {und * 100:.3f} %, bloom outside {int(bad_b.sum())}, decided bytes wrong {int(bad_l.sum())}")


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_model(name):
    hdr, p = case(name)
    ldr, bloom = oracle_run(hdr, p)
    bad_b, bad_l, und, far = check(hdr, p, bloom, ldr)
    _report("oracle", name, bad_b, bad_l, und, far)
    assert not bad_b.any(), np.argwhere(bad_b)[:5]
    assert not bad_l.any(), np.argwhere(bad_l)[:5]
    assert not far.any()
    assert und <= UNDECIDED_MAX


# ---------------------------------------------------------------- dependency model (rows; columns are the same function of W)
def _mat(n_out, n_in, idx_lists):
    M = np.zeros((n_out, n_in), bool)
    for idx in idx_lists: M[np.arange(n_out), idx] = True
    return M


def dependency(n, sizes_1d, mips):
    """-> (out [n, n] bool: HDR lines per output line, down [i] and up [i]: HDR lines per line of mip i) for one axis"""
    down = [np.eye(n, dtype=bool)]
    for i in range(1, mips):
        ni, no = sizes_1d[i - 1], sizes_1d[i]
        down.append((_mat(no, ni, [np.clip(2 * np.arange(no) + b, 0, ni - 1) for b in range(-2, 2)]).astype(int) @ down[-1]) > 0)
    up = list(down)
    for i in range(mips - 1, 0, -1):
        ni, no = sizes_1d[i], sizes_1d[i - 1]
        up[i - 1] = down[i - 1] | ((_mat(no, ni, [np.clip(np.arange(no) // 2 + b + 1, 0, ni - 1) for b in range(-2, 2)]).astype(int) @ up[i]) > 0)
    fetch = _mat(n, n, [np.clip(np.arange(n) - 1, 0, n - 1), np.arange(n)])
    out = np.eye(n, dtype=bool) | ((fetch.astype(int) @ up[0]) > 0)
    return out, down, up


def rows_needed(H, W, p, y0, y1):
    """HDR rows [lo, hi] that output rows [y0, y1) depend on"""
    sizes = mip_sizes(W, H)
    out, _, _ = dependency(H, [s[1] for s in sizes], mip_count(p, W, H))
    r = np.flatnonzero(out[y0:y1].any(0))
    assert np.array_equal(r, np.arange(r[0], r[-1] + 1))                  # an interval
    return int(r[0]), int(r[-1])


def footprint_hit(H, W, p, bad_yx):
    """[H, W] bool: output pixels whose dependency footprint holds one of the texels bad_yx"""
    sizes = mip_sizes(W, H); n = mip_count(p, W, H)
    ro, _, _ = dependency(H, [s[1] for s in sizes], n); co, _, _ = dependency(W, [s[0] for s in sizes], n)
    hit = np.zeros((H, W), bool)
    for y, x in bad_yx: hit |= ro[:, y][:, None] & co[:, x][None, :]
    return hit


@pytest.mark.parametrize("W,H,mips", [(37, 33, 10), (65, 17, 2), (65, 17, 3), (31, 50, 10), (20, 1, 10), (40, 8, 10)])
def test_dependency_model_matches_the_oracle(W, H, mips):
    """Rows outside the model's footprint of [y0, y1) leave the oracle's rows [y0, y1) bit for bit; the footprint's first and last rows do not"""
    p = dict(DEFAULTS, MipCount=mips)
    hdr = _hot(W, H, 4)
    ldr, bloom = oracle_run(hdr, p)
    for y0, y1 in {(0, 1), (H // 2, H // 2 + 1), (max(H - 1, 0), H), (H // 3, max(H // 3 + 1, 2 * H // 3)), (0, H)}:
        lo, hi = rows_needed(H, W, p, y0, y1)
        out = hdr.copy(); out[:lo, :, :3] = 1e4; out[hi + 1:, :, :3] = 1e4
        l2, _ = oracle_run(out, p)
        assert np.array_equal(l2[y0:y1], ldr[y0:y1]), (y0, y1, lo, hi)
        for edge in {lo, hi}:
            e = hdr.copy(); e[edge, :, :3] = 7e3
            l3, b3 = oracle_run(e, p)
            assert not np.array_equal(b3[max(y0 - 1, 0):y1], bloom[max(y0 - 1, 0):y1]), (y0, y1, edge)   # output rows read bloom rows y-1, y


# ---------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def pt():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import vpt_b200
    return vpt_b200


def _tracer(W, H, p=None):
    import vpt_b200 as P
    T = P.PathTracer(0)
    T.set_scene(util.scene_dict("cornell_box")); T.resize(W, H)
    if p is not None: _params(T, p)
    return T


def _params(T, p):
    T.set_bloom(p["BloomThreshold"], p["BloomStrength"], p["MipCount"], p["FalloffRange"]); T.set_tonemap(p["Exposure"], p["Gamma"])


def _gpu_post(hdr, p, T=None):
    H, W = hdr.shape[:2]
    T = T or _tracer(W, H, p)
    T.set_hdr(hdr); T.post_process()
    return T.get_ldr().copy(), T.get_bloom().copy()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_gpu_matches_oracle_and_model(pt, name):
    hdr, p = case(name)
    ldr, bloom = _gpu_post(hdr, p)
    rl, rb = oracle_run(hdr, p)
    bad_b, bad_l, und, far = check(hdr, p, bloom, ldr)
    _report("gpu", name, bad_b, bad_l, und, far)
    assert not bad_b.any(), np.argwhere(bad_b)[:5]
    assert np.allclose(bloom[..., :3], rb[..., :3], rtol=2e-6, atol=1e-6)
    assert not bad_l.any(), np.argwhere(bad_l)[:5]
    assert not far.any()
    assert und <= UNDECIDED_MAX
    _, dec = ldr_of(*model_chain(hdr, p)[1])
    assert np.array_equal(ldr[..., :3][dec], rl[..., :3][dec])              # GPU and oracle differ on undecided bytes only
    assert (ldr[..., 3] == 255).all()


@pytest.mark.gpu
def test_margin_is_tight(pt):
    """K / 10 rejects some GPU answer, K accepts all of them"""
    rejected = 0
    for name in ("317x203", "1023x767", "65x15-gamma4", "63x17-negative", "317x203-mips3"):
        hdr, p = case(name)
        ldr, bloom = _gpu_post(hdr, p)
        bad_b, bad_l, _, _ = check(hdr, p, bloom, ldr, k=K / 10)
        rejected += int(bad_b.sum() + bad_l.sum())
        bad_b, bad_l, _, _ = check(hdr, p, bloom, ldr, k=K)
        assert not bad_b.any() and not bad_l.any()
    print("rejected at K / 10:", rejected)
    assert rejected > 0


BAD = {"inf": np.inf, "-inf": -np.inf, "nan": np.nan, "3e38": 3e38}


@pytest.mark.gpu
@pytest.mark.parametrize("bad", list(BAD))
@pytest.mark.parametrize("W,H,mips", [(65, 15, 10), (33, 9, 2), (37, 1, 10), (317, 203, 10)])
def test_nonfinite_inputs_match_the_oracle(pt, bad, W, H, mips):
    p = dict(DEFAULTS, MipCount=mips)
    clean = _hot(W, H, 12)
    hdr = clean.copy()
    where = sorted({(0, 0), (H - 1, W - 1), (H // 2, min(32, W - 1)), (min(8, H - 1), W // 3)})
    for k, (y, x) in enumerate(where): hdr[y, x, k % 3] = BAD[bad]
    if bad == "3e38": hdr[H // 2, :min(W, 5), :3] = 3e38                    # several in one tap window: the sums overflow
    ldr, bloom = _gpu_post(hdr, p)
    rl, rb = oracle_run(hdr, p)
    cls = lambda a: np.where(np.isnan(a), 2, np.where(np.isinf(a), 1, 0))
    assert np.array_equal(cls(bloom[..., :3]), cls(rb[..., :3]))
    assert np.array_equal(ldr, rl), int((ldr != rl).any(-1).sum())
    bad_yx = [tuple(i) for i in np.argwhere(~np.isfinite(hdr[..., :3]).all(-1) | (np.abs(hdr[..., :3]) > 1e38).any(-1))]
    hit = footprint_hit(H, W, p, bad_yx)
    lc, bc = _gpu_post(clean, p)
    assert np.array_equal(ldr[~hit], lc[~hit])
    assert np.array_equal(bloom[~hit].view(np.uint32), bc[~hit].view(np.uint32))


# ---------------------------------------------------------------- row blocks
def _poisoned(hdr, in0, in1):
    out = hdr.copy(); out[:in0] = np.nan; out[in1:] = np.nan
    return out


def _blocks(H):
    bl = [(y, y + 1) for y in range(H)]
    bl += [(0, c) for c in range(1, H)] + [(c, H) for c in range(1, H)]
    bl += [(y, min(y + 9, H)) for y in range(0, H, 8)]                      # blocks ending one row into an 8-row tile
    return sorted(set(bl))


@pytest.mark.gpu
@pytest.mark.parametrize("W,H,mips", [(33, 9, 10), (63, 17, 10), (65, 15, 2), (65, 15, 3), (40, 33, 10), (517, 389, 10)])
def test_post_input_rows_suffice_for_the_block(pt, W, H, mips):
    """[in0, in1) holds the model's dependency rows; the block computed from an image that is NaN outside them equals the full pass,
    on a fresh handle and on a stale one that has just post-processed another image"""
    p = dict(DEFAULTS, MipCount=mips)
    hdr = _hot(W, H, 21); other = _lognormal(W, H, 22) * np.float32(3.0)
    full, _ = _gpu_post(hdr, p)
    stale = _tracer(W, H, p)
    blocks = _blocks(H) if H < 40 else [(0, 1), (1, 2), (7, 9), (8, 17), (100, 101), (129, 257), (380, 389), (388, 389), (0, 389)]
    excess = []
    for y0, y1 in blocks:
        lo, hi = rows_needed(H, W, p, y0, y1)
        in0, in1 = stale.post_input_rows(y0, y1)
        assert in0 <= lo and in1 >= hi + 1, (y0, y1, in0, in1, lo, hi)
        excess.append((lo - in0) + (in1 - 1 - hi))
        img = _poisoned(hdr, in0, in1)
        stale.set_hdr(other); stale.post_process()
        stale.set_hdr(img); stale.post_process_rows(y0, y1)
        assert np.array_equal(stale.get_ldr_rows(y0, y1), full[y0:y1]), ("stale", y0, y1)
        if (y1 - y0 == 1 and y0 % 4 == 0) or y1 == H or y0 == 0:
            T = _tracer(W, H, p); T.set_hdr(img); T.post_process_rows(y0, y1)
            assert np.array_equal(T.get_ldr_rows(y0, y1), full[y0:y1]), ("fresh", y0, y1)
    print(f"{W}x{H} mips {mips}: post_input_rows exceeds the dependency rows by {min(excess)}..{max(excess)} rows over {len(blocks)} blocks")


@pytest.mark.gpu
def test_post_rows_refuse_bad_ranges(pt, monkeypatch):
    W, H = 33, 17
    T = _tracer(W, H, DEFAULTS); T.set_hdr(_hot(W, H, 3))
    for y0, y1 in ((5, 5), (6, 5), (0, H + 1), (H, H + 1)):
        with pytest.raises(pt.B200ptError) as e: T.post_process_rows(y0, y1)
        assert e.value.code == pt.ERR_WRONG_ARGUMENTS
        with pytest.raises(pt.B200ptError) as e: T.post_input_rows(y0, y1)
        assert e.value.code == pt.ERR_WRONG_ARGUMENTS
    T.set_bloom(2.0, 1.0, 1, 5.0)                                                   # 1-level chain: the unfused path
    with pytest.raises(pt.B200ptError) as e: T.post_process_rows(2, 9)
    assert e.value.code == pt.ERR_NOT_IMPLEMENTED
    T.post_process_rows(0, H)
    T.set_bloom(2.0, 1.0, 10, 5.0)
    monkeypatch.setenv("B200PT_POST_FUSED", "0")
    with pytest.raises(pt.B200ptError) as e: T.post_process_rows(2, 9)
    assert e.value.code == pt.ERR_NOT_IMPLEMENTED
    T.post_process_rows(0, H)


# ---------------------------------------------------------------- accumulate_rows
def _frames(W, H, n, seed):
    rng = np.random.default_rng(seed)
    out = np.ones((n, H, W, 4), np.float32)
    out[..., :3] = (np.exp(rng.normal(0, 2.0, (n, H, W, 3))) * rng.choice([1e-3, 1.0, 1e3], (n, H, W, 1))).astype(np.float32)
    return out


def _accumulate_model(prev, new, f):
    """lerp(prev, new, 1 / (f + 1)) in float64 with the bound of a 2-ulp reciprocal and x (1 - a) + y a; and the oracle's v3lerp in fp32"""
    if f == 0: return E(new.astype(np.float64)), new
    a = E(1.0).div(E(float(np.float32(f + 1))))
    m = E(prev.astype(np.float64)) * (E(1.0) - a) + E(new.astype(np.float64)) * a
    a32 = np.float32(1.0) / np.float32(f + 1)
    return m, prev * (np.float32(1.0) - a32) + new * a32


@pytest.mark.gpu
@pytest.mark.parametrize("W,H", [(1, 1), (37, 5), (65, 17)])
def test_accumulate_rows_is_the_running_mean(pt, W, H):
    import torch
    T = _tracer(W, H)
    fr = _frames(W, H, 6, W + H)
    T.set_hdr(fr[0])
    img = fr[0].copy()
    for f, k in zip((0, 1, 2, 1000, 2 ** 24 - 1), range(1, 6)):
        d = torch.from_numpy(fr[k]).cuda(); torch.cuda.synchronize()
        y0, y1 = (0, H) if H < 3 else (1, H - 1)
        T.accumulate_rows(d.data_ptr(), f, y0, y1)
        got = T.get_hdr()
        m, o32 = _accumulate_model(img[y0:y1, :, :3], fr[k][y0:y1, :, :3], f)
        g = got[y0:y1, :, :3].astype(np.float64)
        assert (np.abs(g - m.v) <= K * m.e).all(), f
        assert (np.abs(o32 - m.v) <= K * m.e).all(), f
        if f == 0: assert np.array_equal(got[y0:y1].view(np.uint32), fr[k][y0:y1].view(np.uint32))
        assert (got[y0:y1, :, 3] == 1.0).all()
        assert np.array_equal(got[:y0].view(np.uint32), img[:y0].view(np.uint32)) and np.array_equal(got[y1:].view(np.uint32), img[y1:].view(np.uint32))
        img = got.copy()


@pytest.mark.gpu
def test_accumulate_rows_in_pieces_and_bad_arguments(pt):
    import torch
    W, H = 33, 19
    fr = _frames(W, H, 2, 5)
    d = torch.from_numpy(fr[1]).cuda(); torch.cuda.synchronize()
    A = _tracer(W, H); A.set_hdr(fr[0]); A.accumulate_rows(d.data_ptr(), 3, 0, H)
    B = _tracer(W, H); B.set_hdr(fr[0])
    for y0, y1 in ((0, 1), (1, 8), (8, 9), (9, 19)): B.accumulate_rows(d.data_ptr(), 3, y0, y1)
    ref = A.get_hdr().copy()
    assert np.array_equal(B.get_hdr().view(np.uint32), ref.view(np.uint32))
    for args in ((0, 3, 0, H), (d.data_ptr(), 3, 5, 5), (d.data_ptr(), 3, 6, 5), (d.data_ptr(), 3, 0, H + 1)):
        with pytest.raises(pt.B200ptError) as e: A.accumulate_rows(*args)
        assert e.value.code == pt.ERR_WRONG_ARGUMENTS
        assert np.array_equal(A.get_hdr().view(np.uint32), ref.view(np.uint32))
    P = _tracer(W, H); P.set_partition(0, 2, 4)
    with pytest.raises(pt.B200ptError) as e: P.accumulate_rows(d.data_ptr(), 3, 0, 4)
    assert e.value.code == pt.ERR_WRONG_ARGUMENTS


# ---------------------------------------------------------------- config 5 on N simulated ranks
@pytest.mark.gpu
@pytest.mark.parametrize("W,H,world", [(65, 15, 2), (33, 9, 3), (63, 17, 8), (517, 389, 3), (640, 360, 2), (640, 360, 3), (640, 360, 8)])
def test_post_on_simulated_ranks_equals_one_handle(pt, W, H, world):
    """bench.py's post loop without bench.py: rank r folds k frames into its rows [in0, in1) of an image that is NaN elsewhere, then
    post-processes its block; the union of the blocks equals one handle's accumulate over [0, H) and full pass, bit for bit"""
    import torch
    k = 3
    fr = _frames(W, H, k + 1, 31)
    fr[..., :3] = np.minimum(fr[..., :3], 50.0)
    dev = [torch.from_numpy(f).cuda() for f in fr[1:]]; torch.cuda.synchronize()
    One = _tracer(W, H, DEFAULTS); One.set_hdr(fr[0])
    for i, d in enumerate(dev): One.accumulate_rows(d.data_ptr(), i + 1, 0, H)
    One.post_process(); full = One.get_ldr().copy()
    cut = lambda r: min((H * r // world + 7) // 8 * 8, H) if r < world else H
    cuts = [cut(r) for r in range(world + 1)]
    if world > 1 and cuts[1] + 3 < cuts[2]: cuts[1] += 3                      # one boundary off the 8-row tiles
    out = np.zeros_like(full); covered = 0
    for r in range(world):
        y0, y1 = cuts[r], cuts[r + 1]
        if y0 >= y1: continue
        T = _tracer(W, H, DEFAULTS)
        in0, in1 = T.post_input_rows(y0, y1)
        T.set_hdr(_poisoned(fr[0], in0, in1))
        for i, d in enumerate(dev): T.accumulate_rows(d.data_ptr(), i + 1, in0, in1)
        T.post_process_rows(y0, y1)
        out[y0:y1] = T.get_ldr_rows(y0, y1); covered += y1 - y0
    assert covered == H
    assert np.array_equal(out, full), int((out != full).any(-1).sum())
