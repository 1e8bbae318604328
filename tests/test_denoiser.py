"""The denoiser of the accumulated image: per-pixel statistics without adaptive sampling (b200pt_set_track_variance), the feature pass
(k_features) and the a-trous filter (b200pt_denoise / b200pt_denoise_image).  The statistics must not change the render; the features and
the filter are pinned against numpy restatements; the handle form must equal the array form; the result must not depend on scheduling,
checkpoints or the post chain's input path.  The last tests need no GPU.
"""
import ctypes as C
import json
import os
import struct
import subprocess

import numpy as np
import pytest

import util
import vpt_b200 as pt
from oracle import orc

gpu = pytest.mark.gpu

W, H, N = 96, 70, 24
LUM = np.array([0.212671, 0.715160, 0.072169])
WORK = ("paths", "extend_rays", "shade_invocations", "surface_hits", "misses", "shadow_rays", "medium_events", "kernel_launches")
FOG = dict(CornerMin=(-4.0, -4.0, -10.0), CornerMax=(4.5, 3.0, -1.0), Density=0.35, Color=(0.8, 0.7, 0.6), Anisotropy=0.4)
H_B3 = np.array([1 / 16, 1 / 4, 3 / 8, 1 / 4, 1 / 16])
FEATURE_SEED = 0x46454154


@pytest.fixture(scope="module")
def gpu_pt():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return pt


def _tracer(scene="cornell_box", depth=6, w=W, h=H, stats=True, adaptive=None, partition=None, **cfg):
    T = util.product_tracer(scene, w, h, MaxDepth=depth, **cfg)
    if partition: T.set_partition(*partition)
    if adaptive is not None: T.set_adaptive(**adaptive)
    if stats: T.set_track_variance(True)
    return T


def _work(T):
    c = T.counters()
    return {k: c[k] for k in WORK}


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _rmse(a, b):
    return float(np.sqrt(np.mean((a[..., :3].astype(np.float64) - b[..., :3]) ** 2)))


# ---------------------------------------------------------------- 1. statistics do not change the render

CASES = {
    "cornell": dict(),
    "glass": dict(scene="cornell_box_glass", depth=8),                 # BVH outside shared memory: k_raygen + the dynamic-fetch kernels
    "volume": dict(Volumes=[FOG]),                                       # pre-pass: k_raygen, k_volume_decide, k_shade_volume
    "two_samples": dict(SamplesPerFrame=2),
}


@gpu
@pytest.mark.parametrize("name", list(CASES))
def test_statistics_do_not_change_the_render(gpu_pt, name):
    case = CASES[name]
    off = _tracer(stats=False, **case); off.path_trace(N, util.BASE_SEED)
    on = _tracer(**case); on.path_trace(N, util.BASE_SEED)
    assert on.get_track_variance() and not off.get_track_variance()
    assert np.array_equal(_bits(on.get_hdr()), _bits(off.get_hdr()))
    assert _work(on) == _work(off)                                       # only the resolve kernel differs, one for one
    counts, rel = on.pixel_stats()
    assert (counts == N).all() and np.isfinite(rel).all()
    assert np.isnan(off.pixel_stats()[1]).all()
    # the records equal those of adaptive sampling with Threshold 0 (nothing stops)
    ad = _tracer(stats=False, adaptive=dict(Enable=1, Threshold=0.0, MinSamples=8, Interval=8), **case); ad.path_trace(N, util.BASE_SEED)
    c2, r2 = ad.pixel_stats()
    assert np.array_equal(c2, counts) and np.array_equal(_bits(r2), _bits(rel))
    assert np.array_equal(_bits(on.denoise_inputs(FeatureSamples=1)[2]), _bits(ad.denoise_inputs(FeatureSamples=1)[2]))


# ---------------------------------------------------------------- 2. feature pass against a numpy model

def _forward(vi, pi):
    t = np.array([pi[8] + pi[12], pi[9] + pi[13], pi[10] + pi[14]], np.float64); t /= np.linalg.norm(t)
    d = np.array([vi[k] * t[0] + vi[4 + k] * t[1] + vi[8 + k] * t[2] for k in range(3)]); return d / np.linalg.norm(d)


def _model_materials(sc, furnace):
    """per material: albedo (pd + pm) * BaseColor + pg with the 1x1 texels of the fixtures"""
    out = []
    texel = lambda i: np.asarray(sc["textures"][i], np.float64).reshape(-1)
    for m in sc["materials"]:
        tb = texel(m["BaseColorTextureIndex"]); base = np.asarray(m["BaseColor"], np.float64) * (tb[:3] / 255.0) ** 2.2
        metal = float(m["Metallic"]) * texel(m["MetallicTextureIndex"])[0] / 255.0; tr = float(m["Transmission"])
        pm, pd, pg = metal, (1 - metal) * (1 - tr), (1 - metal) * tr
        s = pm + pd + pg; pm, pd, pg = pm / s, pd / s, pg / s
        out.append((pd + pm) * (np.ones(3) if furnace else base) + pg)
    return np.array(out)


def _model_features(name, w, h, samples, furnace=False):
    """k_features restated: the PCG stream per pixel, camera_ray's arithmetic, the oracle's closest hit, the fixture's materials"""
    sc = util.scene_dict(name); vi, pi = util.camera(name)
    vi = vi.astype(np.float64); pi = pi.astype(np.float64)
    S = util.oracle_scene(name)
    seed0 = orc.pcg_hash(FEATURE_SEED)
    ys, xs = np.mgrid[0:h, 0:w]
    u = np.stack([orc.rng_floats((int(y) + w * int(x) + seed0) & 0xFFFFFFFF, 4 * samples) for y, x in zip(ys.ravel(), xs.ravel())]).astype(np.float64)
    u = u.reshape(h * w, samples, 4)
    eye = vi[12:15]
    pcx = xs.ravel()[:, None] + 0.5 + (u[..., 0] - 0.5); pcy = ys.ravel()[:, None] + 0.5 + (u[..., 1] - 0.5)
    dx = pcx / w * 2 - 1; dy = pcy / h * 2 - 1
    tgt = np.stack([pi[0] * dx + pi[4] * dy + pi[8] + pi[12], pi[1] * dx + pi[5] * dy + pi[9] + pi[13], pi[2] * dx + pi[6] * dy + pi[10] + pi[14]], -1)
    tgt /= np.linalg.norm(tgt, axis=-1, keepdims=True)
    d = tgt[..., 0:1] * vi[0:3] + tgt[..., 1:2] * vi[4:7] + tgt[..., 2:3] * vi[8:11]   # default DepthOfFieldStrength 0: the origin is the eye
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    o = np.broadcast_to(eye, d.shape)
    t, prim, inst, _ = S.trace_closest(o.reshape(-1, 3), d.reshape(-1, 3), 0.01, 1e5)
    hit = (t > 0).reshape(h * w, samples)
    mat_of_inst = np.array([m for _, _, m in sc["instances"]])
    alb_m = _model_materials(sc, furnace)
    inst = inst.reshape(h * w, samples)
    alb = np.where(hit[..., None], alb_m[mat_of_inst[np.where(hit, inst, 0)]], 1.0).mean(1)
    pos = o + d * t.reshape(h * w, samples, 1)
    z = ((pos - eye) @ _forward(vi, pi))
    nh = hit.sum(1)
    depth = np.where(nh > 0, np.where(hit, z, 0).sum(1) / np.maximum(nh, 1), 0.0)
    return alb.reshape(h, w, 3), (nh / samples).reshape(h, w), depth.reshape(h, w), hit, inst, prim.reshape(h * w, samples), d


def _close(got, want, rtol=1e-4, floor=1e-2):
    return np.abs(got - want) <= rtol * np.maximum(np.abs(want), floor)


@gpu
@pytest.mark.parametrize("name", ["cornell_box", "cornell_box_glass"])
def test_features_match_a_numpy_model(gpu_pt, name):
    w, h, spp = 64, 40, 4
    T = _tracer(scene=name, w=w, h=h)
    a, nd, v = T.denoise_inputs(FeatureSamples=spp)
    alb, cov, depth, hit, inst, prim, dirs = _model_features(name, w, h, spp)
    ok = _close(a[..., :3], alb).all(-1) & _close(a[..., 3], cov) & _close(nd[..., 3], depth)
    assert ok.mean() > 0.99, ok.mean()
    assert (v == np.float32(1e30)).all()                                  # no frames yet: the variance is unknown
    if name == "cornell_box":
        # pixels whose rays all hit one flat triangle plane: the shading normal is the wall's, facing the camera
        S = util.oracle_scene(name)
        tri, tinst, tprim = S.world_triangles()
        nrm = np.cross(tri[:, 3:6] - tri[:, 0:3], tri[:, 6:9] - tri[:, 0:3]); nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
        idx = {(int(i), int(p)): k for k, (i, p) in enumerate(zip(tinst, tprim))}
        flat = hit.all(1)
        wall = np.zeros((h * w, 3))
        for q in np.nonzero(flat)[0]:
            ns = np.array([nrm[idx[(int(inst[q, s]), int(prim[q, s]))]] for s in range(spp)])
            ns *= -np.sign((ns * dirs[q]).sum(1))[:, None]                   # oriented against the rays
            if np.abs(ns - ns[0]).max() < 1e-5: wall[q] = ns[0]
            else: flat[q] = False
        got = nd[..., :3].reshape(-1, 3)[flat]
        assert flat.sum() > 500                                            # of 2,560 pixels; the rest see the sky or an edge
        assert (np.linalg.norm(got - wall[flat], axis=1) < 2e-2).mean() > 0.99
        assert ((got * dirs[flat, 0]).sum(1) < 0).all()


@gpu
def test_features_in_furnace_mode_and_across_a_partition(gpu_pt):
    T = _tracer(FurnaceTestMode=1)
    a, _, _ = T.denoise_inputs(FeatureSamples=3)
    assert np.abs(a[..., :3] - 1.0).max() < 1e-6
    one = _tracer(); one.path_trace(8, util.BASE_SEED)
    full = one.denoise_inputs()
    for rank in (0, 1):
        R = _tracer(partition=(rank, 2, 16)); R.path_trace(8, util.BASE_SEED)
        rows = pt.partition_rows(H, rank, 2, 16)
        for got, want in zip(R.denoise_inputs(), full):
            assert np.array_equal(_bits(got), _bits(want[rows])), rank


# ---------------------------------------------------------------- 3. the filter against a float64 model

def _model_filter(color, albedo_cov, normal_depth, variance, it, sl=4.0, sn=128.0, sz=1.0):
    """section 12 of DESIGN.md in float64"""
    if it == 0: return color.copy()
    c = color.astype(np.float64); a = albedo_cov[..., :3].astype(np.float64); covered = albedo_cov[..., 3] > 0
    n = normal_depth[..., :3].astype(np.float64); z = normal_depth[..., 3].astype(np.float64)
    h, w = z.shape
    am = np.maximum(a, 1e-3)
    i = c[..., :3] / am
    v = variance.astype(np.float64) / np.maximum(a @ LUM, 1e-3) ** 2

    def grad(axis):
        zz = np.moveaxis(z, axis, 0); cc = np.moveaxis(covered, axis, 0); g = np.zeros_like(zz)
        lo = np.zeros_like(cc); lo[1:] = cc[:-1]; hi = np.zeros_like(cc); hi[:-1] = cc[1:]
        zl = np.zeros_like(zz); zl[1:] = zz[:-1]; zh = np.zeros_like(zz); zh[:-1] = zz[1:]
        g = np.where(lo & hi, 0.5 * (zh - zl), np.where(hi, zh - zz, np.where(lo, zz - zl, 0.0)))
        return np.moveaxis(g, 0, axis)
    gx, gy = grad(1), grad(0)

    def shift(arr, dy, dx):
        """arr[y + dy, x + dx] and whether that tap is inside the image"""
        out = np.zeros_like(arr); ok = np.zeros((h, w), bool)
        ys, ye = max(0, -dy), min(h, h - dy); xs, xe = max(0, -dx), min(w, w - dx)
        if ys < ye and xs < xe:
            out[ys:ye, xs:xe] = arr[ys + dy:ye + dy, xs + dx:xe + dx]; ok[ys:ye, xs:xe] = True
        return out, ok
    g1 = np.array([0.25, 0.5, 0.25])
    for k in range(it):
        s = 1 << k
        gs = np.zeros((h, w)); gw = np.zeros((h, w))
        for j in (-1, 0, 1):
            for q in (-1, 0, 1):
                vq, ok = shift(v, j, q); gs += np.where(ok, g1[q + 1] * g1[j + 1] * vq, 0); gw += np.where(ok, g1[q + 1] * g1[j + 1], 0)
        den = sl * np.sqrt(gs / gw) + 1e-6
        lp = i @ LUM
        zfloor = 1e-3 * np.maximum(z, 1e-3)
        sw = np.zeros((h, w)); si = np.zeros((h, w, 3)); sv = np.zeros((h, w))
        for j in range(-2, 3):
            for q in range(-2, 3):
                iq, ok = shift(i, j * s, q * s); vq, _ = shift(v, j * s, q * s); nq, _ = shift(n, j * s, q * s)
                zq, _ = shift(z, j * s, q * s); cq, _ = shift(covered, j * s, q * s)
                wt = H_B3[q + 2] * H_B3[j + 2] * np.exp(-np.abs(lp - iq @ LUM) / den)
                wn = np.maximum(0.0, (n * nq).sum(-1)) ** sn
                wz = np.exp(-np.abs(z - zq) / (sz * np.abs(gx * q * s + gy * j * s) + zfloor))
                wt = np.where(covered & cq, wt * wn * wz, wt)
                wt = np.where(ok & (covered == cq), wt, 0.0)
                sw += wt; si += wt[..., None] * iq; sv += wt * wt * vq
        i = np.where(sw[..., None] > 0, si / np.where(sw > 0, sw, 1)[..., None], i)
        v = np.where(sw > 0, sv / np.where(sw > 0, sw, 1) ** 2, v)
    out = np.empty_like(c); out[..., :3] = i * am; out[..., 3] = c[..., 3]
    return out


def _synthetic(w=67, h=45, seed=7):
    """two planes with different normals and depth slopes, a miss band, partial coverage at the seam, zero and unknown variances"""
    rng = np.random.default_rng(seed)
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
    left = xs < 0.55 * w
    n = np.where(left[..., None], [0.0, 0.0, 1.0], [0.6, 0.0, 0.8])
    z = np.where(left, 5.0 + 0.02 * xs + 0.01 * ys, 3.0 + 0.05 * ys - 0.015 * xs)
    alb = np.where(left[..., None], [0.7, 0.3, 0.2], [0.2, 0.5, 0.8]) * (1 + 0.1 * rng.random((h, w, 3)))
    cov = np.ones((h, w))
    miss = ys < 6
    seam = (np.abs(xs - 0.55 * w) < 1) & ~miss
    cov[seam] = 0.5; n[seam] *= 0.95
    cov[miss] = 0; n[miss] = 0; z[miss] = 0; alb[miss] = 1
    light = 0.5 + 0.3 * np.sin(xs / 9) * np.cos(ys / 7)
    color = np.ones((h, w, 4)); color[..., :3] = alb * light[..., None] * (1 + 0.3 * rng.standard_normal((h, w, 3)))
    color[miss, :3] = 0.2 + 0.05 * rng.random((int(miss.sum()), 3))
    var = 10 ** rng.uniform(-4, -2, (h, w))
    var[rng.random((h, w)) < 0.05] = 0.0; var[30:33, 10:13] = 0.0
    var[20:24, 40:45] = 1e30
    f = np.float32
    return (color.astype(f), np.concatenate([alb, cov[..., None]], -1).astype(f), np.concatenate([n, z[..., None]], -1).astype(f), var.astype(f))


@gpu
@pytest.mark.parametrize("it", [1, 3, 5])
def test_filter_matches_a_float64_model(gpu_pt, it):
    T = _tracer(w=16, h=16)
    c, a, nd, v = _synthetic()
    got = T.denoise_image(c, a, nd, v, Iterations=it)
    want = _model_filter(c, a, nd, v, it)
    ok = _close(got, want, 1e-4, 1e-3)
    assert ok.all(), (int((~ok).sum()), float(np.abs(got - want).max()))
    assert np.abs(got - c).max() > 1e-3                                  # it did filter


@gpu
def test_filter_with_zero_iterations_copies_the_input(gpu_pt):
    T = _tracer(w=16, h=16)
    c, a, nd, v = _synthetic()
    c[0, 0, 0] = np.float32(1e-40)                                        # a denormal survives too
    assert np.array_equal(_bits(T.denoise_image(c, a, nd, v, Iterations=0)), _bits(c))


# ---------------------------------------------------------------- 4. handle form == array form

@gpu
def test_handle_form_equals_the_array_form(gpu_pt):
    T = _tracer(); T.path_trace(16, util.BASE_SEED)
    raw = T.get_hdr().copy()
    ms = T.denoise()
    assert ms > 0
    d = T.get_denoised()
    assert np.array_equal(_bits(T.get_hdr()), _bits(raw))                # the accumulation is not touched
    a, nd, v = T.denoise_inputs()
    assert np.array_equal(_bits(T.denoise_image(raw, a, nd, v)), _bits(d))
    assert np.isfinite(d).all() and not np.array_equal(d, raw)


# ---------------------------------------------------------------- 5. / 6. quality and convergence

# depth, size, bar on RMSE(denoised) / RMSE(raw).  With the default footprint (5 passes, up to 64 pixels wide) the Cornell box needs its own aspect
# and resolution: squeezed into 256 x 256 the filter blurs across its features and the denoised error is 1.5x the raw one (DESIGN.md section 12).
QUALITY = {"cornell_box": (8, 1920, 1080, 0.85), "cornell_box_glass": (16, 256, 256, 0.85)}


@gpu
@pytest.mark.parametrize("name", list(QUALITY))
def test_denoising_lowers_the_error_at_16_frames(gpu_pt, name):
    depth, w, h, bar = QUALITY[name]
    R = _tracer(scene=name, depth=depth, w=w, h=h, stats=False); R.path_trace(1024, util.BASE_SEED + 77)
    ref = R.get_hdr().copy()
    T = _tracer(scene=name, depth=depth, w=w, h=h); T.path_trace(16, util.BASE_SEED)
    T.denoise()
    raw, den = _rmse(T.get_hdr(), ref), _rmse(T.get_denoised(), ref)
    print(f"{name}: RMSE raw {raw:.5f} denoised {den:.5f} ratio {den / raw:.3f}")
    assert den < bar * raw


@gpu
def test_the_filter_backs_off_as_the_render_converges(gpu_pt):
    T = _tracer(w=128, h=128, depth=8)
    done, rel = 0, []
    for frames in (16, 64, 256):
        T.path_trace(frames - done, util.BASE_SEED); done = frames
        T.denoise()
        rel.append(util.rel_l2(T.get_denoised()[..., :3], T.get_hdr()[..., :3]))
    print("relative L2 denoised vs raw at 16 / 64 / 256 frames:", rel)
    assert rel[0] > rel[1] > rel[2]


# ---------------------------------------------------------------- 7. invariance

# fuse2: B200PT_FUSE=2 selected the bounce kernel, which is gone; an unsupported value must keep the default pipeline
VARIANTS = [("fif1", {}, dict(FramesInFlight=1)), ("fuse0", {"B200PT_FUSE": "0"}, {}), ("fuse2", {"B200PT_FUSE": "2"}, {}),
            ("camera0", {"B200PT_CAMERA": "0"}, {}), ("split", {}, {})]
_BASE = {}


@gpu
@pytest.mark.parametrize("name,env,cfg", VARIANTS, ids=[v[0] for v in VARIANTS])
def test_denoised_image_does_not_depend_on_scheduling(gpu_pt, monkeypatch, name, env, cfg):
    if "img" not in _BASE:
        B = _tracer(); B.path_trace(N, util.BASE_SEED); B.denoise(); _BASE["img"] = B.get_denoised()
    for k, v in env.items(): monkeypatch.setenv(k, v)
    T = _tracer(**cfg)
    if name == "split": T.path_trace(5, util.BASE_SEED); T.path_trace(N - 5, util.BASE_SEED)
    else: T.path_trace(N, util.BASE_SEED)
    T.denoise()
    assert np.array_equal(_bits(T.get_denoised()), _bits(_BASE["img"])), name


# ---------------------------------------------------------------- 8. checkpoints

@gpu
def test_checkpoint_resume_gives_the_same_denoised_image(gpu_pt, tmp_path):
    ref = _tracer(); ref.path_trace(N, util.BASE_SEED); ref.denoise()
    A = _tracer(); A.path_trace(10, util.BASE_SEED)
    ck = tmp_path / "s.ckpt"; A.save_checkpoint(ck)
    assert struct.unpack_from("<I", open(ck, "rb").read(12), 8)[0] == 2
    B = _tracer(); B.load_checkpoint(ck); B.path_trace(N - 10, util.BASE_SEED); B.denoise()
    assert np.array_equal(_bits(B.get_denoised()), _bits(ref.get_denoised()))
    assert np.array_equal(B.pixel_stats()[0], ref.pixel_stats()[0])
    plain = _tracer(stats=False); plain.path_trace(3, util.BASE_SEED)
    v1 = tmp_path / "p.ckpt"; plain.save_checkpoint(v1)
    adaptive = _tracer(stats=False, adaptive=dict(Enable=1, Threshold=0.0))
    for T, path in ((_tracer(), v1), (_tracer(stats=False), ck), (adaptive, ck)):
        with pytest.raises(pt.B200ptError) as e:
            T.load_checkpoint(path)
        assert e.value.code == pt.ERR_WRONG_ARGUMENTS


# ---------------------------------------------------------------- 9. post chain

@gpu
def test_post_chain_on_the_denoised_image(gpu_pt):
    T = _tracer(); T.path_trace(16, util.BASE_SEED); T.denoise()
    T.post_process_denoised()
    ldr, bloom = T.get_ldr().copy(), T.get_bloom().copy()                # get_bloom re-runs the chain on the denoised image
    P = _tracer(stats=False); P.set_hdr(T.get_denoised()); P.post_process()
    assert np.array_equal(ldr, P.get_ldr()) and np.array_equal(_bits(bloom), _bits(P.get_bloom()))
    T.post_process()                                                      # and the plain pass reads the accumulation again
    Q = _tracer(stats=False); Q.set_hdr(T.get_hdr()); Q.post_process()
    assert np.array_equal(T.get_ldr(), Q.get_ldr()) and np.array_equal(_bits(T.get_bloom()), _bits(Q.get_bloom()))


# ---------------------------------------------------------------- 10. adaptive sampling

@gpu
def test_denoiser_reads_the_adaptive_records(gpu_pt):
    T = _tracer(stats=False, adaptive=dict(Enable=1, Threshold=0.05, MinSamples=8, Interval=8))
    T.path_trace(48, util.BASE_SEED)
    counts, _ = T.pixel_stats()
    assert counts.min() < 48
    T.denoise()
    a, nd, v = T.denoise_inputs()
    assert np.array_equal(_bits(T.denoise_image(T.get_hdr(), a, nd, v)), _bits(T.get_denoised()))
    assert np.isfinite(v).all() and (v < 1e30).all()


# ---------------------------------------------------------------- 11. validation and CLI

@gpu
def test_argument_validation_with_a_handle(gpu_pt):
    T = _tracer(stats=False)
    assert not T.get_track_variance()
    with pytest.raises(pt.B200ptError) as e: T.denoise()                 # neither statistics nor adaptive sampling
    assert e.value.code == pt.ERR_WRONG_ARGUMENTS
    with pytest.raises(pt.B200ptError) as e: T.denoise_inputs()
    assert e.value.code == pt.ERR_WRONG_ARGUMENTS
    with pytest.raises(pt.B200ptError) as e: T.get_denoised()            # nothing denoised yet
    assert e.value.code == pt.ERR_WRONG_ARGUMENTS
    T.set_track_variance(True)
    c, a, nd, v = _synthetic(9, 7)
    for bad in (dict(Iterations=11), dict(FeatureSamples=0), dict(FeatureSamples=257), dict(SigmaLuminance=-1.0), dict(SigmaNormal=float("nan")),
                dict(SigmaDepth=float("inf"))):
        for call in (lambda: T.denoise(**bad), lambda: T.denoise_inputs(**bad), lambda: T.denoise_image(c, a, nd, v, **bad)):
            with pytest.raises(pt.B200ptError) as e: call()
            assert e.value.code == pt.ERR_WRONG_ARGUMENTS, bad
    cfg = T.get_config(); cfg.ScreenChunkCount = 2
    with pytest.raises(pt.B200ptError) as e: T.set_config(cfg)
    assert e.value.code == pt.ERR_WRONG_ARGUMENTS
    T.set_track_variance(False); T.set_config(cfg)
    with pytest.raises(pt.B200ptError) as e: T.set_track_variance(True)
    assert e.value.code == pt.ERR_WRONG_ARGUMENTS
    R = _tracer(partition=(0, 2, 16))
    with pytest.raises(pt.B200ptError) as e: R.denoise()                 # partitioned: gather the inputs and use denoise_image
    assert e.value.code == pt.ERR_WRONG_ARGUMENTS
    assert R.denoise_inputs()[0].shape == (R.local_rows(), W, 4)
    L = pt.lib(); p = pt.default_denoise()
    assert L.b200pt_denoise_image(T.h, 9, 7, None, None, None, None, C.byref(p), None, 0) == pt.ERR_WRONG_ARGUMENTS
    assert L.b200pt_denoise(T.h, None, None) == pt.ERR_WRONG_ARGUMENTS
    assert L.b200pt_get_denoise_inputs(T.h, None, None, None, None) == pt.ERR_WRONG_ARGUMENTS


def _cli_args(tmp_path):
    hdr = str(tmp_path / "env.hdr"); util.write_rgbe(hdr, util.gltf_ref.synthetic_env(64, 32, 5)[..., :3])
    return ["--scene", util.write_synthetic_gltf(tmp_path), "--env", hdr, "--luts", util.write_luts_dir(tmp_path / "luts"), "--size", "96", "64",
            "--depth", "4", "--batch", "4", "--quiet", "--spp", "8"]


@gpu
def test_cli_writes_the_denoised_png(gpu_pt, tmp_path):
    exe = os.path.join(os.path.dirname(pt.LIB_PATH), "b200pt_render")
    args = _cli_args(tmp_path)
    outs = {}
    for tag, extra in (("raw", []), ("den", ["--denoise", "3", "--checkpoint", str(tmp_path / "d.ckpt")])):
        r = subprocess.run([exe, *args, "--out", str(tmp_path / f"{tag}.png"), *extra], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        assert json.loads(r.stdout.strip().splitlines()[-1])["spp"] == 8
        outs[tag] = pt.decode_image(str(tmp_path / f"{tag}.png"))
    assert not np.array_equal(outs["raw"], outs["den"])
    assert struct.unpack_from("<I", open(tmp_path / "d.ckpt", "rb").read(12), 8)[0] == 2   # the raw accumulation + the records


# ---------------------------------------------------------------- no GPU needed

def test_denoise_defaults_and_null_handles():
    p = pt.default_denoise()
    assert (p.Iterations, p.FeatureSamples, p.SigmaLuminance, p.SigmaNormal, p.SigmaDepth) == (5, 8, 4.0, 128.0, 1.0)
    assert C.sizeof(pt.DenoiseParams) == 20
    L = pt.lib()
    assert L.b200pt_default_denoise(None) == pt.ERR_WRONG_ARGUMENTS
    v = C.c_int32(); f = C.c_float()
    assert L.b200pt_set_track_variance(None, 1) == pt.ERR_WRONG_ARGUMENTS
    assert L.b200pt_get_track_variance(None, C.byref(v)) == pt.ERR_WRONG_ARGUMENTS
    assert L.b200pt_denoise(None, C.byref(p), C.byref(f)) == pt.ERR_WRONG_ARGUMENTS
    assert L.b200pt_get_denoised(None, None, 0) == pt.ERR_WRONG_ARGUMENTS
    assert L.b200pt_get_denoise_inputs(None, C.byref(p), None, None, None) == pt.ERR_WRONG_ARGUMENTS
    buf = np.zeros(4 * 4, np.float32)
    assert L.b200pt_denoise_image(None, 2, 2, buf.ctypes.data, buf.ctypes.data, buf.ctypes.data, buf.ctypes.data, C.byref(p), buf.ctypes.data, 0) == pt.ERR_WRONG_ARGUMENTS
    assert L.b200pt_post_process_denoised(None) == pt.ERR_WRONG_ARGUMENTS


def test_feature_seed_constant():
    assert FEATURE_SEED == int.from_bytes(b"FEAT", "big")


@pytest.mark.parametrize("args,ok", [(["--denoise"], True), (["--denoise", "0"], True), (["--denoise", "10"], True), (["--denoise", "3", "--quiet"], True),
                                     (["--denoise", "11"], False), (["--denoise", "3x"], False), (["--denoise", "-1"], False)])
def test_cli_parses_denoise(args, ok, tmp_path):
    exe = os.path.join(os.path.dirname(pt.LIB_PATH), "b200pt_render")
    missing = str(tmp_path / "missing")
    r = subprocess.run([exe, "--scene", missing + ".gltf", "--env", missing + ".hdr", "--luts", missing, "--out", str(tmp_path / "o.png"), *args],
                       capture_output=True, text=True, timeout=120)
    if ok:   # parsed: the run gets as far as the device / the missing files
        assert r.returncode not in (0, 2) and "usage:" not in r.stderr, r.stderr
    else:
        assert r.returncode == 2 and "--denoise" in r.stderr, r.stderr
