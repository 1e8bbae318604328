"""Per-pixel adaptive sampling (b200pt_set_adaptive).  A pixel is traced from frame 0 until it converges at an interval boundary, and every
path's random stream is keyed on its pixel and dispatch, so a pixel that stopped after n frames must hold bit for bit what the plain renderer
holds after n frames.  The tests pin that, the decisions against a float64 model of the Welford state, the invariance of the result to how
the frames are scheduled, the accounting, and checkpoints.  The last tests need no GPU.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import util
import vpt_b200 as pt

gpu = pytest.mark.gpu

W, H = 96, 70
INTERVAL, MIN_SAMPLES, N = 8, 8, 48                     # six decision points
LUM = np.array([0.212671, 0.715160, 0.072169])
WORK = ("paths", "extend_rays", "shade_invocations", "surface_hits", "misses", "shadow_rays", "medium_events")
FOG = dict(CornerMin=(-4.0, -4.0, -10.0), CornerMax=(4.5, 3.0, -1.0), Density=0.35, Color=(0.8, 0.7, 0.6), Anisotropy=0.4)


@pytest.fixture(scope="module")
def gpu_pt():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return pt


def _four_classes(T):
    """all four material classes (as in test_camera_kernel.py): the class queues, not the one-class pair"""
    n = T.material_count()
    m = T.get_material(1 % n); m.Metallic = 1.0; m.Roughness = 0.3; T.set_material(1 % n, m)
    m = T.get_material(2 % n); m.Metallic = 0.0; m.Transmission = 1.0; m.IOR = 1.5; m.Roughness = 0.05
    m.MediumDensity = 2.0; m.MediumAnisotropy = 0.3; m.MediumColor[0], m.MediumColor[1], m.MediumColor[2] = 0.9, 0.5, 0.3
    T.set_material(2 % n, m)
    m = T.get_material(3 % n); m.Metallic = 0.4; m.Transmission = 0.3; m.Roughness = 0.4; T.set_material(3 % n, m)


CASES = {
    "cornell": dict(),
    "four_classes": dict(edit=_four_classes, depth=8),
    "glass": dict(scene="cornell_box_glass", depth=8),                 # BVH outside shared memory: k_raygen + the dynamic-fetch kernels
    "volume": dict(Volumes=[FOG]),                                       # pre-pass: k_raygen, k_volume_decide, k_shade_volume
    "two_samples": dict(SamplesPerFrame=2),
}


def _tracer(scene="cornell_box", depth=6, edit=None, partition=None, adaptive=None, **cfg):
    T = util.product_tracer(scene, W, H, MaxDepth=depth, **cfg)
    if edit: edit(T)
    if partition: T.set_partition(*partition)
    if adaptive is not None: T.set_adaptive(**dict(dict(Enable=1, MinSamples=MIN_SAMPLES, Interval=INTERVAL), **adaptive))
    return T


def _work(T):
    c = T.counters()
    return {k: c[k] for k in WORK + ("kernel_launches",)}


def _plain_snapshots(case):
    """the plain renderer, one interval per call: snapshot k holds every pixel after (k + 1) * INTERVAL frames"""
    T = _tracer(**case)
    snaps = []
    for _ in range(N // INTERVAL):
        T.path_trace(INTERVAL, util.BASE_SEED)
        snaps.append(T.get_hdr().copy())
    return snaps, _work(T)


def _median_threshold(case):
    """Threshold 0 run (nothing stops) and a threshold at the median final relative error: the pixels well above it never stop, the pixels
    well below it stop at an early boundary"""
    T = _tracer(adaptive=dict(Threshold=0.0), **case)
    done = T.path_trace(N, util.BASE_SEED)
    counts, rel = T.pixel_stats()
    return T.get_hdr().copy(), _work(T), done, counts, rel, float(np.median(rel))


def _check_against_plain(img, counts, snaps):
    assert counts.min() >= MIN_SAMPLES and counts.max() <= N and not (counts % INTERVAL).any()
    for k, snap in enumerate(snaps):
        sel = counts == (k + 1) * INTERVAL
        got, want = img[sel].view(np.uint32), snap[sel].view(np.uint32)
        assert np.array_equal(got, want), (k, int((got != want).any(axis=-1).sum()), int(sel.sum()))


@gpu
@pytest.mark.parametrize("name", list(CASES))
def test_stopped_pixels_equal_the_plain_render_bit_for_bit(gpu_pt, name):
    case = CASES[name]
    snaps, plain_work = _plain_snapshots(case)
    spf = case.get("SamplesPerFrame", 1)
    # threshold 0: nothing converges, image and work counters equal the plain render's (only the two decision launches per interval are extra)
    img0, work0, done0, counts0, _, thr = _median_threshold(case)
    assert not done0 and (counts0 == N).all()
    assert np.array_equal(img0.view(np.uint32), snaps[-1].view(np.uint32))
    assert {k: work0[k] for k in WORK} == {k: plain_work[k] for k in WORK}
    assert thr > 0
    # the median threshold: some pixels stop early, some never do, and every pixel equals the plain render at its own frame count
    T = _tracer(adaptive=dict(Threshold=thr), **case)
    T.path_trace(N, util.BASE_SEED)
    img = T.get_hdr().copy(); counts, rel = T.pixel_stats()
    assert (counts < N).sum() > counts.size // 10 and (counts == N).sum() > counts.size // 10, np.bincount(counts.ravel())
    _check_against_plain(img, counts, snaps)
    assert 0 < T.active_pixels() <= int((counts == N).sum())           # pixels that converged at the last boundary hold N frames but stopped
    # the work counters count the traced paths only
    assert T.counters()["paths"] == int(counts.sum()) * spf


# fuse2: B200PT_FUSE=2 selected the bounce kernel, which is gone; an unsupported value must keep the default pipeline
ENV_VARIANTS = [("fif1", {}, dict(FramesInFlight=1)), ("overlap0", {"B200PT_OVERLAP": "0"}, {}),
                ("fuse0", {"B200PT_FUSE": "0"}, {}), ("fuse1", {"B200PT_FUSE": "1"}, {}), ("fuse2", {"B200PT_FUSE": "2"}, {}),
                ("camera0", {"B200PT_CAMERA": "0"}, {}), ("split", {}, {})]


@gpu
def test_result_does_not_depend_on_scheduling_or_partition(gpu_pt, monkeypatch):
    thr = _median_threshold({})[-1]
    base = _tracer(adaptive=dict(Threshold=thr))
    base.path_trace(N, util.BASE_SEED)
    img, (counts, rel) = base.get_hdr().copy(), base.pixel_stats()
    assert 0 < base.active_pixels() < W * H
    for name, env, cfg in ENV_VARIANTS:
        with monkeypatch.context() as m:
            for k, v in env.items(): m.setenv(k, v)
            T = _tracer(adaptive=dict(Threshold=thr), **cfg)
            if name == "split":
                T.path_trace(5, util.BASE_SEED); T.path_trace(N - 5, util.BASE_SEED)
            else:
                T.path_trace(N, util.BASE_SEED)
            c2, r2 = T.pixel_stats()
            assert np.array_equal(T.get_hdr().view(np.uint32), img.view(np.uint32)), name
            assert np.array_equal(c2, counts) and np.array_equal(r2.view(np.uint32), rel.view(np.uint32)), name
    for rank in (0, 1):                                                  # decisions are per pixel: each rank's rows are the 1-rank image's rows
        T = _tracer(partition=(rank, 2, 16), adaptive=dict(Threshold=thr))
        T.path_trace(N, util.BASE_SEED)
        rows = pt.partition_rows(H, rank, 2, 16)
        c2, _ = T.pixel_stats()
        assert np.array_equal(T.get_hdr().view(np.uint32), img[rows].view(np.uint32)), rank
        assert np.array_equal(c2, counts[rows]), rank


@gpu
def test_decisions_match_a_float64_model(gpu_pt):
    # dispatch f of seed s uses the Seed of dispatch 0 of seed s + f: one frame on a reset handle gives frame f of every pixel exactly
    P = _tracer()
    frames = []
    for f in range(N):
        P.reset(); P.path_trace(1, (util.BASE_SEED + f) & 0xFFFFFFFF)
        frames.append(P.get_hdr()[..., :3].astype(np.float64))
    L = np.stack(frames) @ LUM                                           # [N, H, W]
    thr = _median_threshold({})[-1]
    mean = np.zeros((H, W)); M2 = np.zeros((H, W)); n = np.zeros((H, W), np.int64)
    active = np.ones((H, W), bool); marginal = np.zeros((H, W), bool)
    for f in range(N):
        x = L[f]
        n = np.where(active, n + 1, n)
        d = x - mean
        mean = np.where(active, mean + d / np.maximum(n, 1), mean)
        M2 = np.where(active, M2 + d * (x - mean), M2)
        if (f + 1) % INTERVAL == 0:
            err = np.sqrt(M2 / np.maximum(n - 1, 1) / n); bound = thr * np.maximum(mean, 1e-3)
            ev = active & (n >= MIN_SAMPLES)
            marginal |= ev & (np.abs(err - bound) <= 1e-3 * bound)
            active &= ~(ev & (err <= bound))
    T = _tracer(adaptive=dict(Threshold=thr))
    T.path_trace(N, util.BASE_SEED)
    counts, rel = T.pixel_stats()
    ok = ~marginal
    assert ok.mean() > 0.95
    assert np.array_equal(counts[ok], n[ok]), int((counts[ok] != n[ok]).sum())
    same = ok & (counts == n)
    want = np.sqrt(M2 / (n - 1) / n) / np.maximum(mean, 1e-3)
    assert np.allclose(rel[same], want[same], rtol=1e-4, atol=1e-4 * thr)


@gpu
def test_large_threshold_stops_everything_at_the_first_boundary(gpu_pt):
    T = _tracer(SamplesPerFrame=2, adaptive=dict(Threshold=1e6, MinSamples=10))
    assert T.active_pixels() == W * H
    assert T.path_trace(100, util.BASE_SEED)                             # done: no pixel is active
    counts, _ = T.pixel_stats()
    first = -(-10 // INTERVAL) * INTERVAL                                # the first boundary at or after MinSamples
    assert (counts == first).all() and T.active_pixels() == 0
    assert T.samples_accumulated() == first * 2
    before = T.counters()
    assert T.path_trace(10, util.BASE_SEED)                              # launches nothing, the dispatch counter stays
    after = T.counters()
    assert after["kernel_launches"] == before["kernel_launches"] and after["paths"] == before["paths"] == W * H * first * 2
    assert T.samples_accumulated() == first * 2


@gpu
def test_checkpoint_v2_resumes_bit_exactly(gpu_pt, tmp_path):
    thr = _median_threshold({})[-1]
    ref = _tracer(adaptive=dict(Threshold=thr)); ref.path_trace(N, util.BASE_SEED)
    A = _tracer(adaptive=dict(Threshold=thr)); A.path_trace(20, util.BASE_SEED)
    ck = tmp_path / "a.ckpt"; A.save_checkpoint(ck)
    B = _tracer(adaptive=dict(Threshold=thr)); B.load_checkpoint(ck)
    assert B.samples_accumulated() == 20 and B.active_pixels() == A.active_pixels()
    B.path_trace(N - 20, util.BASE_SEED)
    assert np.array_equal(B.get_hdr().view(np.uint32), ref.get_hdr().view(np.uint32))
    assert np.array_equal(B.pixel_stats()[0], ref.pixel_stats()[0])
    # version / settings mismatches are refused with codes
    plain = _tracer(); plain.path_trace(3, util.BASE_SEED)
    v1 = tmp_path / "p.ckpt"; plain.save_checkpoint(v1)
    for T, path in ((_tracer(adaptive=dict(Threshold=thr)), v1), (_tracer(), ck), (_tracer(adaptive=dict(Threshold=thr * 2)), ck)):
        with pytest.raises(pt.B200ptError) as e:
            T.load_checkpoint(path)
        assert e.value.code == pt.ERR_WRONG_ARGUMENTS
    T = _tracer(); T.load_checkpoint(v1)                                 # version 1 still loads without adaptive sampling
    assert np.array_equal(T.get_hdr().view(np.uint32), plain.get_hdr().view(np.uint32))


@gpu
def test_argument_validation_with_a_handle(gpu_pt):
    T = _tracer()
    assert T.get_adaptive().Enable == 0
    counts, rel = T.pixel_stats()
    assert (counts == 0).all() and np.isnan(rel).all() and T.active_pixels() == W * H
    T.path_trace(3, util.BASE_SEED)
    assert (T.pixel_stats()[0] == 3).all()                               # without adaptive sampling: the frame count everywhere
    for bad in (dict(Threshold=-0.1), dict(Threshold=float("nan")), dict(Threshold=float("inf")), dict(Interval=0), dict(MinSamples=1)):
        with pytest.raises(pt.B200ptError) as e:
            T.set_adaptive(**dict(dict(Enable=1), **bad))
        assert e.value.code == pt.ERR_WRONG_ARGUMENTS, bad
    assert T.get_adaptive().Enable == 0
    T.set_adaptive(Enable=1, Threshold=0.05)
    a = T.get_adaptive()
    assert (a.Enable, a.MinSamples, a.Interval) == (1, 64, 32) and abs(a.Threshold - 0.05) < 1e-7
    cfg = T.get_config(); cfg.ScreenChunkCount = 2
    with pytest.raises(pt.B200ptError) as e:
        T.set_config(cfg)
    assert e.value.code == pt.ERR_WRONG_ARGUMENTS
    T.set_adaptive(Enable=0); T.set_config(cfg)
    with pytest.raises(pt.B200ptError) as e:
        T.set_adaptive(Enable=1)
    assert e.value.code == pt.ERR_WRONG_ARGUMENTS


@gpu
def test_cli_stops_when_every_pixel_has_converged(gpu_pt, tmp_path):
    import json
    exe = os.path.join(os.path.dirname(pt.LIB_PATH), "b200pt_render")
    hdr = str(tmp_path / "env.hdr"); util.write_rgbe(hdr, util.gltf_ref.synthetic_env(64, 32, 5)[..., :3])
    args = ["--scene", util.write_synthetic_gltf(tmp_path), "--env", hdr, "--luts", util.write_luts_dir(tmp_path / "luts"), "--size", "96", "64",
            "--depth", "4", "--batch", "6", "--quiet", "--spp", "64", "--out", str(tmp_path / "a.png")]
    r = subprocess.run([exe, *args, "--adaptive", "1e6,4,4"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    info = json.loads(r.stdout.strip().splitlines()[-1])
    assert info["spp"] == 4 and info["active_pixels"] == 0 and info["paths"] == 4 * 96 * 64   # --spp stays the cap; every pixel stopped at frame 4
    r = subprocess.run([exe, *args], capture_output=True, text=True)
    info = json.loads(r.stdout.strip().splitlines()[-1])
    assert r.returncode == 0 and info["spp"] == 64 and info["active_pixels"] == 96 * 64


# ---------------------------------------------------------------- no GPU needed

def test_adaptive_defaults_and_null_handles():
    a = pt.default_adaptive()
    assert (a.Enable, a.MinSamples, a.Interval) == (0, 64, 32) and a.Threshold == np.float32(0.01)
    assert C.sizeof(pt.Adaptive) == 16
    L = pt.lib()
    assert L.b200pt_default_adaptive(None) == pt.ERR_WRONG_ARGUMENTS
    assert L.b200pt_set_adaptive(None, C.byref(a)) == pt.ERR_WRONG_ARGUMENTS
    assert L.b200pt_get_adaptive(None, C.byref(a)) == pt.ERR_WRONG_ARGUMENTS
    assert L.b200pt_get_pixel_stats(None, None, None) == pt.ERR_WRONG_ARGUMENTS
    n = C.c_uint32()
    assert L.b200pt_active_pixels(None, C.byref(n)) == pt.ERR_WRONG_ARGUMENTS


@pytest.mark.parametrize("arg,ok", [("0.02", True), ("0.02,16", True), ("0.02,16,8", True), ("0", True),
                                    ("abc", False), ("-0.1", False), ("nan", False), ("inf", False), ("0.02,1", False), ("0.02,16,0", False),
                                    ("0.02,16,8,4", False), ("0.02,", False), ("0.02;16", False)])
def test_cli_parses_adaptive(arg, ok, tmp_path):
    exe = os.path.join(os.path.dirname(pt.LIB_PATH), "b200pt_render")
    missing = str(tmp_path / "missing")
    r = subprocess.run([exe, "--scene", missing + ".gltf", "--env", missing + ".hdr", "--luts", missing, "--out", str(tmp_path / "o.png"),
                        "--adaptive", arg, "--quiet"], capture_output=True, text=True, timeout=120)
    if ok:   # parsed: the run gets as far as the device / the missing files
        assert r.returncode not in (0, 2) and "usage:" not in r.stderr, r.stderr
    else:
        assert r.returncode == 2 and "--adaptive" in r.stderr, r.stderr
