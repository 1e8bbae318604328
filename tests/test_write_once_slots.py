"""Sample slots are reused across calls without being cleared where every path of a sub-wave is known to end exactly once (WAVE_STORE:
the path end stores its radiance instead of adding it to the slot).  A handle whose slots still hold another seed's radiance must render
exactly what a fresh handle renders: the same image bit for bit and the same work.  The cases cover every pipeline that reaches a path end:
the two bounce pipelines (and an unsupported B200PT_FUSE value, which must run the default one) with and without k_camera, a second sample per frame (the slot is accumulated, the RNG state carried), chunked
dispatch (overhang paths keep their full camera state), a BVH outside shared memory (k_raygen + the dynamic-fetch kernels), a medium
(the bounce loop can stop on its runaway guard, so the slots are cleared as before) and a volume (pre-pass pipeline, cleared as before).
"""
import numpy as np
import pytest

import util

pytestmark = pytest.mark.gpu

OTHER_SEED = 0x5EED0001
WORK = ("paths", "extend_rays", "shade_invocations", "surface_hits", "misses", "shadow_rays", "medium_events", "kernel_launches")
FOG = dict(CornerMin=(-4.0, -4.0, -10.0), CornerMax=(4.5, 3.0, -1.0), Density=0.35, Color=(0.8, 0.7, 0.6), Anisotropy=0.4)


@pytest.fixture(scope="module")
def pt():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import vpt_b200
    return vpt_b200


def _four_classes(T):
    """all four material classes, one of them glass with a scattering medium inside (as in test_camera_kernel.py)"""
    n = T.material_count()
    m = T.get_material(1 % n); m.Metallic = 1.0; m.Roughness = 0.3; T.set_material(1 % n, m)
    m = T.get_material(2 % n); m.Metallic = 0.0; m.Transmission = 1.0; m.IOR = 1.5; m.Roughness = 0.05
    m.MediumDensity = 2.0; m.MediumAnisotropy = 0.3; m.MediumColor[0], m.MediumColor[1], m.MediumColor[2] = 0.9, 0.5, 0.3
    T.set_material(2 % n, m)
    m = T.get_material(3 % n); m.Metallic = 0.4; m.Transmission = 0.3; m.Roughness = 0.4; T.set_material(3 % n, m)


def _render(T, dispatches, seed, c0):
    """one call; the image and the work it added to the handle's cumulative counters (c0: their values before the call)"""
    T.path_trace(dispatches, seed)
    c1 = T.counters()
    return T.get_hdr().copy(), {k: c1[k] - c0[k] for k in WORK}


def _check(monkeypatch, env=None, scene="cornell_box", W=64, H=48, frames=3, depth=6, edit=None, **cfg):
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    S = cfg.get("ScreenChunkCount", 1)
    n = frames * S * S

    def tracer():
        T = util.product_tracer(scene, W, H, MaxDepth=depth, **cfg)
        if edit: edit(T)
        return T

    used = tracer()
    # two calls: consecutive waves alternate between two sets of wave buffers, so both hold another seed's radiance afterwards
    used.path_trace(n, OTHER_SEED)
    used.path_trace(n, OTHER_SEED + 1)
    used.reset()
    img_used, c_used = _render(used, n, util.BASE_SEED, used.counters())
    img_fresh, c_fresh = _render(tracer(), n, util.BASE_SEED, dict.fromkeys(WORK, 0))   # a fresh handle's counters start at zero
    assert np.isfinite(img_fresh).all() and img_fresh[..., :3].max() > 0
    assert np.array_equal(img_used.view(np.uint32), img_fresh.view(np.uint32)), int((img_used != img_fresh).any(axis=-1).sum())
    assert c_used == c_fresh
    return img_fresh, c_fresh


def _check_fuse(monkeypatch, fuse, env=None, **kw):
    """_check under B200PT_FUSE=fuse.  2 selected the bounce kernel, which is gone: an unsupported value must run the default pipeline, so
    its image and every counter (kernel_launches included) must equal those of a render without the variable."""
    img, c = _check(monkeypatch, dict(env or {}, B200PT_FUSE=fuse), **kw)
    if fuse == "2":
        monkeypatch.delenv("B200PT_FUSE")
        img_d, c_d = _check(monkeypatch, env, **kw)
        assert np.array_equal(img.view(np.uint32), img_d.view(np.uint32)) and c == c_d, (c, c_d)


@pytest.mark.parametrize("camera", ["0", "1"])
@pytest.mark.parametrize("fuse", ["0", "1", "2"])
def test_reused_slots_match_a_fresh_handle_per_pipeline(pt, fuse, camera, monkeypatch):
    _check_fuse(monkeypatch, fuse, {"B200PT_CAMERA": camera}, depth=8)


@pytest.mark.parametrize("camera", ["0", "1"])
def test_reused_slots_match_with_two_samples_per_frame(pt, camera, monkeypatch):
    _check(monkeypatch, {"B200PT_CAMERA": camera}, SamplesPerFrame=2)


@pytest.mark.parametrize("fuse", ["0", "1"])
def test_reused_slots_match_with_screen_chunks(pt, fuse, monkeypatch):
    # 50 x 31 in 2 x 2 chunks: the last chunk row and column overhang the image
    _check(monkeypatch, {"B200PT_FUSE": fuse}, W=50, H=31, ScreenChunkCount=2)


def test_reused_slots_match_with_bvh_outside_shared_memory(pt, monkeypatch):
    _check(monkeypatch, scene="cornell_box_glass", W=48, H=48, frames=2, depth=8)


@pytest.mark.parametrize("fuse", ["1", "2"])
def test_reused_slots_match_with_a_medium(pt, fuse, monkeypatch):
    _check_fuse(monkeypatch, fuse, W=96, H=64, depth=8, edit=_four_classes)


def test_reused_slots_match_with_a_volume(pt, monkeypatch):
    _check(monkeypatch, Volumes=[FOG])
