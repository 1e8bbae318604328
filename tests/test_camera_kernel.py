"""k_camera (camera rays generated and traced in one kernel, scenes whose BVH sits in shared memory) against the k_raygen + k_extend pair it
replaces (B200PT_CAMERA=0).  Both write the same path state, trace the same closest-hit query and fill the same queues, so images must agree
bit for bit and every work counter must agree exactly; only kernel_launches drops, by one per wave and sample.
"""
import numpy as np
import pytest

import util

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pt():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import vpt_b200
    return vpt_b200


def _four_classes(T):
    """a rough conductor, a glass object with a scattering medium inside and a mixed-lobe material: all four material classes, so the
    class queues (not the one-class pair) are filled"""
    n = T.material_count()
    m = T.get_material(1 % n); m.Metallic = 1.0; m.Roughness = 0.3; T.set_material(1 % n, m)
    m = T.get_material(2 % n); m.Metallic = 0.0; m.Transmission = 1.0; m.IOR = 1.5; m.Roughness = 0.05
    m.MediumDensity = 2.0; m.MediumAnisotropy = 0.3; m.MediumColor[0], m.MediumColor[1], m.MediumColor[2] = 0.9, 0.5, 0.3
    T.set_material(2 % n, m)
    m = T.get_material(3 % n); m.Metallic = 0.4; m.Transmission = 0.3; m.Roughness = 0.4; T.set_material(3 % n, m)


WORK = ("paths", "extend_rays", "shade_invocations", "surface_hits", "misses", "shadow_rays", "medium_events")


def _render(monkeypatch, camera, W, H, frames, depth=6, edit=None, partition=None, scene="cornell_box", **cfg):
    monkeypatch.setenv("B200PT_CAMERA", camera)
    T = util.product_tracer(scene, W, H, MaxDepth=depth, **cfg)
    if edit: edit(T)
    if partition: T.set_partition(*partition)
    T.path_trace(frames, util.BASE_SEED)                      # one call on a fresh handle: the counters hold exactly this call's work
    c = T.counters()
    return T.get_hdr().copy(), {k: c[k] for k in WORK + ("kernel_launches",)}, c["waves"]


def _check(monkeypatch, W=96, H=70, frames=4, samples=1, **kw):
    img1, c1, waves = _render(monkeypatch, "1", W, H, frames, **kw)
    img0, c0, _ = _render(monkeypatch, "0", W, H, frames, **kw)
    assert np.isfinite(img0).all() and img0[..., :3].max() > 0
    assert np.array_equal(img1.view(np.uint32), img0.view(np.uint32)), int((img1 != img0).any(axis=-1).sum())
    assert {k: c1[k] for k in WORK} == {k: c0[k] for k in WORK}
    assert c0["kernel_launches"] - c1["kernel_launches"] == waves * samples      # k_camera ran: one launch instead of two per wave and sample
    return img1, c1


def _check_fuse(monkeypatch, fuse, **kw):
    """_check under B200PT_FUSE=fuse.  2 selected the bounce kernel, which is gone: an unsupported value must run the default pipeline, so
    its image and every counter (kernel_launches included) must equal those of a render without the variable."""
    monkeypatch.setenv("B200PT_FUSE", fuse)
    img, c = _check(monkeypatch, **kw)
    if fuse == "2":
        monkeypatch.delenv("B200PT_FUSE")
        img_d, c_d = _check(monkeypatch, **kw)
        assert np.array_equal(img.view(np.uint32), img_d.view(np.uint32)) and c == c_d, (c, c_d)


@pytest.mark.parametrize("fuse", ["0", "1", "2"])
def test_camera_kernel_matches_raygen_extend_per_pipeline(pt, fuse, monkeypatch):
    _check_fuse(monkeypatch, fuse, depth=8)


@pytest.mark.parametrize("fuse", ["1", "2"])
def test_camera_kernel_matches_with_four_material_classes(pt, fuse, monkeypatch):
    _check_fuse(monkeypatch, fuse, W=128, H=96, depth=8, edit=_four_classes)


def test_camera_kernel_matches_with_screen_chunks(pt, monkeypatch):
    # 50 x 31 in 2 x 2 chunks: the last chunk row and column overhang the image (born-dead paths, still traced)
    _check(monkeypatch, W=50, H=31, frames=4 * 4, ScreenChunkCount=2)


def test_camera_kernel_matches_with_two_samples_per_frame(pt, monkeypatch):
    _check(monkeypatch, frames=3, samples=2, SamplesPerFrame=2)


@pytest.mark.parametrize("rank", [0, 1])
def test_camera_kernel_matches_on_a_tile_partition(pt, rank, monkeypatch):
    _check(monkeypatch, partition=(rank, 2, 16))


@pytest.mark.parametrize("fif", [1, 0])
def test_camera_kernel_matches_across_frames_in_flight(pt, fif, monkeypatch):
    _check(monkeypatch, frames=6, FramesInFlight=fif)


def test_camera_kernel_matches_in_big_shared_memory_mode(pt, monkeypatch):
    # the glass scene's 108 KiB BVH: one 512-thread CTA per SM and the hierarchical walk instead of the flat one
    monkeypatch.setenv("B200PT_SMEM_BIG", "1")
    _check(monkeypatch, W=96, H=96, frames=2, depth=12, scene="cornell_box_glass")


def test_camera_kernel_matches_with_depth_of_field(pt, monkeypatch):
    # camera rays from a lens disk start off the camera position: k_camera's warps fall back from the fixed-origin table to the plain walk
    _check(monkeypatch, DepthOfFieldStrength=0.05, FocusDistance=4.0)
