"""CPU-side checks that the host runtime releases every CUDA resource it creates, on error paths too, and that the device view of the scene
holds only live blocks after a failed update: tests/native/alloc_faults.cpp links the built objects against shims of the CUDA runtime that
fail the k-th creation and track every live block, event and stream (no GPU needed)."""
import glob
import os
import re
import shutil
import subprocess

import pytest

import util


@pytest.fixture(scope="module")
def alloc_faults(tmp_path_factory):
    """stdout of the harness: one '<name>: <n> creations, <f> failed' line per case."""
    objs = sorted(glob.glob(os.path.join(util.ROOT, "vulkan-path-tracer_b200", "build", "*.o")))
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not objs or not os.path.exists(nvcc): pytest.skip("needs nvcc and the built objects")
    exe = str(tmp_path_factory.mktemp("alloc_faults") / "alloc_faults")
    cmd = [nvcc, "--cudart", "shared", "-std=c++17", "-O1", "-gencode", "arch=compute_90a,code=sm_90a", "-I" + os.path.join(util.ROOT, "vulkan-path-tracer_b200", "csrc"),
           "-I" + os.path.join(util.ROOT, "include"), os.path.join(util.ROOT, "tests", "native", "alloc_faults.cpp")] + objs + ["-lz", "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.stdout.strip().endswith("ok") and r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    return r.stdout


def _case(out, name):
    m = re.search(r"^" + re.escape(name) + r": (\d+) creations, (\d+) failed$", out, re.M)
    assert m, out
    return int(m.group(1)), int(m.group(2))


def test_engine_creation_failure_and_destroy_leave_nothing_live(alloc_faults):
    """b200pt_create with its k-th stream / event / block creation failing, for every k: nothing is live after the error return, and
    nothing after b200pt_destroy of the engine whose creation succeeded."""
    n, failed = _case(alloc_faults, "engine")
    assert n >= 20 and failed == 0


@pytest.mark.parametrize("name", ["lbvh_build", "ploc_build", "lbvh_ploc_rebuild", "bvh4_collapse_device", "lbvh_build_wide", "lbvh_build_wide_device",
                                  "lbvh_refit", "lbvh_refit (BVH4)"])
def test_bvh_builders_and_first_refit_release_at_every_failed_allocation(alloc_faults, name):
    """The k-th cudaMalloc of the builder fails, for every k: the failing call leaves nothing live, the successful call exactly its outputs
    (lbvh_build: shading records, tri_slot, the node / triangle block and the reference boxes it hands to lbvh_ploc_rebuild).  The first
    lbvh_refit of a tree allocates its refit state: a failing call leaves the tree without refit state and the next call succeeds, a
    successful call leaves exactly the tree and its refit state."""
    n, failed = _case(alloc_faults, name)
    assert n >= (1 if name == "lbvh_build_wide" else 2) and failed == 0   # lbvh_build_wide allocates one block, the BVH4


def test_lbvh_build_rejects_2_28_references_and_releases_every_block(alloc_faults):
    """Split counts that add up to 2^28 references (the leaf slot field is 28 bits): lbvh_build returns an error and every temporary it
    allocated before the check is released."""
    n, failed = _case(alloc_faults, "lbvh_build (2^28 references)")
    assert n == 7 and failed == 0


@pytest.mark.parametrize("name", ["set_env_map", "set_luts", "set_material"])
def test_failed_scene_updates_leave_a_device_view_of_live_blocks(alloc_faults, name):
    """An engine with a one-quad scene, an environment map and the lookup tables; the k-th allocation of set_env_map, set_luts or
    set_material's emissive rebuild fails, for every k.  After each call every non-null pointer of Engine::dev_scene lies in a live block
    and has_env / has_luts agree with the view.  A failed set_env_map / set_luts leaves no map / no tables, and path_trace and the
    shade, miss and bounce queries refuse with B200PT_ERR_NO_SCENE; a failed emissive rebuild keeps the previous tables; a successful call
    leaves exactly its new blocks, in the view."""
    n, failed = _case(alloc_faults, name)
    assert n == (2 if name == "set_material" else 3) and failed == 0
