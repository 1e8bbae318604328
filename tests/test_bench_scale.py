"""The regime bench.py reports from, checked: full-size images of all four workloads, auto and explicit wave sizes past 2^24 paths, two
overlapping wave contexts across path_trace calls, a caller's torch stream and the device-pointer copies.

The sampler is keyed on pixel and dispatch, so wave size, overlap, call split and stream must not change a single bit of the image: every
comparison with the serial render (FramesInFlight = 1, B200PT_OVERLAP=0, the handle's own stream) is exact, work counters included.  Rows of each
benchmark image are also rendered by the CPU oracle, at test_gpu_parity's matched-seed bar for accumulated images.

Synchronisation slips only show when the work they should order is still running, so each ordering is checked where a missing wait gives a
wrong value every time, not by luck:
- a copy on the caller's stream that must follow a render is enqueued right behind a one-frame wave on context 0 and an eight-frame wave on
  context 1, and the test asserts it was enqueued well inside that render's duration;
- a render, copy or kernel that must follow work on the caller's stream has a long device-side sleep (torch.cuda._sleep, a spin loop) on that
  stream right before it, and an event behind the sleep must still be pending once the calls under test are enqueued: a host
  synchronisation in between (growing buffers does one, so the handle's buffers are grown first) would drain the sleep.
Nothing here provokes a fault.
"""
import contextlib
import ctypes
import importlib.util
import json
import math
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import util  # noqa: E402

WORK = ("paths", "extend_rays", "shade_invocations", "surface_hits", "misses", "shadow_rays", "medium_events")
BYTES_PER_PATH = 400          # what path_trace's auto wave size budgets per path and context (engine.cu); the arrays take ~380 B
SLEEP_CYCLES = 1_000_000_000  # ~0.5 s of SM clock: far longer than a few frames of the Cornell box at 1080p and the host calls behind it
SWEEP = "cornell_1080p_d8"    # the default workload; the cheapest scene, so the sweep spends its time on wave sizes, not on shading


def _load_bench():
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    m = importlib.util.module_from_spec(spec); spec.loader.exec_module(m)
    return m


bench = _load_bench()
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pt():
    import torch
    if not torch.cuda.is_available(): pytest.skip("no CUDA device")
    import vpt_b200
    return vpt_b200


@pytest.fixture(scope="module")
def env4k():
    return bench.synthetic_env_4k()


@contextlib.contextmanager
def overlap_off():
    """B200PT_OVERLAP=0 for the path_trace calls inside: one wave at a time on the handle's stream (read at every call)."""
    old = os.environ.get("B200PT_OVERLAP")
    os.environ["B200PT_OVERLAP"] = "0"
    try: yield
    finally:
        if old is None: del os.environ["B200PT_OVERLAP"]
        else: os.environ["B200PT_OVERLAP"] = old


def bench_handle(pt, env, workload, frames_in_flight):
    """A handle set up the way bench.py sets up its own: same fixture, map, tables, config and partition."""
    scene, W, H, depth = bench.WORKLOADS[workload]
    T = pt.PathTracer(0)
    T.set_scene(util.scene_dict(scene)); T.set_env_map(env); T.set_luts(*util.luts())
    T.set_config(pt.default_config(MaxDepth=depth, MaxSamplesAccumulated=0x7FFFFFFF, FramesInFlight=frames_in_flight))
    T.resize(W, H); T.set_partition(0, 1, bench.BAND_ROWS)
    return T


def work(T):
    c = T.counters()
    return {k: c[k] for k in WORK}


def delta(a, b):
    return {k: b[k] - a[k] for k in WORK}


class Serial:
    """The reference render: FramesInFlight = 1, B200PT_OVERLAP=0, the handle's own stream.  advance_to(n) renders frames up to n and returns
    (image, work counters of frames 0 .. n); one call equals several calls (test_samples_per_frame_and_running_mean)."""

    def __init__(self, pt, env, workload):
        self.T = bench_handle(pt, env, workload, 1)
        self.frames = 0; self.w0 = work(self.T)

    def advance_to(self, n):
        assert n >= self.frames
        if n > self.frames:
            with overlap_off(): self.T.path_trace(n - self.frames, bench.BASE_SEED)
            self.frames = n
        return self.T.get_hdr(), delta(self.w0, work(self.T))

    def close(self): self.T.close()


def assert_same(got, want, what):
    if np.array_equal(got, want): return
    bad = np.any(got != want, axis=-1) if got.ndim == 3 else (got != want)
    rows = np.nonzero(bad.reshape(bad.shape[0], -1).any(axis=1))[0]
    d = np.abs(got.astype(np.float64) - want.astype(np.float64))
    pytest.fail(f"{what}: {int(bad.sum())} pixels differ from the serial render (rows {rows[:8].tolist()}{' ...' if len(rows) > 8 else ''}), "
                f"max |diff| {float(np.nanmax(d)):.3g}")


# ---------------------------------------------------------------- 1 + 2: bench.py's own output at full size
_BENCH = {}


def bench_run(pt, env, workload, tmp_path_factory):
    """bench.py in a subprocess (auto wave size, overlap, caller stream) -> (its dumped image, its JSON line, the serial render of the same frames,
    the serial work counters of the timed step)."""
    if workload in _BENCH: return _BENCH[workload]
    out_dir = tmp_path_factory.mktemp("bench_" + workload)
    import torch
    free, _ = torch.cuda.mem_get_info()
    scene, W, H, _ = bench.WORKLOADS[workload]
    print(f"\n{workload}: free HBM {free / 2**30:.1f} GiB -> auto wave size about {min(64 << 20, free // 4 // BYTES_PER_PATH // 2) / 2**20:.1f} M paths "
          f"per context ({W}x{H} = {W * H / 2**20:.2f} M paths per frame)")
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--workload", workload, "--warmup", "1", "--steps", "1",
           "--frames-per-step", "32", "--no-cpu-baseline", "--dump-outputs", str(out_dir)]
    t0 = time.perf_counter()
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-4000:]
    line = json.loads([l for l in r.stdout.splitlines() if l.startswith("{")][-1])
    assert not os.path.exists(os.path.join(out_dir, "hdr_index.npy")), "the full image fits the dump budget: hdr.npy must not be a sample"
    got = np.load(os.path.join(out_dir, "hdr.npy"))
    F, steps = line["config"]["frames_per_step"], line["steps"]
    frames = (line["warmup"] + steps) * F                        # bench.py raises --warmup to its minimum; the JSON line says what ran
    S = Serial(pt, env, workload)
    try:
        _, w_before = S.advance_to(frames - steps * F)
        ref, w_after = S.advance_to(frames)
    finally:
        S.close()
    print(f"{workload}: bench.py {time.perf_counter() - t0:.1f} s incl. serial render, {frames} frames, {line['value']:.0f} Mpaths/s")
    _BENCH[workload] = (got, line, ref, delta(w_before, w_after), frames)
    return _BENCH[workload]


@pytest.mark.parametrize("workload", sorted(bench.WORKLOADS))
def test_bench_image_equals_the_serial_render(pt, env4k, workload, tmp_path_factory):
    got, line, ref, w_timed, frames = bench_run(pt, env4k, workload, tmp_path_factory)
    scene, W, H, _ = bench.WORKLOADS[workload]
    assert got.shape == (H, W, 4) and np.isfinite(got).all()
    assert_same(got, ref, f"{workload}: bench.py's image after {frames} frames")
    # the timed step's work counters: bench.py differences the device counters around its timed steps
    steps = line["steps"]
    assert {k: line["counters_per_step"][k] * steps for k in WORK} == {k: float(v) for k, v in w_timed.items()}


def oracle_rows(workload, rows, frames):
    """The oracle's render of single rows of the full-size image, all `frames` frames: one row per call (rank = row, world = H, 1-row bands), one
    thread per row."""
    scene, W, H, depth = bench.WORKLOADS[workload]
    S, cfg = bench.oracle_scene_for(scene, depth)             # the benchmark's 4K map and its alias table, built by the oracle
    img = np.zeros((H, W, 4), np.float32)
    def one(y): S.render(cfg, W, H, frames, bench.BASE_SEED, image=img, rank=y, world=H, band_rows=1, nthreads=1)
    with ThreadPoolExecutor(len(rows)) as ex: list(ex.map(one, rows))
    return img


# rel L2 of the four rows against the serial render (= bench.py's image), 128 frames, measured on an H100 80GB HBM3 (700 W power limit):
#   cornell_1080p_d8 3.3e-7, glass_1080sq_d16 3.2e-7, breakfast_1080p_d8 7.0e-4 (rows 501 and 528: 6.7e-4, 7.8e-4), viking_1080sq_d8 2.4e-4.
# Both images are deterministic at matched seeds, so these numbers only move when the kernels or the oracle change.
@pytest.mark.parametrize("workload", sorted(bench.WORKLOADS))
def test_bench_rows_match_the_oracle(pt, env4k, workload, tmp_path_factory):
    _, _, ref, _, frames = bench_run(pt, env4k, workload, tmp_path_factory)
    scene, W, H, _ = bench.WORKLOADS[workload]
    lum = ref[1:H - 1, :, :3].astype(np.float64).sum(axis=(1, 2))
    rows = sorted({0, H - 1, 1 + int(np.argmax(lum)), bench.BAND_ROWS * (H // (2 * bench.BAND_ROWS))})   # edges, brightest row, a band boundary
    t0 = time.perf_counter()
    orc_img = oracle_rows(workload, rows, frames)
    l2 = {y: util.rel_l2(ref[y, :, :3], orc_img[y, :, :3]) for y in rows}
    l2_all = util.rel_l2(ref[rows, :, :3], orc_img[rows, :, :3])
    print(f"\n{workload}: oracle rows {rows} ({frames} frames, {time.perf_counter() - t0:.1f} s): rel L2 {l2_all:.3g}; per row "
          + ", ".join(f"{y}: {v:.3g}" for y, v in l2.items()))
    assert l2_all < 1e-3, (l2_all, l2)


# ---------------------------------------------------------------- 3: explicit wave sizes, overlap and call splits
def test_wave_size_overlap_and_call_split_sweep(pt, env4k):
    """The same frames at FramesInFlight just below and above 2^24 and 2^25 paths per wave, the largest that fits, auto, overlap on and off, and
    calls split unevenly: every image equals the serial one bit for bit and every work counter equals it exactly."""
    import torch
    scene, W, H, _ = bench.WORKLOADS[SWEEP]
    P = W * H
    below24, below25 = (1 << 24) // P, (1 << 25) // P          # 8 and 16 frames of 1080p: F * P just below 2^24 / 2^25, F + 1 just above
    S = Serial(pt, env4k, SWEEP)
    T = bench_handle(pt, env4k, SWEEP, 1)
    try:
        free, _ = torch.cuda.mem_get_info()
        budget = free // 2                                        # the GPU is shared: leave at least half of what is free now
        fmax = min(256, budget // (BYTES_PER_PATH * P * 2))
        sizes = [below24, below24 + 1, below25, below25 + 1] + ([fmax] if fmax > below25 + 1 else [])
        cases = [(f, True, [2 * f]) for f in sizes]               # (FramesInFlight, overlap, path_trace calls): two equal waves, one per context
        cases += [(below24, False, [2 * below24]), (below25 + 1, False, [2 * below25 + 2]),
                  # the 1-frame wave queues on context 0 behind 2 frames while context 1 runs 9: its resolve must still come last
                  (below24 + 1, True, [2, below24 + 1, 1]), (below24 + 1, False, [2, below24 + 1, 1]),
                  (0, True, [32]), (0, True, [5, 27, 1]), (0, False, [5, 27, 1])]     # auto wave size, as bench.py runs
        # the handle keeps its largest wave buffers (both contexts): explicit sizes in ascending order, so each case runs in buffers of its own
        # wave size and the budget check above holds for what the handle then holds; the auto cases, sized by the engine, last
        cases.sort(key=lambda c: (c[0] == 0, c[0]))
        serial = {n: S.advance_to(n) for n in sorted({sum(c[2]) for c in cases})}
        for fif, overlap, calls in cases:
            per_wave = P * min(fif, max(calls))
            if fif != 0 and per_wave * BYTES_PER_PATH * (2 if overlap else 1) > budget:
                print(f"\nskip FramesInFlight={fif}: {per_wave / 2**20:.0f} M paths per wave do not fit in half of the free HBM"); continue
            ref, w_ref = serial[sum(calls)]
            T.set_config(pt.default_config(MaxDepth=bench.WORKLOADS[SWEEP][3], MaxSamplesAccumulated=0x7FFFFFFF, FramesInFlight=fif))
            T.reset()
            w0 = work(T)
            with (contextlib.nullcontext() if overlap else overlap_off()):
                for n in calls: T.path_trace(n, bench.BASE_SEED)   # asynchronous: the calls overlap each other
            got = T.get_hdr()
            w = delta(w0, work(T))
            waves = T.counters()["waves"]                          # of the last call
            last_wave_frames = math.ceil(calls[-1] / waves)
            label = f"FramesInFlight={fif} overlap={'on' if overlap else 'off'} calls={calls}"
            print(f"\n{label}: last call {waves} waves of {last_wave_frames * P / 2**20:.1f} M paths ({last_wave_frames * P / 2**24:.2f} x 2^24)")
            if fif != 0 and len(calls) == 1:
                assert waves == math.ceil(calls[0] / fif), label       # the waves really were FramesInFlight frames
            assert_same(got, ref, label)
            assert w == w_ref, (label, w, w_ref)
    finally:
        T.close(); S.close()


# ---------------------------------------------------------------- 4: device-pointer copies on a caller's stream
def device_setup(pt, env):
    """(handle on a caller torch stream, serial handle, the stream).  The handle's two wave contexts (8 frames each) and post buffers are grown
    here: growing them synchronises the caller's stream on the host, which would drain a sleep the test puts on it before anything waits on it.
    After this, wave w of the test runs on context w & 1."""
    import torch
    T = bench_handle(pt, env, SWEEP, 8)
    s = torch.cuda.Stream()
    T.set_stream(s.cuda_stream)
    T.path_trace(16, bench.BASE_SEED); T.post_process(); T.synchronize(); T.reset()   # two waves: the next one runs on context 0
    torch.mul(torch.ones(4, device="cuda"), 2.0); torch.cuda.synchronize()           # the torch kernels used below are loaded
    return T, Serial(pt, env, SWEEP), s


def sleep_on(s):
    """A long device-side sleep on s, and an event behind it: still pending when checked = no host call has waited for the sleep so far."""
    import torch
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
        ev = torch.cuda.Event(); ev.record(s)
    return ev


def assert_pending(ev, what):
    assert not ev.query(), f"{what}: the host waited out the sleep, so it no longer delays the producer"


def render_in_flight(T, s):
    """path_trace(1) then path_trace(8): a one-frame wave on context 0 and an eight-frame wave on context 1, enqueued without delay.  A copy the
    caller enqueues on s right after this meets context 1 still rendering, unless the engine makes s wait for it."""
    T.path_trace(1, bench.BASE_SEED); T.path_trace(8, bench.BASE_SEED)
    return time.perf_counter()


def assert_window(T, host_ms, what):
    """The consumer was enqueued host_ms after render_in_flight returned, well inside context 1's render (counters' ms_total: first kernel of
    the last call's wave .. its resolve), so a missing wait on either context lands it mid-render instead of racing a resolve."""
    render_ms = T.counters()["ms_total"]
    assert host_ms < render_ms / 4, f"{what}: enqueued {host_ms:.2f} ms after the render, which took {render_ms:.2f} ms"


def test_get_hdr_into_device_on_a_caller_stream(pt, env4k):
    import torch
    T, S, s = device_setup(pt, env4k)
    scene, W, H, _ = bench.WORKLOADS[SWEEP]
    try:
        with torch.cuda.stream(s):
            buf1 = torch.empty((H, W, 4), dtype=torch.float32, device="cuda"); buf2 = torch.empty_like(buf1)
            t = render_in_flight(T, s)
            host_ms = (time.perf_counter() - t) * 1e3
            T.get_hdr_into_device(buf1.data_ptr())                # right behind the asynchronous calls: must wait for both contexts
            assert_window(T, host_ms, "first copy")
            ev = sleep_on(s)                                      # delays the copy below; the next call's resolve must wait for it
            T.get_hdr_into_device(buf2.data_ptr())
            T.path_trace(4, bench.BASE_SEED)
            assert_pending(ev, "second copy")
        s.synchronize()
        final = T.get_hdr()
        assert_same(buf1.cpu().numpy(), S.advance_to(9)[0], "get_hdr_into_device after 1 + 8 frames")
        assert_same(buf2.cpu().numpy(), S.advance_to(9)[0], "get_hdr_into_device after 9 frames, the next call in flight")
        assert_same(final, S.advance_to(13)[0], "get_hdr after 13 frames")
    finally:
        T.close(); S.close()


def test_set_hdr_from_device_written_by_a_torch_kernel(pt, env4k):
    import torch
    T, S, s = device_setup(pt, env4k)
    scene, W, H, _ = bench.WORKLOADS[SWEEP]
    try:
        x = np.random.default_rng(11).uniform(0.0, 3.0, (H, W, 4)).astype(np.float32)
        xd = torch.from_numpy(x).cuda(); torch.cuda.synchronize()
        with torch.cuda.stream(s):
            src = torch.zeros_like(xd); src2 = torch.zeros_like(xd); torch.cuda.synchronize()
            ev = sleep_on(s)
            torch.mul(xd, 2.0, out=src)                           # the source, written on the caller's stream right behind the sleep
            assert_pending(ev, "set_hdr_from_device")
            T.set_hdr_from_device(src.data_ptr())                 # must copy after the kernel
            got1 = T.get_hdr()
            t = render_in_flight(T, s)
            torch.mul(xd, 3.0, out=src2)
            host_ms = (time.perf_counter() - t) * 1e3
            T.set_hdr_from_device(src2.data_ptr())                # must land after both contexts' frames
            assert_window(T, host_ms, "set_hdr_from_device")
            T.path_trace(4, bench.BASE_SEED)                      # folds frames 9 .. 12 into 3 x
        s.synchronize()
        got2 = T.get_hdr()
        assert_same(got1, x * 2.0, "set_hdr_from_device behind a torch kernel")
        S.advance_to(9); S.T.set_hdr(x * 3.0)
        assert_same(got2, S.advance_to(13)[0], "1 + 8 frames, set_hdr_from_device, 4 frames")
    finally:
        T.close(); S.close()


def test_post_rows_into_device_on_a_caller_stream(pt, env4k):
    import torch
    T, S, s = device_setup(pt, env4k)
    scene, W, H, _ = bench.WORKLOADS[SWEEP]
    y0, y1 = bench.post_row_block(H, 1, 2)                        # the second rank's block of the post workload
    try:
        with torch.cuda.stream(s):
            ldr1 = torch.empty((H, W, 4), dtype=torch.uint8, device="cuda"); ldr2 = torch.empty((y1 - y0, W, 4), dtype=torch.uint8, device="cuda")
            t = render_in_flight(T, s)
            host_ms = (time.perf_counter() - t) * 1e3
            T.post_process_rows(0, H)                             # must read the image after both contexts' frames
            T.get_ldr_rows_into_device(0, H, ldr1.data_ptr())
            assert_window(T, host_ms, "first post chain")
            T.path_trace(4, bench.BASE_SEED)
            T.flush()
            ev = sleep_on(s)                                      # delays the post chain; the next call's resolve must wait for it
            T.post_process_rows(y0, y1)
            T.get_ldr_rows_into_device(y0, y1, ldr2.data_ptr())
            T.path_trace(4, bench.BASE_SEED)
            assert_pending(ev, "second post chain")
        s.synchronize()
        S.advance_to(9); S.T.post_process_rows(0, H); want1 = S.T.get_ldr_rows(0, H)
        S.advance_to(13); S.T.post_process_rows(y0, y1); want2 = S.T.get_ldr_rows(y0, y1)
        assert_same(ldr1.cpu().numpy(), want1, "post_process_rows(0, H) after 1 + 8 frames")
        assert_same(ldr2.cpu().numpy(), want2, f"post_process_rows({y0}, {y1}) after 13 frames, the next call in flight")
        assert_same(T.get_hdr(), S.advance_to(17)[0], "get_hdr after 17 frames")
    finally:
        T.close(); S.close()


def test_hdr_device_ptr_on_a_caller_stream(pt, env4k):
    import torch
    T, S, s = device_setup(pt, env4k)
    scene, W, H, _ = bench.WORKLOADS[SWEEP]
    try:
        with torch.cuda.stream(s):
            snap1 = torch.empty((H, W, 4), dtype=torch.float32, device="cuda"); snap2 = torch.empty_like(snap1)
            ev = sleep_on(s)                                      # the resolves below wait for it (image_free_ev_)
            T.path_trace(1, bench.BASE_SEED)
            T.path_trace(3, bench.BASE_SEED)
            assert_pending(ev, "hdr_device_ptr")
            p = ctypes.c_void_p()
            T._ck(T.L.b200pt_hdr_device_ptr(T.h, ctypes.byref(p)))   # must wait for the render on the host
            view = torch.as_tensor(_DeviceArray(p.value, (H, W, 4)), device="cuda")
            snap1.copy_(view)
            t = render_in_flight(T, s)
            host_ms = (time.perf_counter() - t) * 1e3
            T.flush()                                             # the caller's own work on the pointer follows every launched wave
            snap2.copy_(view)
            assert_window(T, host_ms, "flush")
        s.synchronize()
        assert view.data_ptr() == p.value
        assert_same(snap1.cpu().numpy(), S.advance_to(4)[0], "hdr_device_ptr after 1 + 3 frames")
        assert_same(snap2.cpu().numpy(), S.advance_to(13)[0], "hdr_device_ptr after 1 + 8 more frames and flush")
    finally:
        T.close(); S.close()


class _DeviceArray:
    """A device pointer as a torch tensor without a copy (__cuda_array_interface__)."""

    def __init__(self, ptr, shape):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": "<f4", "data": (ptr, False), "version": 2, "strides": None}
