"""Does adaptive sampling pay?  Error against a high-frame reference over GPU time, uniform sampling against adaptive sampling at three thresholds.

usage: python profiles/adaptive_quality.py [--frames 1024] [--ref-frames 4096] [--check 32] [--scenes cornell,glass,breakfast] [--out DIR]

For each scene: a reference image from the plain renderer (another base seed, so its noise is independent of the arms'), then every arm renders
`--check` frames per path_trace call up to `--frames`.  After each call the RGB RMSE against the reference is recorded beside the GPU time of the
calls so far (CUDA events on the handle's stream around path_trace + flush) and the paths traced.  Per scene the script prints, for each arm,
the time and paths it needs to reach the RMSE the uniform arm has after a quarter and after all of its frames (linear interpolation in log-log
between check points; "-" = not reached), and the card's name, power limit and max SM clock read in the same run.  Writes nothing but --out.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import util

SCENES = {   # name: (fixture, W, H, MaxDepth)
    "cornell": ("cornell_box", 1920, 1080, 8),
    "glass": ("cornell_box_glass", 540, 540, 16),
    "breakfast": ("breakfast_room", 960, 540, 8),
}
THRESHOLDS = (0.04, 0.02, 0.01)
MIN_SAMPLES, INTERVAL = 32, 32
REF_SEED = 0x5EED0001


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=60).stdout.strip().splitlines()[0]
    except Exception as e:   # the numbers below are still GPU times; the card line is then missing, and says so
        return f"unknown ({e})"


def tracer(scene, W, H, depth, stream):
    T = util.product_tracer(scene, W, H, MaxDepth=depth, MaxSamplesAccumulated=1 << 30)
    T.set_stream(stream.cuda_stream)
    return T


def run_arm(scene, W, H, depth, threshold, frames, check, ref, stream):
    import torch
    T = tracer(scene, W, H, depth, stream)
    if threshold is not None: T.set_adaptive(Enable=1, Threshold=threshold, MinSamples=MIN_SAMPLES, Interval=INTERVAL)
    T.path_trace(check, util.BASE_SEED); T.synchronize(); T.reset()      # module load and wave buffers outside the timed window
    paths0 = int(T.counters()["paths"])
    curve, ms, f = [], 0.0, 0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    while f < frames:
        e0.record(stream)
        done = T.path_trace(check, util.BASE_SEED)
        T.flush(); e1.record(stream); e1.synchronize()
        ms += e0.elapsed_time(e1); f += check
        img = T.get_hdr()[..., :3].astype(np.float64)
        rmse = float(np.sqrt(((img - ref) ** 2).mean()))
        curve.append(dict(frames=f, ms=ms, paths=int(T.counters()["paths"]) - paths0, rmse=rmse, active=T.active_pixels()))
        if done: break
    return curve


def time_to(curve, target):
    """(ms, paths) at which the curve first reaches `target`, log-log interpolation between check points"""
    prev = None
    for c in curve:
        if c["rmse"] <= target:
            if prev is None or prev["rmse"] <= c["rmse"]: return c["ms"], c["paths"]
            t = (np.log(prev["rmse"]) - np.log(target)) / (np.log(prev["rmse"]) - np.log(c["rmse"]))
            lerp = lambda a, b: float(np.exp(np.log(a) + t * (np.log(b) - np.log(a))))
            return lerp(prev["ms"], c["ms"]), lerp(prev["paths"], c["paths"])
        prev = c
    return None, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1024)
    ap.add_argument("--ref-frames", type=int, default=4096)
    ap.add_argument("--check", type=int, default=32)
    ap.add_argument("--scenes", default=",".join(SCENES))
    ap.add_argument("--out", default=None, help="directory for the curves as JSON")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available(): sys.exit("adaptive_quality.py measures GPU time: no CUDA device")
    stream = torch.cuda.Stream()
    print("card:", card())
    results = {}
    for name in args.scenes.split(","):
        scene, W, H, depth = SCENES[name]
        R = tracer(scene, W, H, depth, stream)
        for _ in range(0, args.ref_frames, 256): R.path_trace(256, REF_SEED)
        ref = R.get_hdr()[..., :3].astype(np.float64); del R
        arms = {"uniform": run_arm(scene, W, H, depth, None, args.frames, args.check, ref, stream)}
        for thr in THRESHOLDS:
            arms[f"adaptive {thr:g}"] = run_arm(scene, W, H, depth, thr, args.frames, args.check, ref, stream)
        u = arms["uniform"]
        targets = [u[len(u) // 4 - 1]["rmse"], u[-1]["rmse"]]
        print(f"\n{name}: {W}x{H}, depth {depth}, reference {args.ref_frames} frames; adaptive MinSamples {MIN_SAMPLES}, Interval {INTERVAL}")
        print(f"  {'arm':<16}{'frames':>7}{'Mpaths':>9}{'ms':>9}{'RMSE':>11}{'active':>9}" +
              "".join(f"   to RMSE {t:.3e}: ms / Mpaths" for t in targets))
        for arm, curve in arms.items():
            c = curve[-1]
            cells = []
            for t in targets:
                ms, paths = time_to(curve, t)
                cells.append(f"{'-':>22}" if ms is None else f"{ms:>13.1f} / {paths / 1e6:>7.1f}")
            print(f"  {arm:<16}{c['frames']:>7}{c['paths'] / 1e6:>9.1f}{c['ms']:>9.1f}{c['rmse']:>11.3e}{c['active']:>9}" + "   " + "   ".join(cells))
        results[name] = arms
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "adaptive_quality.json"), "w") as f: json.dump({"card": card(), "scenes": results}, f, indent=1)


if __name__ == "__main__":
    main()
