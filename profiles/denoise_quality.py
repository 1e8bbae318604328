"""Does the denoiser pay?  Error against a high-frame reference over GPU time, raw accumulation against the denoised image.

usage: python profiles/denoise_quality.py [--ref-frames 4096] [--frames 1024] [--scenes cornell,glass,breakfast] [--out DIR]

For each scene: a reference image from the plain renderer (another base seed, so its noise is independent), then one render with per-pixel
statistics on, up to --frames frames in power-of-two steps from 8.  At every step the RGB RMSE of the raw accumulation against the reference is
recorded beside the render's GPU time so far (CUDA events on the handle's stream around path_trace + flush); at 8 .. 256 frames the image is
also denoised with the default b200pt_denoise_params, and the RMSE of the denoised image is recorded with the device time of b200pt_denoise
(feature pass + filter, its elapsed_ms) and of the filter alone (b200pt_denoise_image on device buffers, CUDA events; the feature pass is the
difference).  The script prints the tables and the GPU time each curve needs to reach the raw error of 256 and of 1,024 frames (log-log
interpolation between steps; the denoised curve counts render + denoise time; "-" = not reached), and the card's name, power limit and max SM
clock read in the same run.  Writes nothing but --out.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "profiles"))
import numpy as np
import util
from adaptive_quality import SCENES, REF_SEED, card, tracer, time_to

DENOISE_UP_TO = 256


def filter_ms(T, stream, reps=5):
    """device time of the filter alone on this image size: b200pt_denoise_image on device copies of the handle's inputs"""
    import torch
    img = torch.from_numpy(T.get_hdr()).cuda()
    a, nd, v = (torch.from_numpy(x).cuda() for x in T.denoise_inputs())
    out = torch.empty_like(img)
    H, W = img.shape[:2]
    import vpt_b200 as pt
    p = pt.default_denoise()
    L = pt.lib()
    import ctypes as C
    call = lambda: T._ck(L.b200pt_denoise_image(T.h, W, H, C.c_void_p(img.data_ptr()), C.c_void_p(a.data_ptr()), C.c_void_p(nd.data_ptr()),
                                                 C.c_void_p(v.data_ptr()), C.byref(p), C.c_void_p(out.data_ptr()), 1))
    torch.cuda.synchronize(); call()                                   # scratch allocation outside the timed window
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(reps):
        e0.record(stream); call(); e1.record(stream); e1.synchronize(); ms.append(e0.elapsed_time(e1))
    return float(np.median(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1024)
    ap.add_argument("--ref-frames", type=int, default=4096)
    ap.add_argument("--scenes", default=",".join(SCENES))
    ap.add_argument("--out", default=None, help="directory for the curves as JSON")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available(): sys.exit("denoise_quality.py measures GPU time: no CUDA device")
    stream = torch.cuda.Stream()
    print("card:", card())
    results = {}
    for name in args.scenes.split(","):
        scene, W, H, depth = SCENES[name]
        R = tracer(scene, W, H, depth, stream)
        for _ in range(0, args.ref_frames, 256): R.path_trace(256, REF_SEED)
        ref = R.get_hdr()[..., :3].astype(np.float64); del R
        T = tracer(scene, W, H, depth, stream)
        T.set_track_variance(True)
        T.path_trace(8, util.BASE_SEED); T.synchronize(); T.denoise(); T.reset()   # module load, wave and denoise buffers outside the timed window
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        raw, den, ms, f, step = [], [], 0.0, 0, 8
        while f < args.frames:
            e0.record(stream); T.path_trace(step - f, util.BASE_SEED); T.flush(); e1.record(stream); e1.synchronize()
            ms += e0.elapsed_time(e1); f = step
            rmse = lambda img: float(np.sqrt(((img[..., :3].astype(np.float64) - ref) ** 2).mean()))
            raw.append(dict(frames=f, ms=ms, paths=f, rmse=rmse(T.get_hdr())))
            if f <= DENOISE_UP_TO:
                d_ms = T.denoise()
                fl = filter_ms(T, stream)
                den.append(dict(frames=f, render_ms=ms, ms=ms + d_ms, paths=f, rmse=rmse(T.get_denoised()), denoise_ms=d_ms, filter_ms=fl, feature_ms=d_ms - fl))
            step *= 2
        results[name] = dict(raw=raw, denoised=den)
        print(f"\n{name}: {W}x{H}, depth {depth}, reference {args.ref_frames} frames, denoiser defaults")
        print(f"  {'frames':>7}{'render ms':>11}{'RMSE raw':>11}{'RMSE den':>11}{'ratio':>7}{'denoise ms':>12}{'features':>10}{'filter':>9}")
        for r in raw:
            d = next((x for x in den if x["frames"] == r["frames"]), None)
            cells = f"{d['rmse']:>11.3e}{d['rmse'] / r['rmse']:>7.3f}{d['denoise_ms']:>12.2f}{d['feature_ms']:>10.2f}{d['filter_ms']:>9.2f}" if d else ""
            print(f"  {r['frames']:>7}{r['ms']:>11.1f}{r['rmse']:>11.3e}" + cells)
        for target_frames in (256, 1024):
            t = next((r["rmse"] for r in raw if r["frames"] == target_frames), None)
            if t is None: continue
            a, _ = time_to(raw, t); b, _ = time_to(den, t)
            print(f"  to the raw RMSE of {target_frames} frames ({t:.3e}): raw {a:.1f} ms, denoised " + ("-" if b is None else f"{b:.1f} ms"))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "denoise_quality.json"), "w") as f: json.dump({"card": card(), "scenes": results}, f, indent=1)


if __name__ == "__main__":
    main()
