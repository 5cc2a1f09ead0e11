"""Framerate shaper (hb_filter_vfr_cuda) and its motion metric (hbcu_motion_metric_*) on one GPU.

metric         device time per frame from CUDA events around K enqueues (hbcu_motion_metric_mark / elapsed_ms) on
               torch-owned device frames, at 1080p and 4K, 8 and 10 bits (all on the fast path: the job is >= 1920 wide).
               `bytes` per frame from shapes: the new frame's luma read once, its reduced image written, the previous
               reduced image read; `hbm share` is those bytes at 3.35 TB/s (H100 HBM3 peak) over the measured time
chain fps      wall-clock frames/s of upload -> vfr -> NLMeans (y-strength=6) -> download on a 1080p 8-bit 29.97 clip,
               vfr mode=1 (CFR 23.976: the metric runs and drops are read) against mode=0 (no metric); the difference is
               the metric's cost in a real chain.  Three alternated runs each, median reported
cpu vfr fps    the reference's hb_filter_vfr (oracle/_ref/libhbref_vfr.so, where oracle/vfr.mk built it) mode=1 on host
               frames of the same clip, metric on the CPU, frames/s through the shaper alone (what a chain pays
               for it, before the download / upload hop it would also need)
Prints one JSON line per measurement plus the GPU's name and power limit.

  python tools/bench_vfr.py [--steps K]
"""
import argparse
import ctypes as C
import json
import math
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

REPO = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(REPO))

from handbrake_b200 import LIBHBCU, synth  # noqa: E402

HBM_PEAK = 3.35e12


class MMConfig(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("depth", C.c_int), ("fast", C.c_int), ("device", C.c_int),
                ("slots", C.c_int), ("results", C.c_int), ("gamma_lut", C.c_void_p)]


def gpu_info():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:     # noqa: BLE001
        pl = f"unknown ({e})"
    return name, pl


def gamma_lut(depth):
    maxv = (1 << depth) - 1
    den, e = np.float32(maxv - 1), float(np.float32(2.2))
    return np.array([int(4095 * math.pow(float(np.float32(i) / den), e)) for i in range(maxv + 1)], dtype=np.uint32)


def bench_metric(lib, w, h, depth, steps):
    import torch
    bps = 1 if depth == 8 else 2
    row, pitch = w * bps, (w * bps + 255) // 256 * 256
    nframes = 8
    frames, keep = [], []
    gen = torch.Generator(device="cuda").manual_seed(1)
    for _ in range(nframes):
        t = torch.randint(0, 256, ((h + 2) * pitch,), dtype=torch.uint8, device="cuda", generator=gen)
        if bps == 2:
            t.view(torch.int16).bitwise_and_(0x03FF)
        f = C.c_void_p()
        planes = (C.c_void_p * 3)(t.data_ptr(), t.data_ptr(), t.data_ptr())
        rb, rows, st = (C.c_int * 3)(row, row // 2, row // 2), (C.c_int * 3)(h, h // 2, h // 2), (C.c_int * 3)(pitch, pitch, pitch)
        assert lib.hbcu_frame_wrap(C.byref(f), 0, planes, rb, rows, st, C.c_size_t(2 * pitch), None, None, None) == 0, lib.hbcu_last_error()
        frames.append(f)
        keep.append(t)
    torch.cuda.synchronize()
    lut = gamma_lut(depth)
    cfg = MMConfig(w, h, depth, int(w >= 1920 or h >= 1080), 0, 4, 2, lut.ctypes.data)
    hdl = C.c_void_p()
    assert lib.hbcu_motion_metric_create(C.byref(hdl), C.byref(cfg)) == 0, lib.hbcu_last_error()

    def run(n, i0):
        for i in range(i0, i0 + n):
            assert lib.hbcu_motion_metric_enqueue(hdl, i % 4, (i - 1) % 4 if i > 0 else -1, i % 2, frames[i % nframes], None, 0) == 0
    run(50, 0)
    lib.hbcu_motion_metric_sync(hdl)
    assert lib.hbcu_motion_metric_mark(hdl, 0) == 0
    run(steps, 50)
    assert lib.hbcu_motion_metric_mark(hdl, 1) == 0
    ms = C.c_float()
    assert lib.hbcu_motion_metric_elapsed_ms(hdl, C.byref(ms)) == 0
    lib.hbcu_motion_metric_destroy(hdl)
    for f in frames:
        lib.hbcu_frame_release(f)
    per = ms.value / steps
    red = (w // 4) * (h // 4) * bps
    nbytes = w * h * bps + 2 * red
    return dict(kind="metric", width=w, height=h, depth=depth, frames=steps, device_us_per_frame=round(per * 1e3, 3),
                bytes_per_frame=nbytes, hbm_share=round(nbytes / HBM_PEAK / (per * 1e-3), 3))


def chain_fps(flt, clip, mode, chain):
    w, h = 1920, 1080
    sets = [None, f"mode={mode}:rate=24000/1001", "y-strength=6", None] if chain else [f"mode={mode}:rate=24000/1001"]
    names = (["hb_filter_hbcu_upload", "hb_filter_vfr_cuda", "hb_filter_nlmeans_cuda", "hb_filter_hbcu_download"]
             if chain else ["hb_filter_vfr"])
    t0 = time.perf_counter()
    r = flt.run(names, sets, clip, synth.PIX_FMT_YUV420P, w, h, vrate=(30000, 1001))
    dt = time.perf_counter() - t0
    assert r.init_failed == 0 and r.saw_eof
    return clip.shape[0] / dt, r.frames.shape[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--frames", type=int, default=60)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_vfr: no CUDA device; there is no CPU measurement path")
    name, pl = gpu_info()
    print(json.dumps(dict(gpu=name, power_limit=pl)), flush=True)
    lib = C.CDLL(str(LIBHBCU))
    lib.hbcu_last_error.restype = C.c_char_p
    for fn, at in (("hbcu_motion_metric_create", [C.c_void_p, C.c_void_p]),
                   ("hbcu_motion_metric_enqueue", [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int]),
                   ("hbcu_motion_metric_mark", [C.c_void_p, C.c_int]), ("hbcu_motion_metric_elapsed_ms", [C.c_void_p, C.c_void_p]),
                   ("hbcu_motion_metric_sync", [C.c_void_p]), ("hbcu_motion_metric_destroy", [C.c_void_p]),
                   ("hbcu_frame_release", [C.c_void_p])):
        getattr(lib, fn).argtypes = at
    for w, h in ((1920, 1080), (3840, 2160)):
        for depth in (8, 10):
            runs = [bench_metric(lib, w, h, depth, args.steps) for _ in range(3)]
            best = sorted(runs, key=lambda r: r["device_us_per_frame"])[1]
            best["runs_us"] = [r["device_us_per_frame"] for r in runs]
            print(json.dumps(best), flush=True)

    import handbrake_b200
    flt = handbrake_b200.filters()
    clip = synth.progressive_clip(synth.PIX_FMT_YUV420P, 1920, 1080, args.frames, seed=3)
    chain_fps(flt, clip[:8], 1, True)                                 # warm-up: modules, pools
    res = {0: [], 1: []}
    outs = {}
    for _ in range(3):
        for mode in (1, 0):
            fps, n = chain_fps(flt, clip, mode, True)
            res[mode].append(fps)
            outs[mode] = n
    for mode in (1, 0):
        print(json.dumps(dict(kind="chain", workload="1080p_420p_2997_upload_vfr_nlmeans_download", vfr_mode=mode,
                              frames_in=args.frames, frames_out=outs[mode], fps_median=round(statistics.median(res[mode]), 2),
                              fps_runs=[round(v, 2) for v in res[mode]])), flush=True)
    ref_so = REPO / "oracle" / "_ref" / "libhbref_vfr.so"
    if ref_so.exists():
        from handbrake_b200.hblib import FilterLib
        ref = FilterLib(ref_so)
        runs = [chain_fps(ref, clip, 1, False)[0] for _ in range(3)]
        print(json.dumps(dict(kind="cpu_vfr", workload="1080p_420p_2997_vfr_mode1_reference", fps_median=round(statistics.median(runs), 2),
                              fps_runs=[round(v, 2) for v in runs])), flush=True)
    else:
        print(json.dumps(dict(kind="cpu_vfr", note="oracle/_ref/libhbref_vfr.so not built: not measured")), flush=True)


if __name__ == "__main__":
    main()
