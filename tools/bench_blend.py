"""Subtitle overlay blend (hbcu_blend_*) on one GPU: device time per frame and device-chain frames/s.

Workloads (what libhb's subtitle renderer hands hb_blend_cuda):
  pgs  4K yuv420p10, two 1600x120 YUVA 4:4:4 overlays (subsample path), list unchanged in steady state
  ssa  4K yuv420p10, one 3840x400 YUVA 4:2:0 band (plain path), list unchanged in steady state
  vob  1080p yuv420p, one full-frame YUVA 4:4:4 overlay, a new list every frame (an upload per frame)
and, for a hardware-decoded job, the semi-planar formats NVDEC decodes into next to their planar pairs (same bytes):
  pgs  4K P010 against 4K yuv420p10 above
  ssa  1080p NV12 against 1080p yuv420p, one 1920x200 YUVA 4:2:0 band (plain path)

device ms/frame  CUDA events around K device-frame blends (hbcu_blend_mark / elapsed_ms): the device-to-device copy of
                 the frame plus the one blend launch; `2F share` is the time 2 x frame bytes take at 3.35 TB/s (H100 HBM3
                 peak) over that time
chain fps        wall-clock frames/s of the host loop an hb_blend_cuda.work() runs per device frame: output frame
                 allocation, overlay hand-over (staging + upload when changed), copy + blend, release
cpu ms/frame     the reference's hb_blend (oracle/_ref/libhbref_blend.so, where oracle/blend.mk built it) through the harness's render_sub stand-in,
                 minus the same run without overlays (best of three runs of 8 frames each)
Prints one JSON line per workload plus the GPU's name and power limit.

  python tools/bench_blend.py [--steps K] [--warmup W]
"""
import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

REPO = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "tests"))

from handbrake_b200 import LIBHBCU  # noqa: E402

HBM_PEAK = 3.35e12


class Config(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("depth", C.c_int), ("chroma_shift_w", C.c_int),
                ("chroma_shift_h", C.c_int), ("overlay_shift_w", C.c_int), ("overlay_shift_h", C.c_int),
                ("device", C.c_int), ("chroma_coeffs", C.c_uint32 * 8), ("interleaved_chroma", C.c_int)]


class Overlay(C.Structure):
    _fields_ = [("x", C.c_int), ("y", C.c_int), ("width", C.c_int), ("height", C.c_int),
                ("planes", C.c_void_p * 4), ("strides", C.c_int * 4)]


WORKLOADS = {
    # name: (frame w, h, depth, pix_fmt, overlay shifts, overlays (x, y, w, h), changed every frame, semi-planar)
    "4k_pgs_420p10": (3840, 2160, 10, 62, (0, 0), [(1120, 1880, 1600, 120), (1120, 2010, 1600, 120)], False, False),
    "4k_pgs_p010": (3840, 2160, 10, 158, (0, 0), [(1120, 1880, 1600, 120), (1120, 2010, 1600, 120)], False, True),
    "4k_ssa_band_420p10": (3840, 2160, 10, 62, (1, 1), [(0, 1700, 3840, 400)], False, False),
    "1080p_ssa_band_420p": (1920, 1080, 8, 0, (1, 1), [(0, 850, 1920, 200)], False, False),
    "1080p_ssa_band_nv12": (1920, 1080, 8, 23, (1, 1), [(0, 850, 1920, 200)], False, True),
    "1080p_vobsub_fullframe_420p": (1920, 1080, 8, 0, (0, 0), [(0, 0, 1920, 1080)], True, False),
}


def gpu_info():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:     # noqa: BLE001
        pl = f"unknown ({e})"
    return name, pl


def make_overlays(shifts, rects, seed):
    rng = np.random.default_rng(seed)
    keep, arr = [], (Overlay * len(rects))()
    for i, (x, y, w, h) in enumerate(rects):
        cdim = (-((-w) >> shifts[0]), -((-h) >> shifts[1]))
        dims = [(w, h), cdim, cdim, (w, h)]
        o = arr[i]
        o.x, o.y, o.width, o.height = x, y, w, h
        for p, (pw, ph) in enumerate(dims):
            a = rng.integers(0, 256, (ph, pw), dtype=np.uint8)
            keep.append(a)
            o.planes[p] = a.ctypes.data
            o.strides[p] = pw
    return arr, keep


def bench_gpu(lib, name, steps, warmup):
    w, h, depth, pix, osh, rects, changed, semi = WORKLOADS[name]
    sw, sh = 1, 1
    cfg = Config(w, h, depth, sw, sh, osh[0], osh[1], 0)
    cfg.interleaved_chroma = int(semi)
    for i, v in enumerate([18, 18, 6, 2, 18, 18, 6, 2]):      # center chroma location, 4:2:0
        cfg.chroma_coeffs[i] = v
    hnd = C.c_void_p()
    if lib.hbcu_blend_create(C.byref(hnd), C.byref(cfg)) != 0:
        raise RuntimeError(lib.hbcu_last_error().decode())
    bps = 2 if depth > 8 else 1
    cw, ch = (w + 1) // 2, (h + 1) // 2
    # a semi-planar frame: one plane of Cb/Cr pairs, the third plane absent (0 rows of 0 bytes)
    row_bytes = (C.c_int * 3)(w * bps, 2 * cw * bps, 0) if semi else (C.c_int * 3)(w * bps, cw * bps, cw * bps)
    rows = (C.c_int * 3)(h, ch, 0) if semi else (C.c_int * 3)(h, ch, ch)
    strides = (C.c_int * 3)(*[(rb + 63) // 64 * 64 for rb in row_bytes])
    frame_bytes = sum(strides[p] * rows[p] for p in range(3))
    fin = C.c_void_p()
    assert lib.hbcu_frame_alloc(C.byref(fin), 0, row_bytes, rows, strides) == 0
    lists = [make_overlays(osh, rects, s) for s in range(2)]

    def step(i):
        fout = C.c_void_p()
        assert lib.hbcu_frame_alloc(C.byref(fout), 0, row_bytes, rows, strides) == 0
        arr, _ = lists[i % 2] if changed else lists[0]
        assert lib.hbcu_blend_set_overlays(hnd, arr, len(rects), 1 if changed or i == 0 else 0) == 0
        assert lib.hbcu_blend_frames(hnd, fin, None, None, fout, None, None) == 0, lib.hbcu_last_error()
        lib.hbcu_frame_release(fout)

    for i in range(warmup):
        step(i)
    lib.hbcu_blend_sync(hnd)
    lib.hbcu_blend_mark(hnd, 0)
    t0 = time.perf_counter()
    for i in range(steps):
        step(warmup + i)
    lib.hbcu_blend_mark(hnd, 1)
    ms = C.c_float()
    lib.hbcu_blend_elapsed_ms(hnd, C.byref(ms))
    wall = time.perf_counter() - t0
    lib.hbcu_frame_release(fin)
    lib.hbcu_blend_destroy(hnd)
    dev_ms = ms.value / steps
    return dict(device_ms_per_frame=round(dev_ms, 4), chain_fps=round(steps / wall, 1),
                frame_bytes=frame_bytes, two_f_bound_ms=round(2 * frame_bytes / HBM_PEAK * 1e3, 4),
                two_f_share=round(2 * frame_bytes / HBM_PEAK * 1e3 / dev_ms, 3), uploads_changed_every_frame=changed)


def bench_cpu(name, frames_n=8):
    ref_so = REPO / "oracle" / "_ref" / "libhbref_blend.so"
    if not ref_so.exists():
        return None
    from handbrake_b200.hblib import FilterLib, RENDER_SUB
    w, h, depth, pix, osh, rects, changed, _ = WORKLOADS[name]
    lib = FilterLib(ref_so)
    bps = 2 if depth > 8 else 1
    fb = (w * h + 2 * ((w + 1) // 2) * ((h + 1) // 2)) * bps
    frames = np.zeros((frames_n, fb), np.uint8)
    rng = np.random.default_rng(1)
    ovs = []
    opix = {(0, 0): 79, (1, 1): 33}[osh]
    for f in range(frames_n):
        for (x, y, ow, oh) in rects:
            cwo, cho = -((-ow) >> osh[0]), -((-oh) >> osh[1])
            ovs.append((f, x, y, ow, oh, rng.integers(0, 256, 2 * ow * oh + 2 * cwo * cho, dtype=np.uint8)))
    times = []
    for ov in ([], ovs):
        best = float("inf")
        for _ in range(3):
            t0 = time.perf_counter()
            lib.run_blend("hb_blend", ov, opix, [RENDER_SUB], [None], frames, pix, w, h)
            best = min(best, time.perf_counter() - t0)
        times.append(best)
    return round((times[1] - times[0]) / frames_n * 1e3, 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    a = ap.parse_args()
    lib = C.CDLL(str(LIBHBCU))
    lib.hbcu_last_error.restype = C.c_char_p
    name, pl = gpu_info()
    print(json.dumps(dict(gpu=name, power_limit=pl)))
    for wl in WORKLOADS:
        r = bench_gpu(lib, wl, a.steps, a.warmup)
        r["cpu_hb_blend_ms_per_frame"] = bench_cpu(wl)
        print(json.dumps(dict(workload=wl, **r)), flush=True)


if __name__ == "__main__":
    main()
