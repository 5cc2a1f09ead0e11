"""Rotations and mirrors (hbcu_rotate_*) on one GPU, and what a rotation costs a hardware-decoded 10-bit chain.

Per case (device frames at hb_image_stride pitches, one handle; enough frames in rotation that the working set is four
times the L2, so every launch reads and writes HBM):
  kernel_us        the rotate kernel's own mean duration over --launches launches, from torch.profiler
  device_us        CUDA events around --launches launches after --warmup (hbcu_rotate_mark / elapsed_ms): includes any
                   gap the host leaves between launches
  memcpy_kernel_us a device-to-device copy of the same bytes over the same rotation, timed the same two ways in the same
  memcpy_us        run: the copy's rate on this card is the honest ceiling
  vs_memcpy        kernel_us / memcpy_kernel_us
  hbm_tb_s         (input + output bytes) / kernel_us
Cases: 1080p and 4K x yuv420p, yuv420p10le, nv12, p010le x angle=0:hflip=1, 180:0, 90:0, 90:1.

Chain rate, 4K P010 surfaces (what NVDEC hands a 10-bit job), frames/s of the host loop:
  rotate     surface -> rotate angle=270 -> format(yuv420p10le) -> NLMeans medium -> format(p010le) -> encoder-side
             hbcu_frame_acquire / done
  plain      the same chain without the rotation
The two arms alternate, three runs each.  Prints one JSON line with the GPU's name and power limit.

  python tools/bench_rotate.py [--launches N] [--warmup W] [--frames F]
"""
import argparse
import ctypes as C
import json
import sys
import time
from pathlib import Path

REPO = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "tools"))

import handbrake_b200  # noqa: E402
from handbrake_b200 import LIBHBCU  # noqa: E402
from bench_format import L2_BYTES, FormatConfig, NlmConfig, alloc, check, gpu_info, profiled_us  # noqa: E402


class RotateConfig(C.Structure):
    _fields_ = [("planes", C.c_int), ("width", C.c_int * 3), ("height", C.c_int * 3), ("elem_bytes", C.c_int * 3),
                ("transform", C.c_int), ("device", C.c_int), ("slots", C.c_int)]


# name: (luma element bytes, chroma element bytes, semi-planar)
FORMATS = {"yuv420p": (1, 1, False), "yuv420p10le": (2, 2, False), "nv12": (1, 2, True), "p010le": (2, 4, True)}
# settings: (HBCU_ROTATE_*, transposes)
TRANSFORMS = {"0:1": (1, False), "180:0": (3, False), "90:0": (4, True), "90:1": (5, True), "270:0": (6, True)}
SIZES = {"1080p": (1920, 1080), "4k": (3840, 2160)}


def planes(fmt, w, h):
    """(elements per row, rows, element bytes) of each plane"""
    el, ec, semi = FORMATS[fmt]
    cw, ch = (w + 1) // 2, (h + 1) // 2
    return [(w, h, el), (cw, ch, ec)] + ([] if semi else [(cw, ch, ec)])


def shapes(fmt, w, h):
    """(row bytes, rows, pitch) of the three planes; a semi-planar frame's third plane is (0, 0, 0)"""
    s = [(pw * e, ph, (pw * e + 63) // 64 * 64) for pw, ph, e in planes(fmt, w, h)]
    return s + [(0, 0, 0)] * (3 - len(s))


def create(lib, fmt, w, h, settings, slots=4):
    p = planes(fmt, w, h) + [(0, 0, 0)] * (3 - len(planes(fmt, w, h)))
    cfg = RotateConfig(len(planes(fmt, w, h)), (C.c_int * 3)(*[q[0] for q in p]), (C.c_int * 3)(*[q[1] for q in p]),
                       (C.c_int * 3)(*[q[2] for q in p]), TRANSFORMS[settings][0], 0, slots)
    hd = C.c_void_p()
    check(lib.hbcu_rotate_create(C.byref(hd), C.byref(cfg)), lib)
    return hd


def bench_case(lib, size, fmt, settings, launches, warmup):
    import torch
    w, h = SIZES[size]
    ow, oh = (h, w) if TRANSFORMS[settings][1] else (w, h)
    hd = create(lib, fmt, w, h, settings)
    s_in, s_out = shapes(fmt, w, h), shapes(fmt, ow, oh)
    frame = sum(rb * rows for rb, rows, _ in s_in)
    moved = 2 * frame
    ring = max(2, -(-4 * L2_BYTES // moved))
    fin = [alloc(lib, s_in) for _ in range(ring)]
    fout = [alloc(lib, s_out) for _ in range(ring)]
    ticket = [0]

    def rotate(n):
        for _ in range(n):
            i = ticket[0] % ring
            check(lib.hbcu_rotate_frame(hd, C.c_int64(ticket[0]), fin[i], None, None, fout[i], None, None), lib)
            ticket[0] += 1

    rotate(warmup)
    check(lib.hbcu_rotate_sync(hd), lib)
    check(lib.hbcu_rotate_mark(hd, 0), lib)
    rotate(launches)
    check(lib.hbcu_rotate_mark(hd, 1), lib)
    ms = C.c_float()
    check(lib.hbcu_rotate_elapsed_ms(hd, C.byref(ms)), lib)
    kernel_us = profiled_us(lambda: rotate(launches), "_kernel", launches)
    check(lib.hbcu_rotate_sync(hd), lib)
    for f in fin + fout:
        lib.hbcu_frame_release(f)
    lib.hbcu_rotate_destroy(hd)
    src = [torch.empty(frame, dtype=torch.uint8, device="cuda") for _ in range(ring)]
    dst = [torch.empty_like(t) for t in src]

    def copy(n):
        for i in range(n):
            dst[i % ring].copy_(src[i % ring])

    copy(warmup)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    copy(launches)
    e1.record()
    e1.synchronize()
    copy_kernel_us = profiled_us(lambda: copy(launches), "Memcpy DtoD", launches)
    both = kernel_us is not None and copy_kernel_us is not None
    return dict(case=f"{size}_{fmt}_{settings}", kernel_us=kernel_us and round(kernel_us, 2),
                device_us=round(ms.value * 1e3 / launches, 2), memcpy_kernel_us=copy_kernel_us and round(copy_kernel_us, 2),
                memcpy_us=round(e0.elapsed_time(e1) * 1e3 / launches, 2),
                vs_memcpy=round(kernel_us / copy_kernel_us, 3) if both else None,
                hbm_tb_s=round(moved / kernel_us / 1e6, 2) if kernel_us else None, bytes_moved=moved,
                frames_in_rotation=ring, launches=launches)


def chain_rate(lib, flt, arm, frames, torch):
    """4K P010 surfaces -> (rotate 270) -> format -> NLMeans medium -> format -> encoder acquire / done"""
    w, h = 3840, 2160
    rot = arm == "rotate"
    ow, oh = (h, w) if rot else (w, h)
    s_src, s_semi, s_planar = shapes("p010le", w, h), shapes("p010le", ow, oh), shapes("yuv420p10le", ow, oh)
    cfg = NlmConfig()
    flt.hb_parse_filter_settings.restype = C.c_void_p
    flt.hb_parse_filter_settings.argtypes = [C.c_char_p]
    flt.hb_nlmeans_cuda_build_config.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(NlmConfig), C.c_void_p, C.c_void_p, C.c_void_p]
    check(flt.hb_nlmeans_cuda_build_config(flt.hb_parse_filter_settings(b"y-strength=6"), 62, ow, oh, C.byref(cfg), None, None, None), lib)
    cfg.device, cfg.ring_frames, cfg.out_slots = 0, 8, 4
    nl, f_in, f_out = C.c_void_p(), C.c_void_p(), C.c_void_p()
    check(lib.hbcu_nlmeans_create(C.byref(nl), C.byref(cfg)), lib)
    check(lib.hbcu_format_create(C.byref(f_in), C.byref(FormatConfig(ow, oh, 10, 0, 0, 6))), lib)
    check(lib.hbcu_format_create(C.byref(f_out), C.byref(FormatConfig(ow, oh, 10, 1, 0, 6))), lib)
    rt = create(lib, "p010le", w, h, "270:0", 6) if rot else None
    surfaces = [alloc(lib, s_src) for _ in range(4)]      # what the decoder hands over, decoded once
    enc = torch.cuda.Stream()
    lag = 1                               # NLMeans medium looks one frame ahead

    def emit(k):
        den = alloc(lib, s_planar)
        check(lib.hbcu_nlmeans_filter_frame(nl, C.c_int64(k), lag + 1, den), lib)
        out = alloc(lib, s_semi)
        check(lib.hbcu_format_convert(f_out, C.c_int64(k), den, None, None, out, None, None), lib)
        lib.hbcu_frame_release(den)
        check(lib.hbcu_frame_acquire(out, C.c_void_p(enc.cuda_stream)), lib)
        check(lib.hbcu_frame_done(out, C.c_void_p(enc.cuda_stream)), lib)
        lib.hbcu_frame_release(out)

    t0 = time.perf_counter()
    for t in range(frames):
        src = surfaces[t % len(surfaces)]
        if rot:
            r = alloc(lib, s_semi)
            check(lib.hbcu_rotate_frame(rt, C.c_int64(t), src, None, None, r, None, None), lib)
            src = r
        planar = alloc(lib, s_planar)
        check(lib.hbcu_format_convert(f_in, C.c_int64(t), src, None, None, planar, None, None), lib)
        if rot:
            lib.hbcu_frame_release(src)
        check(lib.hbcu_nlmeans_upload_frame(nl, C.c_int64(t), planar), lib)
        lib.hbcu_frame_release(planar)
        if t >= lag:
            emit(t - lag)
    enc.synchronize()
    check(lib.hbcu_nlmeans_sync(nl), lib)
    wall = time.perf_counter() - t0
    check(lib.hbcu_format_sync(f_out), lib)
    for s in surfaces:
        lib.hbcu_frame_release(s)
    if rt is not None:
        lib.hbcu_rotate_destroy(rt)
    lib.hbcu_format_destroy(f_in)
    lib.hbcu_format_destroy(f_out)
    lib.hbcu_nlmeans_destroy(nl)
    return (frames - lag) / wall


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--frames", type=int, default=120)
    a = ap.parse_args()
    import torch
    lib = C.CDLL(str(LIBHBCU))
    lib.hbcu_last_error.restype = C.c_char_p
    lib.hbcu_frame_release.argtypes = [C.c_void_p]
    if lib.hbcu_device_count() < 1:
        raise SystemExit("no CUDA device: nothing measured")
    flt = handbrake_b200.filters().lib
    name, pl = gpu_info()
    cases = [bench_case(lib, size, fmt, s, a.launches, a.warmup)
             for size in SIZES for fmt in FORMATS for s in ("0:1", "180:0", "90:0", "90:1")]
    chain_rate(lib, flt, "rotate", 8, torch)          # warm-up: modules, pools, NLMeans plans
    chain_rate(lib, flt, "plain", 8, torch)
    runs = {"rotate": [], "plain": []}
    for _ in range(3):
        for arm in ("rotate", "plain"):
            runs[arm].append(round(chain_rate(lib, flt, arm, a.frames, torch), 1))
    lib.hbcu_frame_trim()
    print(json.dumps(dict(gpu=name, power_limit=pl, cases=cases,
                          chain_4k_p010_nlmeans_medium_fps=dict(rotate_270=runs["rotate"], no_rotate=runs["plain"],
                                                                frames_per_run=a.frames - 1))), flush=True)


if __name__ == "__main__":
    main()
