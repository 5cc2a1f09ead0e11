"""Semi-planar <-> planar 4:2:0 repacks (hbcu_format_*) on one GPU, and what they save a hardware-decoded 10-bit chain.

Conversion time, per workload (device frames at hb_image_stride pitches, one handle; enough frames in rotation that
the working set is four times the L2, so every conversion reads and writes HBM):
  device_us        CUDA events around --launches conversions after --warmup (hbcu_format_mark / elapsed_ms): includes any
                   gap the host leaves between launches
  kernel_us        the conversion kernel's own mean duration over another --launches conversions, from torch.profiler
  bytes_moved      input frame + output frame (row bytes x rows of every plane, from the shapes)
  memcpy_us        a device-to-device cudaMemcpyAsync of one frame's bytes (it reads and writes the bytes a conversion
  memcpy_kernel_us moves) over the same rotation, timed the same two ways in the same run: the copy's rate on this card
                   is the honest ceiling
  vs_memcpy        kernel_us / memcpy_kernel_us
  hbm_tb_s         bytes_moved / kernel_us
Workloads: 1080p nv12 -> yuv420p, 4K nv12 -> yuv420p, 4K p010le -> yuv420p10le, 4K yuv420p10le -> p010le.

Chain rate, 4K P010 (what NVDEC hands a 10-bit job, what 10-bit NVENC takes), frames/s of the host loop:
  device     surface -> format(yuv420p10le) -> NLMeans medium -> format(p010le) -> encoder-side hbcu_frame_acquire / done
  download   surface -> format(yuv420p10le) -> NLMeans medium -> download to page-locked memory -> upload -> acquire / done
             (the round trip a job pays today without a device format filter, not counting the CPU repack itself)
The two arms alternate, three runs each.  Prints one JSON line with the GPU's name and power limit.

  python tools/bench_format.py [--launches N] [--warmup W] [--frames F]
"""
import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

REPO = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(REPO))

import handbrake_b200  # noqa: E402
from handbrake_b200 import LIBHBCU  # noqa: E402


L2_BYTES = 50 * 1024 * 1024            # H100 SXM


class FormatConfig(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("depth", C.c_int), ("to_semi_planar", C.c_int),
                ("device", C.c_int), ("slots", C.c_int)]


class NlmPlane(C.Structure):
    _fields_ = [("patch_size", C.c_int), ("range", C.c_int), ("nframes", C.c_int), ("bypass", C.c_int),
                ("origin_tune", C.c_double), ("weight_fact", C.c_float), ("diff_max", C.c_int),
                ("exptable", C.c_float * 128), ("prefilter", C.c_int)]


class NlmConfig(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("depth", C.c_int), ("chroma_shift_w", C.c_int),
                ("chroma_shift_h", C.c_int), ("device", C.c_int), ("ring_frames", C.c_int), ("out_slots", C.c_int),
                ("plane", NlmPlane * 3)]


WORKLOADS = {
    # name: (w, h, depth, source semi-planar)
    "1080p_nv12_to_yuv420p": (1920, 1080, 8, True),
    "4k_nv12_to_yuv420p": (3840, 2160, 8, True),
    "4k_p010_to_yuv420p10": (3840, 2160, 10, True),
    "4k_yuv420p10_to_p010": (3840, 2160, 10, False),
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


def shapes(w, h, depth, semi):
    """(row bytes, rows, pitch) of the three planes; a semi-planar frame's third plane is (0, 0, 0)"""
    bps = 2 if depth > 8 else 1
    cw, ch = (w + 1) // 2, (h + 1) // 2
    planes = [(w * bps, h), (2 * cw * bps, ch), (0, 0)] if semi else [(w * bps, h), (cw * bps, ch), (cw * bps, ch)]
    return [(rb, rows, (rb + 63) // 64 * 64) for rb, rows in planes]


def alloc(lib, shp):
    f = C.c_void_p()
    rb = (C.c_int * 3)(*[s[0] for s in shp]); rows = (C.c_int * 3)(*[s[1] for s in shp]); st = (C.c_int * 3)(*[s[2] for s in shp])
    if lib.hbcu_frame_alloc(C.byref(f), 0, rb, rows, st) != 0:
        raise RuntimeError(lib.hbcu_last_error().decode())
    return f


def check(rc, lib):
    if rc != 0:
        raise RuntimeError(lib.hbcu_last_error().decode())


def profiled_us(run, match, launches):
    """mean device time of the CUDA activities whose name contains `match`, from torch.profiler (CUPTI), over a window
    of its own: the kernel's (or the copy's) own duration, without the host's launch gaps"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    total, count = 0.0, 0
    for k in prof.key_averages():
        if match in k.key:
            total += getattr(k, "device_time_total", None) or getattr(k, "cuda_time_total", 0.0)
            count += k.count
    return total / count if count >= launches else None     # None: not measured (the profiler missed activities)


def bench_conversion(lib, name, launches, warmup):
    import torch
    w, h, depth, semi_src = WORKLOADS[name]
    cfg = FormatConfig(w, h, depth, int(not semi_src), 0, 4)
    hd = C.c_void_p()
    check(lib.hbcu_format_create(C.byref(hd), C.byref(cfg)), lib)
    s_in, s_out = shapes(w, h, depth, semi_src), shapes(w, h, depth, not semi_src)
    frame = sum(rb * rows for rb, rows, _ in s_in)
    moved = frame + sum(rb * rows for rb, rows, _ in s_out)
    # enough frames in rotation that the working set is four times the 50 MB L2: every launch reads and writes HBM
    ring = max(2, -(-4 * L2_BYTES // moved))
    fin = [alloc(lib, s_in) for _ in range(ring)]
    fout = [alloc(lib, s_out) for _ in range(ring)]
    ticket = [0]

    def convert(n):
        for _ in range(n):
            i = ticket[0] % ring
            check(lib.hbcu_format_convert(hd, C.c_int64(ticket[0]), fin[i], None, None, fout[i], None, None), lib)
            ticket[0] += 1

    convert(warmup)
    check(lib.hbcu_format_sync(hd), lib)
    check(lib.hbcu_format_mark(hd, 0), lib)
    convert(launches)
    check(lib.hbcu_format_mark(hd, 1), lib)
    ms = C.c_float()
    check(lib.hbcu_format_elapsed_ms(hd, C.byref(ms)), lib)
    kernel_us = profiled_us(lambda: convert(launches), "format_kernel", launches)
    check(lib.hbcu_format_sync(hd), lib)
    for f in fin + fout:
        lib.hbcu_frame_release(f)
    lib.hbcu_format_destroy(hd)
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
    dev_us = ms.value * 1e3 / launches
    cp_us = e0.elapsed_time(e1) * 1e3 / launches
    both = kernel_us is not None and copy_kernel_us is not None
    return dict(workload=name, device_us=round(dev_us, 2), kernel_us=kernel_us and round(kernel_us, 2), bytes_moved=moved,
                memcpy_us=round(cp_us, 2), memcpy_kernel_us=copy_kernel_us and round(copy_kernel_us, 2),
                vs_memcpy=round(kernel_us / copy_kernel_us, 3) if both else None,
                hbm_tb_s=round(moved / kernel_us / 1e6, 2) if kernel_us else None, frames_in_rotation=ring, launches=launches)


def chain_rate(lib, flt, arm, frames, torch):
    """4K P010 surfaces through format -> NLMeans medium -> (format | download + upload) -> encoder acquire / done"""
    w, h = 3840, 2160
    s_semi, s_planar = shapes(w, h, 10, True), shapes(w, h, 10, False)
    cfg = NlmConfig()
    flt.hb_parse_filter_settings.restype = C.c_void_p
    flt.hb_parse_filter_settings.argtypes = [C.c_char_p]
    flt.hb_nlmeans_cuda_build_config.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(NlmConfig), C.c_void_p, C.c_void_p, C.c_void_p]
    check(flt.hb_nlmeans_cuda_build_config(flt.hb_parse_filter_settings(b"y-strength=6"), 62, w, h, C.byref(cfg), None, None, None), lib)
    cfg.device, cfg.ring_frames, cfg.out_slots = 0, 8, 4
    nl, f_in, f_out, x = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p()
    check(lib.hbcu_nlmeans_create(C.byref(nl), C.byref(cfg)), lib)
    check(lib.hbcu_format_create(C.byref(f_in), C.byref(FormatConfig(w, h, 10, 0, 0, 6))), lib)
    check(lib.hbcu_format_create(C.byref(f_out), C.byref(FormatConfig(w, h, 10, 1, 0, 6))), lib)
    check(lib.hbcu_xfer_create(C.byref(x), 0, 16), lib)
    surfaces = [alloc(lib, s_semi) for _ in range(4)]      # what the decoder hands over, decoded once
    host_ring = 4
    hbytes = sum(p * rows for _, rows, p in s_planar)
    lib.hbcu_host_alloc.restype = C.c_void_p
    host = [lib.hbcu_host_alloc(C.c_size_t(hbytes)) for _ in range(host_ring)]
    hst = (C.c_int * 3)(*[p for _, _, p in s_planar])
    enc = torch.cuda.Stream()
    lag = 1                               # NLMeans medium looks one frame ahead

    def host_planes(i):
        base, off, ptrs = host[i % host_ring], 0, []
        for _, rows, p in s_planar:
            ptrs.append(base + off); off += rows * p
        return (C.c_void_p * 3)(*ptrs)

    def emit(k):
        den = alloc(lib, s_planar)
        check(lib.hbcu_nlmeans_filter_frame(nl, C.c_int64(k), lag + 1, den), lib)
        if arm == "device":
            out = alloc(lib, s_semi)
            check(lib.hbcu_format_convert(f_out, C.c_int64(k), den, None, None, out, None, None), lib)
        else:
            if k >= host_ring:
                check(lib.hbcu_xfer_wait(x, C.c_int64(2 * (k - host_ring) + 1)), lib)
            hp = host_planes(k)
            check(lib.hbcu_xfer_download(x, C.c_int64(2 * k), den, hp, hst), lib)
            out = alloc(lib, s_planar)
            check(lib.hbcu_xfer_upload(x, C.c_int64(2 * k + 1), out, hp, hst), lib)
        lib.hbcu_frame_release(den)
        check(lib.hbcu_frame_acquire(out, C.c_void_p(enc.cuda_stream)), lib)
        check(lib.hbcu_frame_done(out, C.c_void_p(enc.cuda_stream)), lib)
        lib.hbcu_frame_release(out)

    t0 = time.perf_counter()
    for t in range(frames):
        planar = alloc(lib, s_planar)
        check(lib.hbcu_format_convert(f_in, C.c_int64(t), surfaces[t % len(surfaces)], None, None, planar, None, None), lib)
        check(lib.hbcu_nlmeans_upload_frame(nl, C.c_int64(t), planar), lib)
        lib.hbcu_frame_release(planar)
        if t >= lag:
            emit(t - lag)
    enc.synchronize()
    check(lib.hbcu_nlmeans_sync(nl), lib)
    wall = time.perf_counter() - t0
    check(lib.hbcu_format_sync(f_out), lib)
    lib.hbcu_xfer_destroy(x)
    for s in surfaces:
        lib.hbcu_frame_release(s)
    for p in host:
        lib.hbcu_host_free(C.c_void_p(p))
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
    conv = [bench_conversion(lib, wl, a.launches, a.warmup) for wl in WORKLOADS]
    chain_rate(lib, flt, "device", 8, torch)          # warm-up: modules, pools, NLMeans plans
    chain_rate(lib, flt, "download", 8, torch)
    runs = {"device": [], "download": []}
    for _ in range(3):
        for arm in ("device", "download"):
            runs[arm].append(round(chain_rate(lib, flt, arm, a.frames, torch), 1))
    lib.hbcu_frame_trim()
    print(json.dumps(dict(gpu=name, power_limit=pl, conversions=conv,
                          chain_4k_p010_nlmeans_medium_fps=dict(device_format=runs["device"], download_reupload=runs["download"],
                                                                frames_per_run=a.frames - 1))), flush=True)


if __name__ == "__main__":
    main()
