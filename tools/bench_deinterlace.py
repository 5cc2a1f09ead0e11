"""Yadif and Bwdif deinterlacing (hbcu_deint_*) on one GPU.

Per case (device frames at hb_image_stride pitches, one handle; enough frames in rotation that the working set is four
times the L2, so every launch reads and writes HBM):
  kernel_us        the deinterlace kernel's own mean duration over --launches launches, from torch.profiler
  device_us        CUDA events around --launches launches after --warmup (hbcu_deint_mark / elapsed_ms): includes any
                   gap the host leaves between launches
  memcpy_kernel_us a device-to-device copy of the same bytes over the same rotation, timed the same two ways in the same
  memcpy_us        run
  bytes_moved      the algorithm's traffic from the shapes: 3.5 frames per picture in frame mode (all of cur, one whole
                   neighbour frame and half of the other read, one frame written), 5 frames in field mode (3 read, 2
                   written)
  hbm_tb_s         bytes_moved / kernel_us
Cases: 1080p 8-bit, 4K 8-bit and 4K 10-bit (4:2:0) x Yadif, Bwdif x frame and field mode.

Chain rate, 4K 10-bit interlaced P010 frames (what NVDEC hands a 10-bit job; one frame in five static, so comb-detect
marks some frames uncombed), input frames/s of libhb's filter loop (hb_bench_run_chain, lib/libhbshim.so):
  bwdif      upload adapter in its decoder role (HBCU_UPLOAD_EXTERNAL=1: every frame goes on as a WRAPPED device surface)
             -> format(yuv420p10le) -> comb-detect -> bwdif mode=35 -> NLMeans medium -> format(p010le) -> the end of
             the chain, where a device output is released behind its producer as an encoder's acquire / done would be
  decomb     the same chain with decomb mode=39 (its default with the selective bit comb detection adds) in bwdif's place
The host-to-device copy of each input frame is part of both arms.  The two arms alternate, three runs each.  Prints one
JSON line with the GPU's name and power limit.

  python tools/bench_deinterlace.py [--launches N] [--warmup W] [--frames F]
"""
import argparse
import ctypes as C
import json
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "tools"))

import handbrake_b200  # noqa: E402
from handbrake_b200 import LIBHBCU, synth  # noqa: E402
from bench_format import L2_BYTES, alloc, check, gpu_info, profiled_us  # noqa: E402


class DeintConfig(C.Structure):
    _fields_ = [("algorithm", C.c_int), ("width", C.c_int * 3), ("height", C.c_int * 3), ("sample_bytes", C.c_int),
                ("depth", C.c_int), ("device", C.c_int)]


SIZES = {"1080p": (1920, 1080), "4k": (3840, 2160)}
CASES = [("1080p", 8), ("4k", 8), ("4k", 10)]
ALGOS = {"yadif": 1, "bwdif": 2}


def bench_case(lib, size, depth, algo, field, launches, warmup):
    import torch
    w, h = SIZES[size]
    e = 1 if depth == 8 else 2
    dims = [(w, h), ((w + 1) // 2, (h + 1) // 2), ((w + 1) // 2, (h + 1) // 2)]
    shp = [(pw * e, ph, (pw * e + 63) // 64 * 64) for pw, ph in dims]
    cfg = DeintConfig(ALGOS[algo], (C.c_int * 3)(*[d[0] for d in dims]), (C.c_int * 3)(*[d[1] for d in dims]), e, depth, 0)
    hd = C.c_void_p()
    check(lib.hbcu_deint_create(C.byref(hd), C.byref(cfg)), lib)
    frame = sum(rb * rows for rb, rows, _ in shp)
    npics = 2 if field else 1
    moved = int(frame * (5 if field else 3.5))
    ring = max(4, -(-4 * L2_BYTES // ((3 + npics) * frame)))
    fin = [alloc(lib, shp) for _ in range(ring)]
    fout = [alloc(lib, shp) for _ in range(ring * npics)]
    par = (C.c_int * 2)(0, 1)
    intra = (C.c_int * 2)(0, 0)
    t = [0]

    def run(n):
        for _ in range(n):
            i = t[0] % ring
            outs = (C.c_void_p * 2)(fout[npics * i], fout[npics * i + npics - 1])
            check(lib.hbcu_deint_frame(hd, fin[(i + ring - 1) % ring], fin[i], fin[(i + 1) % ring], 1, 1, npics, outs,
                                       par, intra), lib)
            t[0] += 1

    run(warmup)
    check(lib.hbcu_deint_sync(hd), lib)
    check(lib.hbcu_deint_mark(hd, 0), lib)
    run(launches)
    check(lib.hbcu_deint_mark(hd, 1), lib)
    ms = C.c_float()
    check(lib.hbcu_deint_elapsed_ms(hd, C.byref(ms)), lib)
    kernel_us = profiled_us(lambda: run(launches), "deint_kernel", launches)
    check(lib.hbcu_deint_sync(hd), lib)
    for f in fin + fout:
        lib.hbcu_frame_release(f)
    lib.hbcu_deint_destroy(hd)
    src = [torch.empty(moved // 2, dtype=torch.uint8, device="cuda") for _ in range(ring)]
    dst = [torch.empty_like(x) for x in src]

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
    return dict(case=f"{size}_{depth}bit_{algo}_{'field' if field else 'frame'}", kernel_us=kernel_us and round(kernel_us, 2),
                device_us=round(ms.value * 1e3 / launches, 2), memcpy_kernel_us=copy_kernel_us and round(copy_kernel_us, 2),
                memcpy_us=round(e0.elapsed_time(e1) * 1e3 / launches, 2),
                hbm_tb_s=round(moved / kernel_us / 1e6, 2) if kernel_us else None,
                memcpy_hbm_tb_s=round(moved / copy_kernel_us / 1e6, 2) if copy_kernel_us else None,
                bytes_moved=moved, frames_in_rotation=ring, launches=launches)


class BenchStats(C.Structure):
    _fields_ = [("seconds", C.c_double), ("frames_out", C.c_int64), ("bytes_in", C.c_int64), ("bytes_out", C.c_int64),
                ("checksum", C.c_uint64), ("ring_misses", C.c_int64)]


NLM_MEDIUM = "y-strength=6"                     # bench.py's NLMeans medium
CHAINS = {
    "bwdif": ("hb_filter_bwdif_cuda", "mode=35"),
    "decomb": ("hb_filter_decomb_cuda", "mode=39"),
}


def p010_clip(w, h, n):
    """interlaced 4:2:0 10-bit frames as P010 (Cb/Cr interleaved, samples << 6)"""
    import numpy as np
    clip = synth.interlaced_clip(synth.PIX_FMT_YUV420P10, w, h, n)
    cw, ch = (w + 1) // 2, (h + 1) // 2
    out = []
    for f in clip:
        v = f.view(np.uint16)
        y, u, cr = v[: w * h], v[w * h: w * h + cw * ch], v[w * h + cw * ch:]
        uv = np.empty(2 * cw * ch, np.uint16)
        uv[0::2], uv[1::2] = u, cr
        out.append(np.concatenate([y, uv]) << 6)
    return np.ascontiguousarray(np.stack(out)).view(np.uint8)


def chain_rate(flt, arm, clip, frames):
    w, h = 3840, 2160
    deint, deint_set = CHAINS[arm]
    names = ["hb_filter_hbcu_upload", "hb_filter_format_cuda", "hb_filter_comb_detect_cuda", deint, "hb_filter_nlmeans_cuda",
             "hb_filter_format_cuda"]
    sets = [None, "format=yuv420p10le", None, deint_set, NLM_MEDIUM, "format=p010le"]
    protos = (C.c_void_p * len(names))(*[C.addressof(C.c_char.in_dll(flt, n)) for n in names])
    cs = (C.c_char_p * len(names))(*[x.encode() if x else None for x in sets])
    st = BenchStats()
    rc = flt.hb_bench_run_chain(len(names), protos, cs, 158, w, h, synth.PIC_FLAG_TOP_FIELD_FIRST,
                                clip.ctypes.data, clip.shape[0], frames, C.byref(st))
    if rc != 0:
        raise RuntimeError(f"chain {arm} failed")
    return frames / st.seconds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--frames", type=int, default=120)
    a = ap.parse_args()
    lib = C.CDLL(str(LIBHBCU))
    lib.hbcu_last_error.restype = C.c_char_p
    lib.hbcu_frame_release.argtypes = [C.c_void_p]
    lib.hbcu_deint_frame.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                     C.c_void_p, C.c_void_p, C.c_void_p]
    if lib.hbcu_device_count() < 1:
        raise SystemExit("no CUDA device: nothing measured")
    name, pl = gpu_info()
    cases = [bench_case(lib, size, depth, algo, field, a.launches, a.warmup)
             for size, depth in CASES for algo in ALGOS for field in (False, True)]
    lib.hbcu_frame_trim()
    import os
    os.environ["HBCU_UPLOAD_EXTERNAL"] = "1"
    flt = handbrake_b200.filters().lib
    flt.hb_bench_run_chain.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                       C.c_int, C.c_int, C.c_void_p]
    clip = p010_clip(3840, 2160, 10)
    for arm in CHAINS:                                  # warm-up: modules, pools, NLMeans plans
        chain_rate(flt, arm, clip, 10)
    runs = {arm: [] for arm in CHAINS}
    for _ in range(3):
        for arm in CHAINS:
            runs[arm].append(round(chain_rate(flt, arm, clip, a.frames), 1))
    print(json.dumps(dict(gpu=name, power_limit=pl, cases=cases,
                          chain_4k_p010_comb_detect_deint_nlmeans_medium_fps=dict(bwdif_mode35=runs["bwdif"],
                                                                                  decomb_mode39=runs["decomb"],
                                                                                  frames_per_run=a.frames))), flush=True)


if __name__ == "__main__":
    main()
