"""hb_filter_yadif_cuda and hb_filter_bwdif_cuda: Yadif and Bwdif deinterlacing on the GPU (handbrake_b200/csrc/
deinterlace.cu), the drop-ins for libhb's Deinterlace filter (deinterlace.c, FFmpeg's yadif / bwdif behind an avfilter
graph).

Expected values come from a numpy restatement of the rules in DESIGN.md 4.9, written here independently of the C
restatement in oracle/deint/deint_port.c: the per-sample arithmetic, the frame window, the field order, Bwdif's
field-end state, timestamps and flags.  CPU tests run the filters' host side (deinterlace_cuda.c, untouched) over the C
restatement in oracle/_ref/libhostlogic_deint.so (oracle/deint.mk) and compare it with numpy; GPU tests compare the CUDA
filters with that host logic.  Yadif's interior rows (3 .. h-4) are also pinned against the reference's own decomb
(mode=1, whose yadif_filter_line is the same arithmetic there) through the stored digests of tests/golden/."""
import ctypes as C

import numpy as np
import pytest

from golden_ref import REPO
from handbrake_b200 import synth
from handbrake_b200.hblib import FilterLib
from test_format_gpu import CLOSE_FN, INIT_FN, WORK_FN, Buffer, FilterInit, FilterObject, clear_next
from test_oracle import decomb_inputs

HOSTLOGIC_DEINT_SO = REPO / "oracle" / "_ref" / "libhostlogic_deint.so"
YADIF, BWDIF = "hb_filter_yadif_cuda", "hb_filter_bwdif_cuda"
UP, DOWN = "hb_filter_hbcu_upload", "hb_filter_hbcu_download"
TFF, PROG = synth.PIC_FLAG_TOP_FIELD_FIRST, synth.PIC_FLAG_PROGRESSIVE_FRAME

# name -> (pix_fmt, log2 chroma w, log2 chroma h, depth)
FORMATS = {
    "yuv420p": (0, 1, 1, 8), "yuv422p": (4, 1, 0, 8), "yuv444p": (5, 0, 0, 8),
    "yuv420p10le": (62, 1, 1, 10), "yuv422p10le": (64, 1, 0, 10), "yuv444p10le": (68, 0, 0, 10),
    "yuv420p12le": (123, 1, 1, 12), "yuv420p16le": (47, 1, 1, 16),
}
END, NORMAL, BACK_END = "end", "normal", "back_end"


# ------------------------------------------------------------------------------------------------- numpy restatement
def plane_dims(fmt, w, h):
    _, sw, sh, _ = FORMATS[fmt]
    cw, ch = -((-w) >> sw), -((-h) >> sh)
    return [(w, h), (cw, ch), (cw, ch)]


def dtype_of(fmt):
    return np.uint8 if FORMATS[fmt][3] == 8 else np.uint16


def split(frame, fmt, w, h):
    dt, out, off = dtype_of(fmt), [], 0
    for pw, ph in plane_dims(fmt, w, h):
        n = pw * ph * np.dtype(dt).itemsize
        out.append(np.ascontiguousarray(frame[off: off + n]).view(dt).reshape(ph, pw).astype(np.int64))
        off += n
    return out


def pack(planes, fmt):
    return np.concatenate([p.astype(dtype_of(fmt)).view(np.uint8).ravel() for p in planes])


def yadif_plane(P, Cu, N, parity, tff, spatial):
    h, w = Cu.shape
    P2, N2 = (P, Cu) if parity ^ tff else (Cu, N)
    out = Cu.copy()
    for y in range(h):
        if not (y ^ parity) & 1:
            continue
        m, n = (-1 if y else 1), (1 if y + 1 < h else -1)
        U, D = Cu[y + m], Cu[y + n]
        d = (P2[y] + N2[y]) >> 1
        td0 = np.abs(P2[y] - N2[y])
        td1 = (np.abs(P[y + m] - U) + np.abs(P[y + n] - D)) >> 1
        td2 = (np.abs(N[y + m] - U) + np.abs(N[y + n] - D)) >> 1
        diff = np.maximum(np.maximum(td0 >> 1, td1), td2)
        pred = (U + D) >> 1
        if w > 6:
            xs = np.arange(3, w - 3)
            score = np.abs(U[xs - 1] - D[xs - 1]) + np.abs(U[xs] - D[xs]) + np.abs(U[xs + 1] - D[xs + 1]) - 1
            pr = pred[xs].copy()
            for side in (-1, 1):
                improved = np.ones(len(xs), bool)
                for j in (side, 2 * side):
                    s = sum(np.abs(U[xs + i + j] - D[xs + i - j]) for i in (-1, 0, 1))
                    better = improved & (s < score)
                    score = np.where(better, s, score)
                    pr = np.where(better, (U[xs + j] + D[xs - j]) >> 1, pr)
                    improved = better
            pred[xs] = pr
        if spatial and y != 1 and y != h - 2:
            b = (P2[y + 2 * m] + N2[y + 2 * m]) >> 1
            f = (P2[y + 2 * n] + N2[y + 2 * n]) >> 1
            mx = np.maximum(np.maximum(d - D, d - U), np.minimum(b - U, f - D))
            mn = np.minimum(np.minimum(d - D, d - U), np.maximum(b - U, f - D))
            diff = np.maximum(np.maximum(diff, mn), -mx)
        out[y] = np.minimum(np.maximum(pred, d - diff), d + diff)
    return out


def bwdif_plane(P, Cu, N, parity, tff, intra, depth):
    h, w = Cu.shape
    P2, N2 = (P, Cu) if parity ^ tff else (Cu, N)
    df, maxv = (1 if depth == 8 else 2), (1 << depth) - 1
    out = Cu.copy()
    row = lambda a, y: a[min(max(y, 0), h - 1)]       # intra rows the row-step quirk puts outside the plane
    for y in range(h):
        if not (y ^ parity) & 1:
            continue
        m, n = (-1 if y > df - 1 else 1), (1 if y + df < h else -1)
        if intra:
            m3, n3 = (-3 if y > 3 * df - 1 else 1), (3 if y + 3 * df < h else -1)
            v = (5077 * (Cu[y + m] + Cu[y + n]) - 981 * (row(Cu, y + m3) + row(Cu, y + n3))) >> 13
            out[y] = np.clip(v, 0, maxv)
            continue
        edge = y < 4 or y + 5 > h
        if not edge:
            m, n = -1, 1
        c, e = Cu[y + m], Cu[y + n]
        d = (P2[y] + N2[y]) >> 1
        td0 = np.abs(P2[y] - N2[y])
        td1 = (np.abs(P[y + m] - c) + np.abs(P[y + n] - e)) >> 1
        td2 = (np.abs(N[y + m] - c) + np.abs(N[y + n] - e)) >> 1
        diff = np.maximum(np.maximum(td0 >> 1, td1), td2)
        still = diff == 0
        if not edge or not (y < 2 or y + 3 > h):
            b = ((P2[y - 2] + N2[y - 2]) >> 1) - c
            f = ((P2[y + 2] + N2[y + 2]) >> 1) - e
            mx = np.maximum(np.maximum(d - e, d - c), np.minimum(b, f))
            mn = np.minimum(np.minimum(d - e, d - c), np.maximum(b, f))
            diff = np.maximum(np.maximum(diff, mn), -mx)
        if edge:
            interp = (c + e) >> 1
        else:
            r3 = Cu[y - 3] + Cu[y + 3]
            hf = (((5570 * (P2[y] + N2[y]) - 3801 * (P2[y - 2] + N2[y - 2] + P2[y + 2] + N2[y + 2])
                    + 1016 * (P2[y - 4] + N2[y - 4] + P2[y + 4] + N2[y + 4])) >> 2) + 4309 * (c + e) - 213 * r3) >> 13
            sp = (5077 * (c + e) - 981 * r3) >> 13
            interp = np.where(np.abs(c - e) > td0, hf, sp)
        v = np.clip(np.minimum(np.maximum(interp, d - diff), d + diff), 0, maxv)
        out[y] = np.where(still, d, v)
    return out


def halve(v):
    return (v + 1) // 2 if v >= 0 else -((-v + 1) // 2)


def deint_stream(clip, fmt, w, h, bwdif, mode, parity, flags, combed, start, stop, new_chap):
    """the whole filter: (frames, start, stop, flags, combed, new_chap) of every output, in order"""
    n = len(clip)
    if not mode & 1:
        return clip, list(start), list(stop), list(flags), list(combed), list(new_chap)
    field, sel, spatial = bool(mode & 4), bool(mode & 32), bool(mode & 2)
    state, outs = END, []
    planes = [split(f, fmt, w, h) for f in clip]
    for t in range(n):
        last = t == n - 1
        if last:
            state = BACK_END
        s_next = 2 * start[t] - start[max(t - 1, 0)] if last else start[t + 1]
        stop_last = stop[t] if last else start[t + 1]
        if sel and combed[t] == 0:
            outs.append((clip[t], start[t], stop_last, flags[t] | PROG, 0, new_chap[t]))
            continue
        tff = 1 if parity == 0 else 0 if parity == 1 else (int(bool(flags[t] & TFF)) if combed[t] else 1)
        P, Cu, N = planes[max(t - 1, 0)], planes[t], planes[min(t + 1, n - 1)]
        npics = 2 if field else 1
        mid = halve(start[t] + s_next)
        for k in range(npics):
            par = (1 - tff) ^ k
            if k == 1 and state == BACK_END:
                state = END
            intra = bwdif and state == END
            if state == END:
                state = NORMAL
            if bwdif:
                pl = [bwdif_plane(P[i], Cu[i], N[i], par, tff, intra, FORMATS[fmt][3]) for i in range(3)]
            else:
                pl = [yadif_plane(P[i], Cu[i], N[i], par, tff, spatial) for i in range(3)]
            outs.append((pack(pl, fmt), start[t] if k == 0 else mid, mid if k + 1 < npics else stop_last,
                         flags[t] | PROG, 0, new_chap[t] if k == 0 else 0))
    cols = list(zip(*outs))
    return (np.stack(cols[0]),) + tuple(list(c) for c in cols[1:])


def clip_of(fmt, w, h, n, seed):
    """an interlaced-looking clip (the fields of each frame from different times) with full-range noise mixed in"""
    rng = np.random.default_rng(seed + 31 * w + h)
    depth, out = FORMATS[fmt][3], []
    for t in range(n):
        pl = []
        for pw, ph in plane_dims(fmt, w, h):
            yy, xx = np.mgrid[0:ph, 0:pw]
            base = ((xx * 7 + (yy + 3 * t + (yy & 1) * 5) * 11) % 97) << (depth - 7)
            noise = rng.integers(0, 1 << depth, (ph, pw))
            pl.append(np.where(rng.random((ph, pw)) < 0.15, noise, base) & ((1 << depth) - 1))
        out.append(pack(pl, fmt))
    return np.stack(out)


def stream_inputs(n, seed, odd_times=False):
    rng = np.random.default_rng(seed)
    flags = np.array([TFF if rng.random() < 0.6 else 0 for _ in range(n)], np.uint16)
    combed = np.array([(2, 0, 1, 2, 0, 0, 2)[(i + seed) % 7] for i in range(n)], np.uint8)
    if odd_times:
        start = np.cumsum(rng.integers(1000, 4000, n)) - 1501          # odd S_t + S_t+1 sums, one negative start
        start[0] = -7
    else:
        start = np.arange(n, dtype=np.int64) * 3003
    stop = start + 3003
    return flags, combed, start.astype(np.int64), stop.astype(np.int64), np.arange(n, dtype=np.int32) + 1


def run_filter(lib, name, settings, clip, fmt, w, h, n, seed, odd_times=False, chain=None):
    flags, combed, start, stop, chap = stream_inputs(n, seed, odd_times)
    names, sets = [name], [settings]
    if chain == "device":
        names, sets = [UP, name, DOWN], [None, settings, None]
    r = lib.run(names, sets, clip, FORMATS[fmt][0], w, h, flags=flags, combed=combed, start=start, stop=stop, new_chap=chap)
    return r, (flags, combed, start, stop, chap)


def expect(r, want):
    frames, start, stop, flags, combed, chap = want
    assert not r.init_failed and r.saw_eof
    assert r.frames.shape == frames.shape, (r.frames.shape, frames.shape)
    for i in range(len(frames)):
        assert np.array_equal(r.frames[i], frames[i]), f"output {i} differs"
    assert list(r.start) == list(start) and list(r.stop) == list(stop)
    assert list(r.duration) == [float(b - a) for a, b in zip(start, stop)]
    assert list(r.flags) == list(flags) and list(r.combed) == list(combed) and list(r.new_chap) == list(chap)


# the case grid: (filter, mode, parity, format, w, h, frames)
CASES = [
    (YADIF, 1, -1, "yuv420p", 37, 23, 7), (YADIF, 3, -1, "yuv420p10le", 37, 23, 7), (YADIF, 5, 0, "yuv422p", 30, 19, 7),
    (YADIF, 7, 1, "yuv444p10le", 21, 17, 2), (YADIF, 39, -1, "yuv420p12le", 37, 23, 7), (YADIF, 35, 1, "yuv420p16le", 26, 15, 7),
    (YADIF, 7, -1, "yuv420p", 3, 3, 2), (YADIF, 3, 0, "yuv444p", 3, 3, 1), (YADIF, 5, -1, "yuv422p10le", 9, 7, 1),
    (BWDIF, 3, -1, "yuv420p", 37, 23, 7), (BWDIF, 7, -1, "yuv420p10le", 37, 23, 7), (BWDIF, 7, 0, "yuv444p", 29, 13, 2),
    (BWDIF, 35, -1, "yuv420p16le", 33, 21, 7), (BWDIF, 39, 1, "yuv422p", 24, 11, 7), (BWDIF, 7, 1, "yuv420p12le", 11, 13, 1),
    (BWDIF, 7, -1, "yuv420p10le", 5, 7, 2), (BWDIF, 3, 0, "yuv444p10le", 3, 4, 7), (BWDIF, 7, -1, "yuv420p", 5, 7, 1),
    (BWDIF, 7, 0, "yuv422p10le", 6, 5, 2), (BWDIF, 39, -1, "yuv444p10le", 4, 6, 7),
]


def case_id(c):
    return f"{c[0][10:15]}-m{c[1]}-p{c[2]}-{c[3]}-{c[4]}x{c[5]}-n{c[6]}"


def expected(case, clip, inputs):
    name, mode, parity, fmt, w, h, n = case
    return deint_stream(clip, fmt, w, h, name == BWDIF, mode, parity, *inputs)


# ------------------------------------------------------------------------------------------------- CPU tests
@pytest.fixture(scope="module")
def host():
    return FilterLib(HOSTLOGIC_DEINT_SO)


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_restatement_equals_numpy(host, case):
    """the host logic over the C restatement == the numpy restatement: pictures, times, flags, combed, chapters"""
    name, mode, parity, fmt, w, h, n = case
    clip = clip_of(fmt, w, h, n, seed=n)
    for odd in (False, True):
        r, inputs = run_filter(host, name, f"mode={mode}:parity={parity}" if parity >= 0 else f"mode={mode}",
                               clip, fmt, w, h, n, seed=n + w, odd_times=odd)
        expect(r, expected(case, clip, inputs))
        assert r.vrate == ((60000, 1001) if mode & 4 else (30000, 1001))
    assert host.buffers_alive() == 0


@pytest.mark.parametrize("name", [YADIF, BWDIF])
def test_identity_fields_and_registry(host, name):
    obj = FilterObject.in_dll(host.lib, name)
    want = (7, b"deinterlace", b"Deinterlace") if name == YADIF else (9, b"bwdif", b"Bwdif")
    assert (obj.id, obj.short_name, obj.skip, obj.enforce_order) == (want[0], want[1], 0, 1)
    assert obj.name == want[2]
    assert obj.settings_template == b"mode=^([0-9]+)$:parity=^([01])$"
    import handbrake_b200
    flt = handbrake_b200.filters()
    flt.lib.hb_filter_get.restype = C.c_void_p
    assert flt.lib.hb_filter_get(want[0]) == flt.filter_object(name)


@pytest.mark.parametrize("name", [YADIF, BWDIF])
def test_pass_through_without_mode_1(host, name):
    clip = clip_of("yuv420p", 16, 8, 3, seed=1)
    for s in ("mode=0", "mode=4", "mode=38"):
        r, _ = run_filter(host, name, s, clip, "yuv420p", 16, 8, 3, seed=2)
        assert np.array_equal(r.frames, clip) and r.vrate == (30000, 1001) and not r.init_failed
        assert list(r.start) == [0, 3003, 6006]
    assert host.buffers_alive() == 0


@pytest.mark.parametrize("name,fmt,w,h,refused", [
    (YADIF, "nv12", 16, 8, True), (YADIF, "p010le", 16, 8, True), (YADIF, "gray", 16, 8, True),
    (YADIF, "yuva420p", 16, 8, True), (BWDIF, "yuva444p", 16, 8, True), (BWDIF, "nv12", 16, 8, True),
    (YADIF, "yuv420p", 2, 8, True), (YADIF, "yuv420p", 8, 2, True), (YADIF, "yuv420p", 3, 3, False),
    (BWDIF, "yuv420p", 5, 7, False), (BWDIF, "yuv420p", 4, 7, True), (BWDIF, "yuv420p", 5, 6, True),
    (BWDIF, "yuv444p", 3, 4, False), (BWDIF, "yuv444p", 2, 4, True), (BWDIF, "yuv444p", 3, 3, True),
])
def test_init_refusals(host, name, fmt, w, h, refused):
    """init fails (and leaves vrate alone) for semi-planar, gray and YUVA input and for planes under the minimum"""
    pix = {"nv12": 23, "p010le": 158, "gray": 8, "yuva420p": 33, "yuva444p": 79}.get(fmt) or FORMATS[fmt][0]
    obj = FilterObject.from_buffer_copy(FilterObject.in_dll(host.lib, name))
    host.lib.hb_parse_filter_settings.restype = C.c_void_p
    host.lib.hb_parse_filter_settings.argtypes = [C.c_char_p]
    obj.settings = host.lib.hb_parse_filter_settings(b"mode=7")
    init = FilterInit(pix_fmt=pix, hw_pix_fmt=-1, width=w, height=h, par_num=1, par_den=1)
    init.vrate[0], init.vrate[1] = 30000, 1001
    rc = INIT_FN(obj.init)(C.addressof(obj), C.addressof(init))
    assert (rc != 0) == refused
    assert init.vrate[0] == (30000 if refused else 60000)
    if rc == 0:
        CLOSE_FN(obj.close)(C.addressof(obj))
    host.lib.hb_dict_free.argtypes = [C.POINTER(C.c_void_p)]
    host.lib.hb_dict_free(C.byref(C.c_void_p(obj.settings)))
    assert host.buffers_alive() == 0


def test_bwdif_field_end_state(host):
    """intra pictures: the first deinterlaced picture (after a selective run of uncombed frames) and, in field mode, the
    last frame's second picture; the numpy stream marks them, and an intra picture differs from the normal rule's"""
    fmt, w, h, n = "yuv420p", 24, 16, 6
    clip = clip_of(fmt, w, h, n, seed=4)
    flags = np.full(n, TFF, np.uint16)
    combed = np.array([0, 0, 2, 2, 0, 2], np.uint8)
    start = np.arange(n, dtype=np.int64) * 3003
    chap = np.zeros(n, np.int32)
    for mode in (7, 39, 3):
        r = host.run(BWDIF, f"mode={mode}", clip, 0, w, h, flags=flags, combed=combed, start=start, stop=start + 3003,
                     new_chap=chap)
        want = deint_stream(clip, fmt, w, h, True, mode, -1, flags, combed, start, start + 3003, chap)
        expect(r, want)
    # frames 0 and 1 pass through in selective mode: frame 2's picture is the intra one (the top rows follow the intra rule)
    r = host.run(BWDIF, "mode=35", clip, 0, w, h, flags=flags, combed=combed, start=start, stop=start + 3003, new_chap=chap)
    assert np.array_equal(r.frames[0], clip[0]) and np.array_equal(r.frames[1], clip[1])
    P = [split(f, fmt, w, h) for f in clip]
    intra = pack([bwdif_plane(P[1][i], P[2][i], P[3][i], 0, 1, True, 8) for i in range(3)], fmt)
    assert np.array_equal(r.frames[2], intra)
    assert host.buffers_alive() == 0


@pytest.mark.parametrize("depth", [8, 10])
def test_yadif_interior_rows_match_reference_decomb(ref, depth):
    """the anchor: rows 3 .. h-4 of every plane of every picture of Yadif mode=3:parity=0 == the reference's decomb
    mode=1:parity=0 (yadif_filter_line, tff = 1 on both sides) on the stored calls of test_oracle.py"""
    fmt = "yuv420p" if depth == 8 else "yuv420p10le"
    w, h = 96, 50
    clip, flags, combed = decomb_inputs(depth, w, h, 6)
    r = ref.run("hb_filter_decomb", "mode=1:parity=0", clip, FORMATS[fmt][0], w, h, flags=flags)
    n = len(clip)
    start = np.arange(n, dtype=np.int64) * 3003
    mine = deint_stream(clip, fmt, w, h, False, 3, 0, flags, np.ones(n, np.uint8), start, start + 3003, np.arange(n))[0]
    assert r.frames.shape == mine.shape
    for a, b in zip(r.frames, mine):
        for pa, pb in zip(split(a, fmt, w, h), split(b, fmt, w, h)):
            assert np.array_equal(pa[3: pa.shape[0] - 3], pb[3: pb.shape[0] - 3])
    assert ref.buffers_alive() == 0


def drive(lib, name, settings, bufs):
    """init / work / close of one filter instance by hand, as libhb calls them: the addresses of every output buffer
    (EOF included), in order, and their (flags, combed) as they left the filter; the outputs are closed"""
    lib.hb_parse_filter_settings.restype = C.c_void_p
    lib.hb_parse_filter_settings.argtypes = [C.c_char_p]
    lib.hb_buffer_close.argtypes = [C.POINTER(C.c_void_p)]
    lib.hb_buffer_eof_init.restype = C.c_void_p
    lib.hb_dict_free.argtypes = [C.POINTER(C.c_void_p)]
    obj = FilterObject.from_buffer_copy(FilterObject.in_dll(lib, name))
    obj.settings = lib.hb_parse_filter_settings(settings.encode())
    b0 = Buffer.from_address(bufs[0])
    init = FilterInit(pix_fmt=b0.f.fmt, hw_pix_fmt=-1, width=b0.f.width, height=b0.f.height, par_num=1, par_den=1)
    init.vrate[0], init.vrate[1] = 30000, 1001
    assert INIT_FN(obj.init)(C.addressof(obj), C.addressof(init)) == 0
    outs = []
    for b in list(bufs) + [lib.hb_buffer_eof_init()]:
        bin_, bout = C.c_void_p(b), C.c_void_p()
        WORK_FN(obj.work)(C.addressof(obj), C.byref(bin_), C.byref(bout))
        p = bout.value
        while p:
            outs.append(p)
            p = C.c_void_p.from_address(p + Buffer.next_offset).value
    CLOSE_FN(obj.close)(C.addressof(obj))
    lib.hb_dict_free(C.byref(C.c_void_p(obj.settings)))
    seen = [(o, Buffer.from_address(o).s.flags, Buffer.from_address(o).s.combed, Buffer.from_address(o).plane[0].data)
            for o in outs]
    for o in outs:
        clear_next(o)
        lib.hb_buffer_close(C.byref(C.c_void_p(o)))
    return seen


def selective_not_a_copy(lib, name, device):
    """mode=39: the uncombed frames leave as the input itself (a host buffer) or as a shallow duplicate sharing the input's
    device frame, never as a copy (a copy is made while the input is still held, so it cannot share its planes)"""
    w, h, n = 32, 16, 5
    combed = [2, 0, 2, 0, 0]
    lib.hb_harness_frame_from_packed.restype = C.c_void_p
    lib.hb_harness_frame_from_packed.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.hbcu_device_frame_buffer_init.restype = C.c_void_p
    lib.hbcu_device_frame_buffer_init.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int]
    clip = clip_of("yuv420p", w, h, n, seed=3)
    bufs, planes = [], []
    for t in range(n):
        b = lib.hbcu_device_frame_buffer_init(0, w, h, 0) if device else \
            lib.hb_harness_frame_from_packed(0, w, h, np.ascontiguousarray(clip[t]).ctypes.data)
        bb = Buffer.from_address(b)
        bb.s.start, bb.s.stop, bb.s.flags, bb.s.combed = 3003 * t, 3003 * (t + 1), TFF, combed[t]
        bufs.append(b)
        planes.append(bb.plane[0].data)
    seen = drive(lib, name, "mode=39", bufs)
    pics = [x for x in seen if not x[1] & 0x0400]                  # HB_BUF_FLAG_EOF
    assert len(pics) == 2 * 2 + 3
    k = 0
    for t in range(n):
        if combed[t]:
            for _ in range(2):
                assert pics[k][2] == 0 and pics[k][1] & PROG
                k += 1
        else:
            out, flags, cb, plane0 = pics[k]
            assert plane0 == planes[t], "an uncombed frame was copied"
            assert (out == bufs[t]) != device and flags & PROG and cb == 0
            k += 1


@pytest.mark.parametrize("name", [YADIF, BWDIF])
@pytest.mark.parametrize("device", [False, True])
def test_selective_pass_through_is_not_a_copy(host, name, device):
    selective_not_a_copy(host.lib, name, device)
    assert host.buffers_alive() == 0


# ------------------------------------------------------------------------------------------------- GPU tests
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_cuda_equals_host_logic(host, cuda_filters, case):
    """host buffers, and device buffers behind the upload adapter: the same pictures, times, flags and combed"""
    name, mode, parity, fmt, w, h, n = case
    clip = clip_of(fmt, w, h, n, seed=n)
    s = f"mode={mode}:parity={parity}" if parity >= 0 else f"mode={mode}"
    want, _ = run_filter(host, name, s, clip, fmt, w, h, n, seed=n + w, odd_times=True)
    for chain in (None, "device"):
        g, _ = run_filter(cuda_filters, name, s, clip, fmt, w, h, n, seed=n + w, odd_times=True, chain=chain)
        expect(g, (want.frames, want.start, want.stop, want.flags, want.combed, want.new_chap))
    assert cuda_filters.buffers_alive() == 0


@pytest.mark.gpu
@pytest.mark.parametrize("name,mode,fmt,w,h", [(BWDIF, 7, "yuv420p", 1920, 1080), (YADIF, 3, "yuv420p", 1920, 1080),
                                               (BWDIF, 3, "yuv420p10le", 3840, 2160), (YADIF, 7, "yuv420p10le", 3840, 2160)])
def test_full_size_frames(host, cuda_filters, name, mode, fmt, w, h):
    clip = clip_of(fmt, w, h, 3, seed=9)
    want, _ = run_filter(host, name, f"mode={mode}", clip, fmt, w, h, 3, seed=5)
    for chain in (None, "device"):
        g, _ = run_filter(cuda_filters, name, f"mode={mode}", clip, fmt, w, h, 3, seed=5, chain=chain)
        assert g.frames.shape == want.frames.shape
        bad = [i for i in range(len(g.frames)) if not np.array_equal(g.frames[i], want.frames[i])]
        assert not bad, f"pictures {bad} differ"
        assert list(g.start) == list(want.start) and list(g.stop) == list(want.stop)
    assert cuda_filters.buffers_alive() == 0


@pytest.mark.gpu
@pytest.mark.parametrize("depth", [8, 10])
def test_yadif_anchor_on_gpu(ref, cuda_filters, depth):
    """the anchor on the GPU: Yadif mode=3:parity=0 against the reference's decomb mode=1:parity=0 on the 200 x 106
    clips of test_decomb_gpu.py, rows 3 .. h-4 of every plane"""
    fmt = "yuv420p" if depth == 8 else "yuv420p10le"
    w, h = 200, 106
    clip, flags, combed = decomb_inputs(depth, w, h, 7)
    r = ref.run("hb_filter_decomb", "mode=1:parity=0", clip, FORMATS[fmt][0], w, h, flags=flags)
    g = cuda_filters.run(YADIF, "mode=3:parity=0", clip, FORMATS[fmt][0], w, h, flags=flags)
    assert g.frames.shape == r.frames.shape
    for a, b in zip(r.frames, g.frames):
        for pa, pb in zip(split(a, fmt, w, h), split(b, fmt, w, h)):
            assert np.array_equal(pa[3: pa.shape[0] - 3], pb[3: pb.shape[0] - 3])
    assert cuda_filters.buffers_alive() == 0


@pytest.mark.gpu
def test_device_chain_comb_detect_bwdif_nlmeans(host, cuda_filters):
    """upload -> comb_detect -> bwdif mode=35 -> NLMeans -> download == the same chain through the host logic, with
    both combed and uncombed frames in the stream"""
    w, h = 192, 108
    clip, flags, _ = decomb_inputs(8, w, h, 10, seed=9)
    names = [UP, "hb_filter_comb_detect_cuda", BWDIF, "hb_filter_nlmeans_cuda", DOWN]
    sets = [None, None, "mode=35", "y-strength=6", None]
    want = host.run(names, sets, clip, 0, w, h, flags=flags)
    g = cuda_filters.run(names, sets, clip, 0, w, h, flags=flags)
    assert g.frames.shape == want.frames.shape and np.array_equal(g.frames, want.frames)
    assert list(g.start) == list(want.start) and list(g.flags) == list(want.flags)
    passed = [np.array_equal(f, c) for f, c in zip(host.run(names[:3] + [DOWN], sets[:3] + [None], clip, 0, w, h,
                                                                  flags=flags).frames, clip)]
    assert any(passed) and not all(passed), "the chain should see both combed and uncombed frames"
    assert cuda_filters.buffers_alive() == 0 and host.buffers_alive() == 0


@pytest.mark.gpu
@pytest.mark.parametrize("name", [YADIF, BWDIF])
@pytest.mark.parametrize("device", [False, True])
def test_selective_pass_through_is_not_a_copy_on_gpu(cuda_filters, name, device):
    selective_not_a_copy(cuda_filters.lib, name, device)
    assert cuda_filters.buffers_alive() == 0


@pytest.mark.gpu
def test_decoder_pitch_surfaces_through_format_and_bwdif():
    """NV12 surfaces as NVDEC hands them over (torch-allocated, a 512-byte-aligned pitch wider than the row, written on
    their own stream) wrapped with hbcu_frame_wrap -> hbcu_format_* to yuv420p -> hbcu_deint_* Bwdif, field mode: both
    pictures equal the numpy restatement on the de-interleaved frames, and every surface goes back to its owner"""
    import sys
    import torch
    from test_rotate_gpu import REL, core, to_nv12, wrap_torch
    sys.path.insert(0, str(REPO / "tools"))
    from bench_deinterlace import DeintConfig
    from bench_format import FormatConfig, alloc
    lib = core()
    lib.hbcu_deint_frame.argtypes = [C.c_void_p] * 4 + [C.c_int] * 3 + [C.c_void_p] * 3
    w, h = 1280, 720
    clip = clip_of("yuv420p", w, h, 3, seed=12)
    semi = to_nv12(clip, w, h)
    released = []
    rel = REL(lambda opaque: released.append(int(opaque or 0)))
    side = torch.cuda.Stream()
    pitch = (w + 511) // 512 * 512 + 512
    fmt_h, deint_h, xfer = C.c_void_p(), C.c_void_p(), C.c_void_p()
    assert lib.hbcu_format_create(C.byref(fmt_h), C.byref(FormatConfig(w, h, 8, 0, 0, 4))) == 0, lib.hbcu_last_error()
    cfg = DeintConfig(2, (C.c_int * 3)(w, w // 2, w // 2), (C.c_int * 3)(h, h // 2, h // 2), 1, 8, 0)
    assert lib.hbcu_deint_create(C.byref(deint_h), C.byref(cfg)) == 0, lib.hbcu_last_error()
    assert lib.hbcu_xfer_create(C.byref(xfer), 0, 8) == 0
    shp = [(w, h, (w + 63) // 64 * 64), (w // 2, h // 2, (w // 2 + 63) // 64 * 64), (w // 2, h // 2, (w // 2 + 63) // 64 * 64)]
    planar, surfs = [], []
    for t in range(3):
        fin, surf, _ = wrap_torch(lib, torch, "nv12", w, h, pitch, 0, side, semi[t], rel, t + 1)
        surfs.append(surf)
        f = alloc(lib, shp)
        assert lib.hbcu_format_convert(fmt_h, C.c_int64(t), fin, None, None, f, None, None) == 0, lib.hbcu_last_error()
        lib.hbcu_frame_release(fin)
        planar.append(f)
    outs = [alloc(lib, shp) for _ in range(2)]
    assert lib.hbcu_deint_frame(deint_h, planar[0], planar[1], planar[2], 1, 1, 2, (C.c_void_p * 2)(*outs),
                                (C.c_int * 2)(0, 1), (C.c_int * 2)(0, 0)) == 0, lib.hbcu_last_error()
    P, Cu, N = [split(f, "yuv420p", w, h) for f in clip]
    for k, o in enumerate(outs):
        got = [np.zeros((rows, pt), np.uint8) for _, rows, pt in shp]
        ps = (C.c_void_p * 3)(*[g.ctypes.data for g in got])
        st = (C.c_int * 3)(*[pt for _, _, pt in shp])
        assert lib.hbcu_xfer_download(xfer, C.c_int64(k), o, ps, st) == 0 and lib.hbcu_xfer_wait(xfer, C.c_int64(k)) == 0
        for i in range(3):
            want = bwdif_plane(P[i], Cu[i], N[i], k, 1, False, 8)
            assert np.array_equal(got[i][:, : shp[i][0]], want), (k, i)
    assert lib.hbcu_deint_sync(deint_h) == 0 and lib.hbcu_format_sync(fmt_h) == 0
    assert sorted(released) == [1, 2, 3]
    for f in planar + outs:
        lib.hbcu_frame_release(f)
    lib.hbcu_deint_destroy(deint_h)
    lib.hbcu_format_destroy(fmt_h)
    lib.hbcu_xfer_destroy(xfer)
    del surfs
    assert lib.hbcu_frames_alive() == 0
