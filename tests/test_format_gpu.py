"""hb_filter_format_cuda: nv12 <-> yuv420p and p010le <-> yuv420p10le on the GPU (handbrake_b200/csrc/format.cu), the
drop-in for libhb's format filter (format.c) at the two ends of a hardware-decoded, hardware-encoded chain.

Expected values are computed here in numpy from FFmpeg's pixel-format descriptors: luma copied (>> 6 from P010, << 6 to
it), the Cb/Cr pairs of the semi-planar plane 1 split into planes 1 and 2 or interleaved back.  Chains that run other
filters behind the format filter are compared with the reference's planar chain on the de-interleaved input, whose
results are stored in tests/golden/format_chain_ref_digests.json (`HBCU_RECORD_REF=1` with the reference built records
them through the CPU tests, which make every reference call the GPU tests make).

CPU tests run the host side of the filter (init, pass-through, refusals, props, EOF, buffer ownership) over the plain-C
restatement of the repacks in oracle/_ref/libhostlogic_format.so (oracle/format.mk)."""
import ctypes as C
import json
import os
import re
from pathlib import Path

import numpy as np
import pytest

from golden_ref import REPO, GoldenRef, _h
from handbrake_b200 import LIBHBCU, synth
from handbrake_b200.hblib import FilterLib
from test_oracle import decomb_inputs

STORE = Path(__file__).resolve().parent / "golden" / "format_chain_ref_digests.json"
HOSTLOGIC_FORMAT_SO = REPO / "oracle" / "_ref" / "libhostlogic_format.so"
UP, DOWN = "hb_filter_hbcu_upload", "hb_filter_hbcu_download"
FMT = "hb_filter_format_cuda"
AV_PIX_FMT_CUDA = 117

# name -> (pix_fmt, depth, semi-planar)
FORMATS = {"nv12": (synth.PIX_FMT_NV12, 8, True), "yuv420p": (synth.PIX_FMT_YUV420P, 8, False),
           "p010le": (synth.PIX_FMT_P010, 10, True), "yuv420p10le": (synth.PIX_FMT_YUV420P10, 10, False)}
PAIRS = [("nv12", "yuv420p"), ("yuv420p", "nv12"), ("p010le", "yuv420p10le"), ("yuv420p10le", "p010le")]
SIZES = [(1, 1), (2, 2), (33, 17), (64, 48), (1920, 1080), (3840, 2160)]


# ------------------------------------------------------------------------------------------------- numpy restatement
def cdims(w, h):
    return (w + 1) // 2, (h + 1) // 2


def samples(frame, depth):
    return frame.view(np.uint16) if depth > 8 else frame


def convert(frame, src, dst, w, h):
    """one packed frame (planes back to back, rows at their widths) of format src as format dst"""
    depth, semi = FORMATS[src][1], FORMATS[src][2]
    a = samples(np.ascontiguousarray(frame), depth).astype(np.uint32)
    cw, ch = cdims(w, h)
    shift = 6 if depth == 10 else 0
    y = a[: w * h]
    dt = np.uint16 if depth > 8 else np.uint8
    if semi:
        uv = a[w * h:].reshape(ch, 2 * cw) >> shift
        out = np.concatenate([y >> shift, uv[:, 0::2].ravel(), uv[:, 1::2].ravel()])
    else:
        u, v = a[w * h: w * h + cw * ch].reshape(ch, cw), a[w * h + cw * ch:].reshape(ch, cw)
        uv = np.empty((ch, 2 * cw), np.uint32)
        uv[:, 0::2], uv[:, 1::2] = u, v
        out = (np.concatenate([y, uv.ravel()]) << shift) & 0xFFFF
    return out.astype(dt).view(np.uint8)


def clip_of(fmt, w, h, n, seed):
    """random frames of `fmt`; P010 samples carry non-zero padding bits, which the conversion drops"""
    depth = FORMATS[fmt][1]
    rng = np.random.default_rng(seed + 7 * w + h)
    count = w * h + 2 * np.prod(cdims(w, h))
    if depth == 8:
        return rng.integers(0, 256, (n, count), dtype=np.uint8)
    top = 1 << 16 if fmt == "p010le" else 1 << 10
    return rng.integers(0, top, (n, count), dtype=np.uint16).view(np.uint8)


def to_semi_clip(planar, depth, w, h):
    src = "yuv420p" if depth == 8 else "yuv420p10le"
    return np.stack([convert(f, src, "nv12" if depth == 8 else "p010le", w, h) for f in planar])


# ------------------------------------------------------------------------------------------------- direct calls
class FilterInit(C.Structure):
    _fields_ = [("job", C.c_void_p), ("pix_fmt", C.c_int), ("hw_pix_fmt", C.c_int), ("hw_frames_ctx", C.c_void_p),
                ("color_prim", C.c_int), ("color_transfer", C.c_int), ("color_matrix", C.c_int), ("color_range", C.c_int),
                ("chroma_location", C.c_int), ("width", C.c_int), ("height", C.c_int), ("par_num", C.c_int),
                ("par_den", C.c_int), ("crop", C.c_int * 4), ("grayscale", C.c_int), ("vrate", C.c_int * 2), ("cfr", C.c_int),
                ("time_base", C.c_int * 2), ("samplerate", C.c_int), ("sample_fmt", C.c_int),
                ("ch_order", C.c_int), ("ch_nb", C.c_int), ("ch_mask", C.c_uint64), ("ch_opaque", C.c_void_p)]


class FilterObject(C.Structure):
    _fields_ = [("id", C.c_int), ("enforce_order", C.c_int), ("skip", C.c_int), ("aliased", C.c_int),
                ("name", C.c_char_p), ("short_name", C.c_char_p), ("settings", C.c_void_p),
                ("init", C.c_void_p), ("init_thread", C.c_void_p), ("post_init", C.c_void_p), ("work", C.c_void_p),
                ("work_thread", C.c_void_p), ("close", C.c_void_p), ("info", C.c_void_p),
                ("settings_template", C.c_char_p), ("fifo_in", C.c_void_p), ("fifo_out", C.c_void_p),
                ("subtitle", C.c_void_p), ("private_data", C.c_void_p), ("thread", C.c_void_p), ("done", C.c_void_p),
                ("status", C.c_int), ("chapter_val", C.c_int), ("chapter_time", C.c_int64), ("sub_filter", C.c_void_p)]


class BufSettings(C.Structure):
    _fields_ = [("type", C.c_int), ("id", C.c_int), ("start", C.c_int64), ("duration", C.c_double), ("stop", C.c_int64),
                ("renderOffset", C.c_int64), ("pcr", C.c_int64), ("scr_sequence", C.c_int), ("split", C.c_int),
                ("discontinuity", C.c_uint8), ("new_chap", C.c_int), ("frametype", C.c_uint8), ("flags", C.c_uint16),
                ("combed", C.c_uint8)]


class ImageFormat(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("x", "y", "width", "height", "fmt", "color_prim", "color_transfer", "color_matrix",
                                       "color_range", "chroma_location", "max_plane", "window_width", "window_height")]


class Plane(C.Structure):
    _fields_ = [("data", C.c_void_p), ("stride", C.c_int), ("width", C.c_int), ("height", C.c_int), ("size", C.c_int)]


class Buffer(C.Structure):
    _fields_ = [("size", C.c_int), ("alloc", C.c_int), ("data", C.c_void_p), ("offset", C.c_int), ("s", BufSettings),
                ("f", ImageFormat), ("plane", Plane * 4), ("storage", C.c_void_p), ("storage_type", C.c_int)]


HBCU_DEVICE = 4
HB_FILTER_OK, HB_FILTER_DONE = 0, 4
INIT_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p)
WORK_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p))
CLOSE_FN = C.CFUNCTYPE(None, C.c_void_p)


class Direct:
    """one hb_filter_format_cuda instance driven by hand: init / work / close as libhb calls them"""

    def __init__(self, lib, settings, pix_fmt, w, h, hw_pix_fmt=-1):
        self.lib = lib
        lib.hb_parse_filter_settings.restype = C.c_void_p
        lib.hb_parse_filter_settings.argtypes = [C.c_char_p]
        lib.hb_harness_frame_from_packed.restype = C.c_void_p
        lib.hb_harness_frame_from_packed.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p]
        lib.hb_buffer_close.argtypes = [C.POINTER(C.c_void_p)]
        lib.hb_buffer_eof_init.restype = C.c_void_p
        self.obj = FilterObject.from_buffer_copy(FilterObject.in_dll(lib, FMT))
        self.obj.settings = lib.hb_parse_filter_settings(settings.encode()) if settings else None
        self.init = FilterInit(pix_fmt=pix_fmt, hw_pix_fmt=hw_pix_fmt, color_prim=5, color_transfer=6, color_matrix=7,
                               color_range=2, chroma_location=3, width=w, height=h, par_num=1, par_den=1)
        self.rc = INIT_FN(self.obj.init)(C.addressof(self.obj), C.addressof(self.init))

    def frame(self, pix_fmt, w, h, packed, t):
        b = self.lib.hb_harness_frame_from_packed(pix_fmt, w, h, np.ascontiguousarray(packed).ctypes.data)
        buf = Buffer.from_address(b)
        buf.s.start, buf.s.stop, buf.s.new_chap, buf.s.flags, buf.s.combed = 3003 * t, 3003 * (t + 1), t + 10, 0x18, 1
        buf.f.color_prim, buf.f.color_transfer, buf.f.color_matrix, buf.f.color_range, buf.f.chroma_location = 9, 16, 9, 2, 2
        return b

    def work(self, b):
        bin_, bout = C.c_void_p(b), C.c_void_p()
        st = WORK_FN(self.obj.work)(C.addressof(self.obj), C.byref(bin_), C.byref(bout))
        if bin_.value:
            self.lib.hb_buffer_close(C.byref(bin_))
        outs, p = [], bout.value
        while p:
            outs.append(p)
            p = C.c_void_p.from_address(p + Buffer.next_offset).value
        return st, outs

    def close_buffers(self, bufs):
        for b in bufs:
            clear_next(b)
            self.lib.hb_buffer_close(C.byref(C.c_void_p(b)))

    def close(self):
        if self.rc == 0:
            CLOSE_FN(self.obj.close)(C.addressof(self.obj))
        if self.obj.settings:
            self.lib.hb_dict_free.argtypes = [C.POINTER(C.c_void_p)]
            self.lib.hb_dict_free(C.byref(C.c_void_p(self.obj.settings)))


# hb_buffer_t.palette, side_data, nb_side_data, next follow storage_type
Buffer.next_offset = (Buffer.storage_type.offset + 4 + 7) // 8 * 8 + 8 + 8 + 8


def clear_next(b):
    C.c_void_p.from_address(b + Buffer.next_offset).value = None


def packed_of(buf_addr, lib):
    """the host buffer's planes, packed (the harness's own packing)"""
    b = Buffer.from_address(buf_addr)
    depth = 10 if b.f.fmt in (FORMATS["p010le"][0], FORMATS["yuv420p10le"][0]) else 8
    nbytes = (b.f.width * b.f.height + 2 * int(np.prod(cdims(b.f.width, b.f.height)))) * (2 if depth > 8 else 1)
    out = np.zeros(nbytes, np.uint8)
    lib.hb_harness_frame_to_packed.argtypes = [C.c_void_p, C.c_void_p]
    lib.hb_harness_frame_to_packed(buf_addr, out.ctypes.data)
    return out


# ------------------------------------------------------------------------------------------------- the reference
class FormatRef(GoldenRef):
    """GoldenRef over this file's store: the reference's planar chains on the de-interleaved inputs, and the digest of
    format.c's settings template"""

    def __init__(self):
        super().__init__()
        self.store = json.loads(STORE.read_text()) if STORE.exists() else {}

    def _save(self):
        STORE.write_text(json.dumps(dict(sorted(self.store.items())), indent=0) + "\n")

    def template_digest(self):
        if self.recording:
            tree = Path(os.environ["HANDBRAKE_SRC"])      # the HandBrake tree the reference was built from
            common = (tree / "libhb" / "handbrake" / "common.h").read_text()
            fmt_c = (tree / "libhb" / "format.c").read_text()
            all_reg = re.search(r'#define\s+HB_ALL_REG\s+"((?:[^"\\]|\\.)*)"', common).group(1)
            body = re.search(r"format_template\[\]\s*=\s*((?:\s*(?:\"(?:[^\"\\]|\\.)*\"|HB_ALL_REG))+)\s*;", fmt_c).group(1)
            parts = re.findall(r'"((?:[^"\\]|\\.)*)"|(HB_ALL_REG)', body)
            template = "".join(all_reg if macro else lit for lit, macro in parts)
            self.store["format_template"] = _h(template)
            self._save()
        return self.store["format_template"]


@pytest.fixture(scope="module")
def fref():
    return FormatRef()


NV12_CHAIN = (["hb_filter_comb_detect", "hb_filter_decomb", "hb_filter_nlmeans"], [None, "mode=39", "y-strength=6"])
P010_CHAIN = (["hb_filter_nlmeans"], ["y-strength=6:cb-strength=4"])


def nv12_chain_inputs():
    w, h = 256, 144
    clip, flags, _ = decomb_inputs(8, w, h, 8, seed=23)
    return w, h, clip, flags


def p010_chain_inputs():
    w, h = 320, 180
    return w, h, synth.progressive_clip(synth.PIX_FMT_YUV420P10, w, h, 6, seed=29)


def nv12_chain_ref(fref):
    w, h, clip, flags = nv12_chain_inputs()
    return fref.run(*NV12_CHAIN, clip, synth.PIX_FMT_YUV420P, w, h, flags=flags)


def p010_chain_ref(fref):
    w, h, clip = p010_chain_inputs()
    return fref.run(*P010_CHAIN, clip, synth.PIX_FMT_YUV420P10, w, h)


def product(names):
    return [n + "_cuda" for n in names]


# ------------------------------------------------------------------------------------------------- CPU tests
def semi_lib():
    return FilterLib(HOSTLOGIC_FORMAT_SO)


def test_pix_fmt_names():
    lib = semi_lib().lib
    lib.av_get_pix_fmt.argtypes = [C.c_char_p]
    lib.av_get_pix_fmt_name.restype = C.c_char_p
    for name, pix in (("nv12", 23), ("yuv420p", 0), ("p010le", 158), ("p010", 158), ("yuv420p10le", 62),
                      ("yuv420p10", 62), ("p016", 169), ("yuv422p", 4), ("gray", 8), ("bogus", -1), ("p010be", -1)):
        assert lib.av_get_pix_fmt(name.encode()) == pix, name
    for pix, name in ((23, b"nv12"), (158, b"p010le"), (62, b"yuv420p10le"), (0, b"yuv420p"), (9999, None)):
        assert lib.av_get_pix_fmt_name(pix) == name


def test_identity_fields_and_template(fref):
    lib = semi_lib().lib
    obj = FilterObject.in_dll(lib, FMT)
    assert (obj.id, obj.short_name, obj.skip, obj.enforce_order) == (33, b"format", 0, 1)
    assert obj.settings_template == b"format=^(.*)$"
    assert _h(obj.settings_template.decode()) == fref.template_digest()
    import handbrake_b200
    flt = handbrake_b200.filters()
    flt.lib.hb_filter_get.restype = C.c_void_p
    assert flt.lib.hb_filter_get(33) == flt.filter_object(FMT)      # HB_FILTER_FORMAT


@pytest.mark.parametrize("src,dst", PAIRS)
@pytest.mark.parametrize("w,h", SIZES[:4])
def test_host_contract_conversions(src, dst, w, h):
    """the filter over the restatement: host frames and device-frame stand-ins, props travel with their frame"""
    lib = semi_lib()
    clip = clip_of(src, w, h, 3, seed=1)
    want = np.stack([convert(f, src, dst, w, h) for f in clip])
    for chain in ([FMT], [UP, FMT, DOWN]):
        r = lib.run(chain, [f"format={dst}" if c == FMT else None for c in chain], clip, FORMATS[src][0], w, h)
        assert r.init_failed == 0 and r.saw_eof and np.array_equal(r.frames, want), chain
        assert list(r.start) == [3003 * i for i in range(3)] and list(r.new_chap) == [0, 1, 2]
    assert lib.buffers_alive() == 0


def check_passthrough_and_refusals(lib, device=False):
    w, h = 64, 48
    for settings, pix in ((None, FORMATS["nv12"][0]), ("format=nv12", FORMATS["nv12"][0]), ("format=p010", FORMATS["p010le"][0]),
                          ("format=yuv420p10", FORMATS["yuv420p10le"][0]), (None, synth.PIX_FMT_P016)):
        d = Direct(lib, settings, pix, w, h)
        assert d.rc == 0 and d.init.pix_fmt == pix, settings
        launches = core().hbcu_kernel_launches() if device else 0
        b = d.frame(pix, w, h, clip_of("nv12" if pix in (23, 0) else "p010le", w, h, 1, 3)[0], 0)
        st, outs = d.work(b)
        assert st == HB_FILTER_OK and outs == [b], "a pass-through hands on the buffer it was given"
        d.close_buffers(outs)
        eof = lib.hb_buffer_eof_init()
        st, outs = d.work(eof)
        assert st == HB_FILTER_DONE and outs == [eof]
        d.close_buffers(outs)
        d.close()
        if device:
            assert core().hbcu_kernel_launches() == launches
    for settings, pix in (("format=yuv420p10le", synth.PIX_FMT_P016), ("format=yuv420p10le", FORMATS["nv12"][0]),
                          ("format=nv12", 4),   # 4: yuv422p
                          ("format=nv12", FORMATS["yuv420p10le"][0]),
                          ("format=p016le", FORMATS["yuv420p"][0]), ("format=yuv444p", FORMATS["nv12"][0]),
                          ("format=no-such-format", FORMATS["nv12"][0])):
        d = Direct(lib, settings, pix, w, h)
        assert d.rc != 0 and d.init.pix_fmt == pix, settings
        d.close()


def test_passthrough_and_refusals_host_side():
    lib = semi_lib()
    check_passthrough_and_refusals(lib.lib)
    assert lib.buffers_alive() == 0


def check_props(lib, src, dst, hw_pix_fmt=-1):
    w, h, n = 33, 17, 5
    d = Direct(lib, f"format={dst}", FORMATS[src][0], w, h, hw_pix_fmt=hw_pix_fmt)
    assert d.rc == 0 and d.init.pix_fmt == FORMATS[dst][0]
    clip = clip_of(src, w, h, n, seed=4)
    got = []
    for t in range(n + 1):
        b = d.frame(FORMATS[src][0], w, h, clip[t], t) if t < n else lib.hb_buffer_eof_init()
        st, outs = d.work(b)
        assert st == (HB_FILTER_OK if t < n else HB_FILTER_DONE)
        got += outs
    assert len(got) == n + 1 and Buffer.from_address(got[-1]).s.flags & 0x400
    for t, b in enumerate(got[:-1]):
        buf = Buffer.from_address(b)
        assert (buf.s.start, buf.s.stop, buf.s.new_chap, buf.s.flags, buf.s.combed) == (3003 * t, 3003 * (t + 1), t + 10, 0x18, 1)
        assert (buf.f.fmt, buf.f.width, buf.f.height) == (FORMATS[dst][0], w, h)
        assert (buf.f.color_prim, buf.f.color_transfer, buf.f.color_matrix, buf.f.color_range, buf.f.chroma_location) == (9, 16, 9, 2, 2)
        assert buf.f.max_plane == (1 if FORMATS[dst][2] else 2)
        assert (buf.storage_type == HBCU_DEVICE) == (hw_pix_fmt == AV_PIX_FMT_CUDA)
    frames = [packed_of(b, lib) for b in got[:-1]] if hw_pix_fmt != AV_PIX_FMT_CUDA else None
    d.close_buffers(got)
    d.close()
    if frames is not None:
        assert all(np.array_equal(f, convert(clip[t], src, dst, w, h)) for t, f in enumerate(frames))
    return got


@pytest.mark.parametrize("src,dst", PAIRS)
def test_props_and_eof_host_side(src, dst):
    lib = semi_lib()
    check_props(lib.lib, src, dst)
    assert lib.buffers_alive() == 0


def test_restatement_reproduces_reference_chains(fref):
    """the reference calls of the chain tests, and the same chains behind the format filter over the restatement"""
    lib = semi_lib()
    r = nv12_chain_ref(fref)
    w, h, clip, flags = nv12_chain_inputs()
    g = lib.run([FMT] + product(NV12_CHAIN[0]), ["format=yuv420p"] + NV12_CHAIN[1], to_semi_clip(clip, 8, w, h), 23, w, h, flags=flags)
    assert np.array_equal(g.frames, r.frames) and list(g.combed) == list(r.combed)
    r = p010_chain_ref(fref)
    w, h, clip = p010_chain_inputs()
    g = lib.run([FMT] + product(P010_CHAIN[0]) + [FMT], ["format=yuv420p10le"] + P010_CHAIN[1] + ["format=p010le"],
                to_semi_clip(clip, 10, w, h), 158, w, h)
    assert np.array_equal(g.frames, to_semi_clip(r.frames, 10, w, h))
    assert lib.buffers_alive() == 0


# ------------------------------------------------------------------------------------------------- GPU tests
def core():
    lib = C.CDLL(str(LIBHBCU))
    lib.hbcu_frames_alive.restype = C.c_long
    lib.hbcu_last_error.restype = C.c_char_p
    lib.hbcu_kernel_launches.restype = C.c_uint64
    lib.hbcu_frame_plane.restype = C.c_void_p
    lib.hbcu_frame_plane.argtypes = [C.c_void_p, C.c_int]
    lib.hbcu_frame_release.argtypes = [C.c_void_p]
    return lib


class FormatConfig(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("depth", C.c_int), ("to_semi_planar", C.c_int),
                ("device", C.c_int), ("slots", C.c_int)]


def plane_shapes(fmt, w, h):
    """(row bytes, rows) of each plane of `fmt`; a semi-planar format's third plane is (0, 0)"""
    depth, semi = FORMATS[fmt][1], FORMATS[fmt][2]
    bps = 2 if depth > 8 else 1
    cw, ch = cdims(w, h)
    if semi:
        return [(w * bps, h), (2 * cw * bps, ch), (0, 0)]
    return [(w * bps, h), (cw * bps, ch), (cw * bps, ch)]


def split_packed(frame, shapes):
    out, off = [], 0
    for rb, rows in shapes:
        out.append(frame[off: off + rb * rows].reshape(rows, rb) if rows else None)
        off += rb * rows
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("src,dst", PAIRS)
@pytest.mark.parametrize("w,h", SIZES)
def test_exact_every_pair(cuda_filters, src, dst, w, h):
    """host frames, and device frames behind the upload adapter (the format filter's output stays a device frame)"""
    n = 2
    clip = clip_of(src, w, h, n, seed=2)
    want = np.stack([convert(f, src, dst, w, h) for f in clip])
    for chain in ([FMT], [UP, FMT, DOWN]):
        g = cuda_filters.run(chain, [f"format={dst}" if c == FMT else None for c in chain], clip, FORMATS[src][0], w, h)
        assert g.init_failed == 0 and g.saw_eof
        assert np.array_equal(g.frames, want), chain
        assert list(g.start) == [3003 * i for i in range(n)] and list(g.new_chap) == list(range(n))
    if src == "p010le":
        assert np.any(samples(clip, 10) & 0x3F), "the P010 input carries padding bits"
    assert core().hbcu_frames_alive() == 0 and cuda_filters.buffers_alive() == 0


@pytest.mark.gpu
@pytest.mark.parametrize("src,dst", PAIRS)
def test_c_abi_guard_bands_and_odd_linesizes(src, dst):
    """host planes inside guard bands, at linesizes that are neither even nor aligned, on both sides of the call"""
    lib = core()
    w, h = 333, 211
    frame = clip_of(src, w, h, 1, seed=6)[0]
    want = convert(frame, src, dst, w, h)
    cfg = FormatConfig(w, h, FORMATS[src][1], int(FORMATS[dst][2]), 0, 4)
    hd = C.c_void_p()
    assert lib.hbcu_format_create(C.byref(hd), C.byref(cfg)) == 0, lib.hbcu_last_error()
    GUARD, GB = 0xA5, 37
    keep, ins, outs = [], [], []
    for (rb, rows), pl in zip(plane_shapes(src, w, h), split_packed(frame, plane_shapes(src, w, h))):
        if rows == 0:
            ins.append((None, 0)); continue
        stride = rb + 13
        buf = np.full(GB * 2 + stride * rows, GUARD, np.uint8)
        view = buf[GB: GB + stride * rows].reshape(rows, stride)
        view[:, :rb] = pl
        keep.append(buf); ins.append((view.ctypes.data, stride))
    for rb, rows in plane_shapes(dst, w, h):
        if rows == 0:
            outs.append((None, 0, None, 0, 0)); continue
        stride = rb + 7
        buf = np.full(GB * 2 + stride * rows, GUARD, np.uint8)
        keep.append(buf); outs.append((buf.ctypes.data + GB, stride, buf, rb, rows))
    ip = (C.c_void_p * 3)(*[p for p, _ in ins]); ist = (C.c_int * 3)(*[s for _, s in ins])
    op = (C.c_void_p * 3)(*[o[0] for o in outs]); ost = (C.c_int * 3)(*[o[1] for o in outs])
    assert lib.hbcu_format_convert(hd, C.c_int64(0), None, ip, ist, None, op, ost) == 0, lib.hbcu_last_error()
    assert lib.hbcu_format_wait(hd, C.c_int64(0)) == 0
    got = []
    for _, stride, buf, rb, rows in outs:
        if buf is None:
            continue
        body = buf[GB: GB + stride * rows].reshape(rows, stride)
        got.append(body[:, :rb].ravel())
        assert np.all(body[:, rb:] == GUARD) and np.all(buf[:GB] == GUARD) and np.all(buf[GB + stride * rows:] == GUARD)
    assert np.array_equal(np.concatenate(got), want)
    lib.hbcu_format_destroy(hd)


def wrap_surface(lib, torch, packed, fmt, w, h, pitch, side, rel, opaque):
    """a torch-owned surface at a decoder pitch (chroma after the 16-aligned luma height), written on `side`, wrapped"""
    shapes = plane_shapes(fmt, w, h)
    hal = (h + 15) // 16 * 16
    surf = torch.zeros(pitch * (hal + 2 * hal) + 4096, dtype=torch.uint8, device="cuda")
    offs = [0, pitch * hal, pitch * (hal + hal // 2 + 8)]
    with torch.cuda.stream(side):
        for (rb, rows), pl, off in zip(shapes, split_packed(packed, shapes), offs):
            if rows:
                surf[off: off + rows * pitch].view(rows, pitch)[:, :rb].copy_(torch.from_numpy(np.ascontiguousarray(pl)))
    fr = C.c_void_p()
    dplanes = (C.c_void_p * 3)(*[surf.data_ptr() + off if rows else None for (rb, rows), off in zip(shapes, offs)])
    rb = (C.c_int * 3)(*[s[0] for s in shapes]); rows = (C.c_int * 3)(*[s[1] for s in shapes])
    st = (C.c_int * 3)(*[pitch if s[1] else 0 for s in shapes])
    assert lib.hbcu_frame_wrap(C.byref(fr), 0, dplanes, rb, rows, st, C.c_size_t(4096), C.c_void_p(side.cuda_stream), rel,
                               C.c_void_p(opaque)) == 0, lib.hbcu_last_error()
    return fr, surf


def pooled_frame(lib, fmt, w, h):
    shapes = plane_shapes(fmt, w, h)
    fr = C.c_void_p()
    rb = (C.c_int * 3)(*[s[0] for s in shapes]); rows = (C.c_int * 3)(*[s[1] for s in shapes])
    st = (C.c_int * 3)(*[(s[0] + 63) // 64 * 64 for s in shapes])
    assert lib.hbcu_frame_alloc(C.byref(fr), 0, rb, rows, st) == 0, lib.hbcu_last_error()
    return fr, st


def download(lib, fr, fmt, w, h, st):
    shapes = plane_shapes(fmt, w, h)
    x = C.c_void_p()
    assert lib.hbcu_xfer_create(C.byref(x), 0, 4) == 0
    bufs = [np.zeros((rows, st[p]), np.uint8) if rows else None for p, (rb, rows) in enumerate(shapes)]
    hp = (C.c_void_p * 3)(*[b.ctypes.data if b is not None else None for b in bufs])
    assert lib.hbcu_xfer_download(x, C.c_int64(0), fr, hp, st) == 0, lib.hbcu_last_error()
    assert lib.hbcu_xfer_wait(x, C.c_int64(0)) == 0
    lib.hbcu_xfer_destroy(x)
    return np.concatenate([b[:, :rb].ravel() for b, (rb, rows) in zip(bufs, shapes) if rows])


REL = C.CFUNCTYPE(None, C.c_void_p)


@pytest.mark.gpu
@pytest.mark.parametrize("src,dst", PAIRS)
def test_torch_surface_at_decoder_pitch(src, dst):
    """a torch-allocated surface at a 512-byte-aligned pitch, written on its own stream, wrapped at the C-ABI and
    converted into a pooled device frame; the surface is released once, when the kernel has read it"""
    import torch
    lib = core()
    w, h = 1280, 720
    frame = clip_of(src, w, h, 1, seed=8)[0]
    released = []
    rel = REL(lambda opaque: released.append(int(opaque or 0)))
    side = torch.cuda.Stream()
    pitch = (plane_shapes(src, w, h)[0][0] + 511) // 512 * 512 + 512
    fin, surf = wrap_surface(lib, torch, frame, src, w, h, pitch, side, rel, 7)
    cfg = FormatConfig(w, h, FORMATS[src][1], int(FORMATS[dst][2]), 0, 4)
    hd = C.c_void_p()
    assert lib.hbcu_format_create(C.byref(hd), C.byref(cfg)) == 0, lib.hbcu_last_error()
    fout, st = pooled_frame(lib, dst, w, h)
    assert lib.hbcu_format_convert(hd, C.c_int64(0), fin, None, None, fout, None, None) == 0, lib.hbcu_last_error()
    lib.hbcu_frame_release(fin)
    assert released == [7]
    assert np.array_equal(download(lib, fout, dst, w, h, st), convert(frame, src, dst, w, h))
    lib.hbcu_frame_release(fout)
    lib.hbcu_format_destroy(hd)
    del surf
    assert lib.hbcu_frames_alive() == 0


@pytest.mark.gpu
@pytest.mark.parametrize("src,dst", PAIRS)
def test_host_input_device_output(cuda_filters, src, dst):
    """hw_pix_fmt = AV_PIX_FMT_CUDA: host frames in, device frames out, props and colour fields carried"""
    lib = core()
    w, h, n = 33, 17, 5
    got = check_props(cuda_filters.lib, src, dst, hw_pix_fmt=AV_PIX_FMT_CUDA)
    assert len(got) == n + 1 and lib.hbcu_frames_alive() == 0 and cuda_filters.buffers_alive() == 0
    # the content of such an output, downloaded by the adapter
    clip = clip_of(src, w, h, n, seed=4)
    g = cuda_filters.run([FMT, DOWN], [f"format={dst}", None], clip, FORMATS[src][0], w, h)
    assert np.array_equal(g.frames, np.stack([convert(f, src, dst, w, h) for f in clip]))


@pytest.mark.gpu
@pytest.mark.parametrize("depth", [8, 10])
@pytest.mark.parametrize("device", [False, True])
def test_round_trip_is_identity(cuda_filters, depth, device):
    w, h = 1921, 1081
    planar, semi = ("yuv420p", "nv12") if depth == 8 else ("yuv420p10le", "p010le")
    clip = clip_of(planar, w, h, 3, seed=5)
    chain = [FMT, FMT] if not device else [UP, FMT, FMT, DOWN]
    sets = [f"format={semi}", f"format={planar}"] if not device else [None, f"format={semi}", f"format={planar}", None]
    g = cuda_filters.run(chain, sets, clip, FORMATS[planar][0], w, h)
    assert np.array_equal(g.frames, clip)
    assert core().hbcu_frames_alive() == 0 and cuda_filters.buffers_alive() == 0


@pytest.mark.gpu
def test_passthrough_and_refusals(cuda_filters):
    check_passthrough_and_refusals(cuda_filters.lib, device=True)
    assert core().hbcu_frames_alive() == 0 and cuda_filters.buffers_alive() == 0


@pytest.mark.gpu
def test_nv12_surfaces_chain_matches_reference(fref, cuda_filters, monkeypatch):
    """wrapped NV12 surfaces (the upload adapter playing NVDEC) -> format=yuv420p -> comb-detect -> decomb -> NLMeans ->
    download: the reference's planar chain on the de-interleaved input"""
    r = nv12_chain_ref(fref)
    w, h, clip, flags = nv12_chain_inputs()
    monkeypatch.setenv("HBCU_UPLOAD_EXTERNAL", "1")
    cuda_filters.lib.hbcu_test_surfaces_returned.restype = C.c_long
    before = cuda_filters.lib.hbcu_test_surfaces_returned()
    g = cuda_filters.run([UP, FMT] + product(NV12_CHAIN[0]) + [DOWN], [None, "format=yuv420p"] + NV12_CHAIN[1] + [None],
                         to_semi_clip(clip, 8, w, h), 23, w, h, flags=flags)
    assert g.init_failed == 0 and np.array_equal(g.frames, r.frames) and list(g.combed) == list(r.combed)
    assert cuda_filters.lib.hbcu_test_surfaces_returned() - before == len(clip)
    assert core().hbcu_frames_alive() == 0 and cuda_filters.buffers_alive() == 0


@pytest.mark.gpu
def test_p010_surfaces_chain_matches_reference(fref, cuda_filters, monkeypatch):
    """wrapped P010 surfaces -> format=yuv420p10le -> NLMeans -> format=p010le -> download: the reference's NLMeans on the
    de-interleaved input, shifted back and interleaved"""
    r = p010_chain_ref(fref)
    w, h, clip = p010_chain_inputs()
    monkeypatch.setenv("HBCU_UPLOAD_EXTERNAL", "1")
    g = cuda_filters.run([UP, FMT] + product(P010_CHAIN[0]) + [FMT, DOWN],
                         [None, "format=yuv420p10le"] + P010_CHAIN[1] + ["format=p010le", None],
                         to_semi_clip(clip, 10, w, h), 158, w, h)
    assert g.init_failed == 0 and np.array_equal(g.frames, to_semi_clip(r.frames, 10, w, h))
    assert core().hbcu_frames_alive() == 0 and cuda_filters.buffers_alive() == 0


class NlmPlane(C.Structure):
    _fields_ = [("patch_size", C.c_int), ("range", C.c_int), ("nframes", C.c_int), ("bypass", C.c_int),
                ("origin_tune", C.c_double), ("weight_fact", C.c_float), ("diff_max", C.c_int),
                ("exptable", C.c_float * 128), ("prefilter", C.c_int)]


class NlmConfig(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("depth", C.c_int), ("chroma_shift_w", C.c_int),
                ("chroma_shift_h", C.c_int), ("device", C.c_int), ("ring_frames", C.c_int), ("out_slots", C.c_int),
                ("plane", NlmPlane * 3)]


@pytest.mark.gpu
def test_surfaces_return_before_the_nlmeans_window_moves_on(cuda_filters):
    """wrapped NV12 surfaces -> format -> NLMeans frame-count=4 at the C-ABI: a surface goes back to its owner once the
    conversion has read it, so no more than the format filter's in-flight bound are ever out, while NLMeans holds 4
    frames; the denoised frames equal those of planar host input"""
    import torch
    lib = core()
    flt = cuda_filters.lib
    w, h, n = 640, 360, 10
    bound = 4                   # FORMAT_INFLIGHT of format_cuda.c
    planar = synth.progressive_clip(synth.PIX_FMT_YUV420P, w, h, n, seed=12)
    semi = to_semi_clip(planar, 8, w, h)
    cfg = NlmConfig()
    flt.hb_parse_filter_settings.restype = C.c_void_p
    flt.hb_parse_filter_settings.argtypes = [C.c_char_p]
    flt.hb_nlmeans_cuda_build_config.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(NlmConfig), C.c_void_p, C.c_void_p, C.c_void_p]
    assert flt.hb_nlmeans_cuda_build_config(flt.hb_parse_filter_settings(b"y-strength=6:frame-count=4"), 0, w, h,
                                            C.byref(cfg), None, None, None) == 0
    cfg.device, cfg.ring_frames, cfg.out_slots = 0, 12, 4
    fcfg = FormatConfig(w, h, 8, 0, 0, 6)
    nl, fm = C.c_void_p(), C.c_void_p()
    assert lib.hbcu_nlmeans_create(C.byref(nl), C.byref(cfg)) == 0, lib.hbcu_last_error()
    assert lib.hbcu_format_create(C.byref(fm), C.byref(fcfg)) == 0, lib.hbcu_last_error()
    released, wrapped, keep, most_out = [], 0, [], 0
    rel = REL(lambda opaque: released.append(int(opaque or 0)))
    side = torch.cuda.Stream()
    pitch = 1024
    outs = []
    for t in range(n):
        fin, surf = wrap_surface(lib, torch, semi[t], "nv12", w, h, pitch, side, rel, t + 1)
        keep.append(surf)
        wrapped += 1
        fpl, st = pooled_frame(lib, "yuv420p", w, h)
        assert lib.hbcu_format_convert(fm, C.c_int64(t), fin, None, None, fpl, None, None) == 0, lib.hbcu_last_error()
        lib.hbcu_frame_release(fin)                      # what format_cuda.c does once the conversion is queued
        assert lib.hbcu_nlmeans_upload_frame(nl, C.c_int64(t), fpl) == 0, lib.hbcu_last_error()
        lib.hbcu_frame_release(fpl)
        most_out = max(most_out, wrapped - len(released))
        if t >= 3:
            k = t - 3
            dims = synth.plane_dims(w, h)
            o = [np.zeros((ph, pw), np.uint8) for pw, ph in dims]
            ptrs = (C.c_void_p * 3)(*[a.ctypes.data for a in o]); ost = (C.c_int * 3)(*[pw for pw, _ in dims])
            assert lib.hbcu_nlmeans_filter(nl, C.c_int64(k), 4, ptrs, ost) == 0, lib.hbcu_last_error()
            assert lib.hbcu_nlmeans_wait(nl, C.c_int64(k)) == 0
            outs.append(np.concatenate([a.ravel() for a in o]))
    assert most_out <= bound and sorted(released) == list(range(1, n + 1))
    lib.hbcu_format_destroy(fm)
    lib.hbcu_nlmeans_destroy(nl)
    # the same frames from planar host input through the filter
    want = cuda_filters.run("hb_filter_nlmeans_cuda", "y-strength=6:frame-count=4", planar, 0, w, h)
    assert np.array_equal(np.stack(outs), want.frames[: len(outs)])
    assert lib.hbcu_frames_alive() == 0
