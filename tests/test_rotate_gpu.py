"""hb_filter_rotate_cuda: rotations by 90, 180 and 270 degrees and mirrors on the GPU (handbrake_b200/csrc/rotate.cu), the
drop-in for libhb's rotate filter (rotate.c), and the decoder's auto-rotation done with it.

Expected values are computed here in numpy, plane by plane: np.rot90 / flips of the plane arrays, with a semi-planar
chroma plane viewed as one uint16 (NV12) or uint32 (P010, P016) per Cb/Cr pair, so that a pair moves as one unit.
Chains that run other filters behind the rotation are compared with the reference's filters on the numpy-rotated input,
whose results are stored in tests/golden/rotate_chain_ref_digests.json (`HBCU_RECORD_REF=1` with the reference built
records them through the CPU tests, which make every reference call the GPU tests make).

CPU tests run the host side of the filter (init, geometry and PAR, pass-through, refusals, props, EOF, buffer ownership)
over the plain-C restatement of the transforms in oracle/_ref/libhostlogic_rotate.so (oracle/rotate.mk)."""
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
from test_format_gpu import (AV_PIX_FMT_CUDA, CLOSE_FN, HB_FILTER_DONE, HB_FILTER_OK, HBCU_DEVICE, INIT_FN, REL, WORK_FN,
                             Buffer, FilterInit, FilterObject, NlmConfig, clear_next)

STORE = Path(__file__).resolve().parent / "golden" / "rotate_chain_ref_digests.json"
HOSTLOGIC_ROTATE_SO = REPO / "oracle" / "_ref" / "libhostlogic_rotate.so"
UP, DOWN = "hb_filter_hbcu_upload", "hb_filter_hbcu_download"
ROT, FMT = "hb_filter_rotate_cuda", "hb_filter_format_cuda"

# name -> (pix_fmt, log2 chroma w, log2 chroma h, luma element bytes, chroma element bytes, semi-planar, depth)
FORMATS = {
    "yuv420p": (0, 1, 1, 1, 1, False, 8), "yuv420p10le": (62, 1, 1, 2, 2, False, 10),
    "yuv420p12le": (123, 1, 1, 2, 2, False, 12), "yuv420p16le": (47, 1, 1, 2, 2, False, 16),
    "yuv444p": (5, 0, 0, 1, 1, False, 8), "yuv444p10le": (68, 0, 0, 2, 2, False, 10),
    "yuv422p": (4, 1, 0, 1, 1, False, 8),
    "nv12": (23, 1, 1, 1, 2, True, 8), "p010le": (158, 1, 1, 2, 4, True, 10), "p016le": (169, 1, 1, 2, 4, True, 16),
}
# settings -> (transform, the numpy restatement of one plane array, swaps the geometry)
TRANSFORMS = {
    "angle=0:hflip=1":   (1, lambda a: a[:, ::-1], False),
    "angle=180:hflip=1": (2, lambda a: a[::-1], False),
    "angle=180:hflip=0": (3, lambda a: a[::-1, ::-1], False),
    "angle=90:hflip=0":  (4, lambda a: np.rot90(a, -1), True),
    "angle=90:hflip=1":  (5, lambda a: a[::-1, ::-1].T, True),
    "angle=270:hflip=0": (6, lambda a: np.rot90(a, 1), True),
    "angle=270:hflip=1": (7, lambda a: a.T, True),
}
FLIPS = [s for s, t in TRANSFORMS.items() if not t[2]]
# the decoder's auto-rotation (decavcodec.c): title->rotation -> the graph it builds, as the rotate filter's settings
DECODER_ROTATIONS = {90: "angle=270:hflip=0", 180: "angle=180:hflip=0", 270: "angle=90:hflip=0"}


# ------------------------------------------------------------------------------------------------- numpy restatement
def plane_shapes(fmt, w, h):
    """(elements per row, rows, element bytes) of each plane; a semi-planar format has two"""
    _, sw, sh, el, ec, semi, _ = FORMATS[fmt]
    cw, ch = -((-w) >> sw), -((-h) >> sh)
    return [(w, h, el), (cw, ch, ec)] + ([] if semi else [(cw, ch, ec)])


def frame_bytes(fmt, w, h):
    return sum(pw * ph * e for pw, ph, e in plane_shapes(fmt, w, h))


def out_dims(settings, w, h):
    return (h, w) if TRANSFORMS[settings][2] else (w, h)


def elem_view(raw, pw, ph, e):
    return raw.view({1: np.uint8, 2: np.uint16, 4: np.uint32}[e]).reshape(ph, pw)


def rotate_frame(frame, fmt, w, h, settings):
    """one packed frame (planes back to back, rows at their widths) through the transform, packed again"""
    fn = TRANSFORMS[settings][1]
    out, off = [], 0
    frame = np.ascontiguousarray(frame)
    for pw, ph, e in plane_shapes(fmt, w, h):
        out.append(np.ascontiguousarray(fn(elem_view(frame[off: off + pw * ph * e], pw, ph, e))).view(np.uint8).ravel())
        off += pw * ph * e
    return np.concatenate(out)


def rotate_clip(clip, fmt, w, h, settings):
    return np.stack([rotate_frame(f, fmt, w, h, settings) for f in clip])


def clip_of(fmt, w, h, n, seed):
    """random frames of `fmt`; every bit of a sample may be set (the rotation moves samples, it never reads them)"""
    rng = np.random.default_rng(seed + 7 * w + h)
    return rng.integers(0, 256, (n, frame_bytes(fmt, w, h)), dtype=np.uint8)


# ------------------------------------------------------------------------------------------------- direct calls
class Direct:
    """one hb_filter_rotate_cuda instance driven by hand: init / work / close as libhb calls them"""

    def __init__(self, lib, settings, pix_fmt, w, h, hw_pix_fmt=-1, par=(1, 1)):
        self.lib = lib
        lib.hb_parse_filter_settings.restype = C.c_void_p
        lib.hb_parse_filter_settings.argtypes = [C.c_char_p]
        lib.hb_harness_frame_from_packed.restype = C.c_void_p
        lib.hb_harness_frame_from_packed.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p]
        lib.hb_buffer_close.argtypes = [C.POINTER(C.c_void_p)]
        lib.hb_buffer_eof_init.restype = C.c_void_p
        self.obj = FilterObject.from_buffer_copy(FilterObject.in_dll(lib, ROT))
        self.obj.settings = lib.hb_parse_filter_settings(settings.encode()) if settings else None
        self.init = FilterInit(pix_fmt=pix_fmt, hw_pix_fmt=hw_pix_fmt, color_prim=5, color_transfer=6, color_matrix=7,
                               color_range=2, chroma_location=3, width=w, height=h, par_num=par[0], par_den=par[1])
        self.rc = INIT_FN(self.obj.init)(C.addressof(self.obj), C.addressof(self.init))

    def has_handle(self):
        """hb_filter_private_t.gpu, its first field"""
        return C.c_void_p.from_address(self.obj.private_data).value is not None

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


def packed_of(buf_addr, lib):
    b = Buffer.from_address(buf_addr)
    name = next(n for n, f in FORMATS.items() if f[0] == b.f.fmt)
    out = np.zeros(frame_bytes(name, b.f.width, b.f.height), np.uint8)
    lib.hb_harness_frame_to_packed.argtypes = [C.c_void_p, C.c_void_p]
    lib.hb_harness_frame_to_packed(buf_addr, out.ctypes.data)
    return out


# ------------------------------------------------------------------------------------------------- the reference
class RotateRef(GoldenRef):
    """GoldenRef over this file's store: the reference's filters on the numpy-rotated inputs, and the digest of
    rotate.c's settings template"""

    def __init__(self):
        super().__init__()
        self.store = json.loads(STORE.read_text()) if STORE.exists() else {}

    def _save(self):
        STORE.write_text(json.dumps(dict(sorted(self.store.items())), indent=0) + "\n")

    def template_digest(self):
        if self.recording:
            tree = Path(os.environ["HANDBRAKE_SRC"])      # the HandBrake tree the reference was built from
            common = (tree / "libhb" / "handbrake" / "common.h").read_text()
            rot_c = (tree / "libhb" / "rotate.c").read_text()
            bool_reg = re.search(r'#define\s+HB_BOOL_REG\s+"((?:[^"\\]|\\.)*)"', common).group(1)
            body = re.search(r"rotate_template\[\]\s*=\s*((?:\s*(?:\"(?:[^\"\\]|\\.)*\"|HB_BOOL_REG))+)\s*;", rot_c).group(1)
            parts = re.findall(r'"((?:[^"\\]|\\.)*)"|(HB_BOOL_REG)', body)
            template = "".join(bool_reg if macro else lit for lit, macro in parts)
            self.store["rotate_template"] = _h(template)
            self._save()
        return self.store["rotate_template"]


@pytest.fixture(scope="module")
def rref():
    return RotateRef()


# rotate -> NLMeans -> lapsharp, against the reference's NLMeans -> lapsharp on the numpy-rotated input
CHAIN = (["hb_filter_nlmeans", "hb_filter_lapsharp"], ["y-strength=6:cb-strength=4", "y-strength=0.2:y-kernel=isolap"])
CHAIN_CASES = [("yuv420p", 96, 64, "angle=90:hflip=0"), ("yuv420p10le", 80, 48, "angle=270:hflip=1")]
# wrapped NV12 surfaces -> rotate angle=90 -> format yuv420p -> NLMeans
NV12_CHAIN = (["hb_filter_nlmeans"], ["y-strength=6:frame-count=3"])


def chain_inputs(fmt, w, h):
    return synth.progressive_clip(FORMATS[fmt][0], w, h, 5, seed=31)


def chain_ref(rref, fmt, w, h, settings):
    clip = chain_inputs(fmt, w, h)
    ow, oh = out_dims(settings, w, h)
    return rref.run(*CHAIN, rotate_clip(clip, fmt, w, h, settings), FORMATS[fmt][0], ow, oh)


def nv12_chain_inputs():
    w, h = 192, 112
    return w, h, synth.progressive_clip(synth.PIX_FMT_YUV420P, w, h, 6, seed=37)


def to_nv12(planar, w, h):
    """yuv420p frames as NV12 (Cb/Cr interleaved)"""
    cw, ch = (w + 1) // 2, (h + 1) // 2
    out = []
    for f in planar:
        u, v = f[w * h: w * h + cw * ch].reshape(ch, cw), f[w * h + cw * ch:].reshape(ch, cw)
        uv = np.empty((ch, 2 * cw), np.uint8)
        uv[:, 0::2], uv[:, 1::2] = u, v
        out.append(np.concatenate([f[: w * h], uv.ravel()]))
    return np.stack(out)


def nv12_chain_ref(rref):
    w, h, clip = nv12_chain_inputs()
    return rref.run(*NV12_CHAIN, rotate_clip(clip, "yuv420p", w, h, "angle=90:hflip=0"), synth.PIX_FMT_YUV420P, h, w)


def product(names):
    return [n + "_cuda" for n in names]


# ------------------------------------------------------------------------------------------------- CPU tests
def host_lib():
    return FilterLib(HOSTLOGIC_ROTATE_SO)


def test_identity_fields_and_template(rref):
    lib = host_lib().lib
    obj = FilterObject.in_dll(lib, ROT)
    assert (obj.id, obj.short_name, obj.skip, obj.enforce_order) == (19, b"rotate", 0, 1)
    assert obj.settings_template == b"angle=^(0|90|180|270)$:hflip=^(yes|no|true|false|[01])$:disable=^(yes|no|true|false|[01])$"
    assert _h(obj.settings_template.decode()) == rref.template_digest()
    import handbrake_b200
    flt = handbrake_b200.filters()
    flt.lib.hb_filter_get.restype = C.c_void_p
    assert flt.lib.hb_filter_get(19) == flt.filter_object(ROT)      # HB_FILTER_ROTATE


@pytest.mark.parametrize("w,h", [(33, 17), (64, 36)])
@pytest.mark.parametrize("settings", ["angle=0:hflip=0"] + list(TRANSFORMS))
def test_geometry_and_par_after_init(settings, w, h):
    """rotate_init: 90 and 270 swap the width and height and the PAR's terms, the others keep them"""
    lib = host_lib()
    swap = settings in TRANSFORMS and TRANSFORMS[settings][2]
    clip = clip_of("yuv420p", w, h, 1, seed=3)
    r = lib.run([ROT], [settings], clip, 0, w, h, par=(8, 9))
    assert r.init_failed == 0
    assert (r.width, r.height, r.par) == ((h, w, (9, 8)) if swap else (w, h, (8, 9)))
    d = Direct(lib.lib, settings, 0, w, h, par=(8, 9))
    assert d.rc == 0 and (d.init.width, d.init.height, d.init.par_num, d.init.par_den) == ((h, w, 9, 8) if swap else (w, h, 8, 9))
    d.close()
    assert lib.buffers_alive() == 0


def check_passthrough_and_refusals(lib, device=False, launches=None):
    w, h = 64, 48
    for settings in ("angle=0:hflip=0", "angle=0", None, "angle=45:hflip=1", "angle=45"):
        d = Direct(lib, settings, 0, w, h, par=(4, 3))
        assert d.rc == 0 and not d.has_handle(), settings
        assert (d.init.width, d.init.height, d.init.par_num, d.init.par_den) == (w, h, 4, 3)
        before = launches() if launches else 0
        b = d.frame(0, w, h, clip_of("yuv420p", w, h, 1, 3)[0], 0)
        st, outs = d.work(b)
        assert st == HB_FILTER_OK and outs == [b], "a pass-through hands on the buffer it was given"
        d.close_buffers(outs)
        eof = lib.hb_buffer_eof_init()
        st, outs = d.work(eof)
        assert st == HB_FILTER_DONE and outs == [eof]
        d.close_buffers(outs)
        d.close()
        if launches:
            assert launches() == before
    refused = [(s, pix) for s in ("angle=90:hflip=0", "angle=270:hflip=1") for pix in (4, 64)]      # yuv422p, yuv422p10le
    refused += [("angle=0:hflip=1", 8), ("angle=90", 8),                                            # gray: one plane
                ("angle=180", 33), ("angle=0:hflip=1", 9999)]                                       # yuva420p, unknown
    for settings, pix in refused:
        d = Direct(lib, settings, pix, w, h)
        assert d.rc != 0, (settings, pix)
        assert (d.init.width, d.init.height) == (w, h)
        d.close()
    for settings in FLIPS:                                                                          # 4:2:2 flips are taken
        d = Direct(lib, settings, 4, w, h)
        assert d.rc == 0 and d.has_handle(), settings
        d.close()


def test_passthrough_and_refusals_host_side():
    lib = host_lib()
    check_passthrough_and_refusals(lib.lib)
    assert lib.buffers_alive() == 0


def check_props(lib, fmt, settings, hw_pix_fmt=-1):
    w, h, n = 33, 17, 5
    pix = FORMATS[fmt][0]
    d = Direct(lib, settings, pix, w, h, hw_pix_fmt=hw_pix_fmt)
    assert d.rc == 0
    ow, oh = out_dims(settings, w, h)
    clip = clip_of(fmt, w, h, n, seed=4)
    got = []
    for t in range(n + 1):
        b = d.frame(pix, w, h, clip[t], t) if t < n else lib.hb_buffer_eof_init()
        st, outs = d.work(b)
        assert st == (HB_FILTER_OK if t < n else HB_FILTER_DONE)
        got += outs
    assert len(got) == n + 1 and Buffer.from_address(got[-1]).s.flags & 0x400
    for t, b in enumerate(got[:-1]):
        buf = Buffer.from_address(b)
        assert (buf.s.start, buf.s.stop, buf.s.new_chap, buf.s.flags, buf.s.combed) == (3003 * t, 3003 * (t + 1), t + 10, 0x18, 1)
        assert (buf.f.fmt, buf.f.width, buf.f.height) == (pix, ow, oh)
        assert (buf.f.color_prim, buf.f.color_transfer, buf.f.color_matrix, buf.f.color_range, buf.f.chroma_location) == (9, 16, 9, 2, 2)
        assert (buf.storage_type == HBCU_DEVICE) == (hw_pix_fmt == AV_PIX_FMT_CUDA)
    frames = [packed_of(b, lib) for b in got[:-1]] if hw_pix_fmt != AV_PIX_FMT_CUDA else None
    d.close_buffers(got)
    d.close()
    if frames is not None:
        assert all(np.array_equal(f, rotate_frame(clip[t], fmt, w, h, settings)) for t, f in enumerate(frames))
    return got


@pytest.mark.parametrize("fmt,settings", [("yuv420p", "angle=90:hflip=0"), ("nv12", "angle=0:hflip=1"),
                                          ("p010le", "angle=270:hflip=1"), ("yuv420p10le", "angle=180:hflip=0")])
def test_props_and_eof_host_side(fmt, settings):
    lib = host_lib()
    check_props(lib.lib, fmt, settings)
    assert lib.buffers_alive() == 0


@pytest.mark.parametrize("fmt", list(FORMATS))
@pytest.mark.parametrize("w,h", [(1, 1), (2, 3), (33, 17), (17, 33)])
def test_restatement_matches_numpy(fmt, w, h):
    """the filter over the restatement, on host frames and on device-frame stand-ins"""
    lib = host_lib()
    clip = clip_of(fmt, w, h, 2, seed=1)
    for settings in (FLIPS if fmt == "yuv422p" else TRANSFORMS):
        want = rotate_clip(clip, fmt, w, h, settings)
        for chain in ([ROT], [UP, ROT, DOWN]):
            r = lib.run(chain, [settings if c == ROT else None for c in chain], clip, FORMATS[fmt][0], w, h)
            assert r.init_failed == 0 and r.saw_eof and np.array_equal(r.frames, want), (settings, chain)
            assert (r.width, r.height) == out_dims(settings, w, h)
            assert list(r.start) == [0, 3003] and list(r.new_chap) == [0, 1]
    assert lib.buffers_alive() == 0


def test_restatement_reproduces_reference_chains(rref):
    """every reference call of the chain tests, and the same chains behind the rotate filter over the restatement: the
    next filter sees the new geometry"""
    lib = host_lib()
    for fmt, w, h, settings in CHAIN_CASES:
        r = chain_ref(rref, fmt, w, h, settings)
        g = lib.run([ROT] + product(CHAIN[0]), [settings] + CHAIN[1], chain_inputs(fmt, w, h), FORMATS[fmt][0], w, h)
        assert g.init_failed == 0 and np.array_equal(g.frames, r.frames), (fmt, settings)
    r = nv12_chain_ref(rref)
    w, h, clip = nv12_chain_inputs()
    g = lib.run([ROT, FMT] + product(NV12_CHAIN[0]), ["angle=90:hflip=0", "format=yuv420p"] + NV12_CHAIN[1],
                to_nv12(clip, w, h), 23, w, h)
    assert g.init_failed == 0 and np.array_equal(g.frames, r.frames)
    assert lib.buffers_alive() == 0


# ------------------------------------------------------------------------------------------------- GPU tests
def core():
    lib = C.CDLL(str(LIBHBCU))
    lib.hbcu_frames_alive.restype = C.c_long
    lib.hbcu_last_error.restype = C.c_char_p
    lib.hbcu_kernel_launches.restype = C.c_uint64
    lib.hbcu_frame_release.argtypes = [C.c_void_p]
    return lib


class RotateConfig(C.Structure):
    _fields_ = [("planes", C.c_int), ("width", C.c_int * 3), ("height", C.c_int * 3), ("elem_bytes", C.c_int * 3),
                ("transform", C.c_int), ("device", C.c_int), ("slots", C.c_int)]


def config_of(fmt, w, h, settings):
    shapes = plane_shapes(fmt, w, h)
    pad = [(0, 0, 0)] * (3 - len(shapes))
    return RotateConfig(len(shapes), (C.c_int * 3)(*[s[0] for s in shapes + pad]), (C.c_int * 3)(*[s[1] for s in shapes + pad]),
                        (C.c_int * 3)(*[s[2] for s in shapes + pad]), TRANSFORMS[settings][0], 0, 4)


def byte_shapes(fmt, w, h):
    """(row bytes, rows) of the three planes; a semi-planar format's third is (0, 0)"""
    s = [(pw * e, ph) for pw, ph, e in plane_shapes(fmt, w, h)]
    return s + [(0, 0)] * (3 - len(s))


def split_packed(frame, shapes):
    out, off = [], 0
    for rb, rows in shapes:
        out.append(frame[off: off + rb * rows].reshape(rows, rb) if rows else None)
        off += rb * rows
    return out


EDGE_SIZES = [(1, 1), (2, 2), (1, 77), (77, 1), (33, 17), (17, 33), (127, 63), (128, 64), (129, 65), (63, 129),
              (64, 128), (65, 127), (31, 33), (257, 130)]
FULL = [(1920, 1080), (3840, 2160)]


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", list(FORMATS))
@pytest.mark.parametrize("w,h", EDGE_SIZES + FULL)
def test_exact_every_transform(cuda_filters, fmt, w, h):
    """host frames, and device frames behind the upload adapter (the rotate filter's output stays a device frame);
    full-size frames on yuv420p, yuv420p10le, NV12 and P010"""
    if (w, h) in FULL and fmt not in ("yuv420p", "yuv420p10le", "nv12", "p010le"):
        pytest.skip("full-size frames run on the four formats of a hardware-decoded job")
    n = 1 if (w, h) in FULL else 2
    clip = clip_of(fmt, w, h, n, seed=2)
    for settings in (FLIPS if fmt == "yuv422p" else TRANSFORMS):
        want = rotate_clip(clip, fmt, w, h, settings)
        for chain in ([ROT], [UP, ROT, DOWN]):
            g = cuda_filters.run(chain, [settings if c == ROT else None for c in chain], clip, FORMATS[fmt][0], w, h)
            assert g.init_failed == 0 and g.saw_eof and (g.width, g.height) == out_dims(settings, w, h)
            assert np.array_equal(g.frames, want), (settings, chain)
            assert list(g.start) == [3003 * i for i in range(n)]
    assert core().hbcu_frames_alive() == 0 and cuda_filters.buffers_alive() == 0


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["yuv420p", "yuv420p10le", "nv12", "p010le"])
@pytest.mark.parametrize("settings", list(TRANSFORMS))
def test_c_abi_guard_bands_and_odd_linesizes(fmt, settings):
    """host planes inside guard bands, at linesizes that are neither even nor aligned, on both sides of the call"""
    lib = core()
    w, h = 333, 211
    ow, oh = out_dims(settings, w, h)
    frame = clip_of(fmt, w, h, 1, seed=6)[0]
    want = rotate_frame(frame, fmt, w, h, settings)
    cfg = config_of(fmt, w, h, settings)
    hd = C.c_void_p()
    assert lib.hbcu_rotate_create(C.byref(hd), C.byref(cfg)) == 0, lib.hbcu_last_error()
    GUARD, GB = 0xA5, 37
    keep, ins, outs = [], [], []
    for (rb, rows), pl in zip(byte_shapes(fmt, w, h), split_packed(frame, byte_shapes(fmt, w, h))):
        if rows == 0:
            ins.append((None, 0)); continue
        stride = rb + 13
        buf = np.full(GB * 2 + stride * rows, GUARD, np.uint8)
        view = buf[GB: GB + stride * rows].reshape(rows, stride)
        view[:, :rb] = pl
        keep.append(buf); ins.append((view.ctypes.data, stride))
    for rb, rows in byte_shapes(fmt, ow, oh):
        if rows == 0:
            outs.append((None, 0, None, 0, 0)); continue
        stride = rb + 7
        buf = np.full(GB * 2 + stride * rows, GUARD, np.uint8)
        keep.append(buf); outs.append((buf.ctypes.data + GB, stride, buf, rb, rows))
    ip = (C.c_void_p * 3)(*[p for p, _ in ins]); ist = (C.c_int * 3)(*[s for _, s in ins])
    op = (C.c_void_p * 3)(*[o[0] for o in outs]); ost = (C.c_int * 3)(*[o[1] for o in outs])
    assert lib.hbcu_rotate_frame(hd, C.c_int64(0), None, ip, ist, None, op, ost) == 0, lib.hbcu_last_error()
    assert lib.hbcu_rotate_wait(hd, C.c_int64(0)) == 0
    got = []
    for _, stride, buf, rb, rows in outs:
        if buf is None:
            continue
        body = buf[GB: GB + stride * rows].reshape(rows, stride)
        got.append(body[:, :rb].ravel())
        assert np.all(body[:, rb:] == GUARD) and np.all(buf[:GB] == GUARD) and np.all(buf[GB + stride * rows:] == GUARD)
    assert np.array_equal(np.concatenate(got), want)
    lib.hbcu_rotate_destroy(hd)


def wrap_torch(lib, torch, fmt, w, h, pitch, fill, side=None, packed=None, rel=None, opaque=0):
    """a torch-owned surface at `pitch` (chroma after the 16-aligned luma height) filled with `fill`, the planes of
    `packed` written into it on `side`, wrapped as a device frame"""
    shapes = byte_shapes(fmt, w, h)
    hal = (h + 15) // 16 * 16
    surf = torch.full((pitch * (hal + 2 * hal) + 4096,), fill, dtype=torch.uint8, device="cuda")
    offs = [0, pitch * hal, pitch * (hal + hal // 2 + 8)]
    if packed is not None:
        with torch.cuda.stream(side):
            for (rb, rows), pl, off in zip(shapes, split_packed(packed, shapes), offs):
                if rows:
                    surf[off: off + rows * pitch].view(rows, pitch)[:, :rb].copy_(torch.from_numpy(np.ascontiguousarray(pl)))
    fr = C.c_void_p()
    dplanes = (C.c_void_p * 3)(*[surf.data_ptr() + off if rows else None for (rb, rows), off in zip(shapes, offs)])
    rb = (C.c_int * 3)(*[s[0] for s in shapes]); rows = (C.c_int * 3)(*[s[1] for s in shapes])
    st = (C.c_int * 3)(*[pitch if s[1] else 0 for s in shapes])
    stream = C.c_void_p(side.cuda_stream) if side is not None else None
    assert lib.hbcu_frame_wrap(C.byref(fr), 0, dplanes, rb, rows, st, C.c_size_t(4096), stream,
                               rel, C.c_void_p(opaque)) == 0, lib.hbcu_last_error()
    return fr, surf, offs


def surface_planes(surf, offs, fmt, w, h, pitch):
    """the packed planes of a surface, and every byte of its rows past the planes' row bytes"""
    host = surf.cpu().numpy()
    planes, tails = [], []
    for (rb, rows), off in zip(byte_shapes(fmt, w, h), offs):
        if rows:
            body = host[off: off + rows * pitch].reshape(rows, pitch)
            planes.append(body[:, :rb].ravel())
            tails.append(body[:, rb:].ravel())
    return np.concatenate(planes), np.concatenate(tails)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["nv12", "p010le"])
@pytest.mark.parametrize("rotation", [90, 180, 270])
def test_decoder_rotation_on_torch_surfaces(fmt, rotation):
    """decoder auto-rotation: a torch-allocated surface at a 512-byte-aligned pitch, written on its own stream, wrapped
    and rotated into another wrapped surface; the input surface is released once the kernel has read it, the output
    rows' pitch bytes stay at their sentinel"""
    import torch
    lib = core()
    w, h = 1280, 720
    settings = DECODER_ROTATIONS[rotation]
    ow, oh = out_dims(settings, w, h)
    frame = clip_of(fmt, w, h, 1, seed=8)[0]
    # the decoder's graph (decavcodec.c): 90 -> transpose=cclock, 180 -> hflip, vflip, 270 -> transpose=clock
    graph = {90: lambda a: np.rot90(a, 1), 180: lambda a: a[:, ::-1][::-1], 270: lambda a: np.rot90(a, -1)}[rotation]
    want, off = [], 0
    for pw, ph, e in plane_shapes(fmt, w, h):
        want.append(np.ascontiguousarray(graph(elem_view(frame[off: off + pw * ph * e], pw, ph, e))).view(np.uint8).ravel())
        off += pw * ph * e
    want = np.concatenate(want)
    released = []
    rel = REL(lambda opaque: released.append(int(opaque or 0)))
    side = torch.cuda.Stream()
    pitch_in = (byte_shapes(fmt, w, h)[0][0] + 511) // 512 * 512 + 512
    pitch_out = (byte_shapes(fmt, ow, oh)[0][0] + 511) // 512 * 512
    fin, surf_in, _ = wrap_torch(lib, torch, fmt, w, h, pitch_in, 0, side, frame, rel, 7)
    fout, surf_out, offs_out = wrap_torch(lib, torch, fmt, ow, oh, pitch_out, 0x5C)
    cfg = config_of(fmt, w, h, settings)
    hd = C.c_void_p()
    assert lib.hbcu_rotate_create(C.byref(hd), C.byref(cfg)) == 0, lib.hbcu_last_error()
    assert lib.hbcu_rotate_frame(hd, C.c_int64(0), fin, None, None, fout, None, None) == 0, lib.hbcu_last_error()
    lib.hbcu_frame_release(fin)
    assert released == [7]
    assert lib.hbcu_rotate_sync(hd) == 0
    got, tails = surface_planes(surf_out, offs_out, fmt, ow, oh, pitch_out)
    assert np.array_equal(got, want)
    assert np.all(tails == 0x5C), "a byte past a row's samples was written"
    lib.hbcu_frame_release(fout)
    lib.hbcu_rotate_destroy(hd)
    del surf_in, surf_out
    assert lib.hbcu_frames_alive() == 0


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,settings", [("yuv420p", "angle=90:hflip=0"), ("nv12", "angle=0:hflip=1"),
                                          ("p010le", "angle=270:hflip=1"), ("yuv420p10le", "angle=180:hflip=0")])
def test_host_input_device_output(cuda_filters, fmt, settings):
    """hw_pix_fmt = AV_PIX_FMT_CUDA: host frames in, device frames out, props and colour fields carried"""
    lib = core()
    w, h, n = 33, 17, 5
    got = check_props(cuda_filters.lib, fmt, settings, hw_pix_fmt=AV_PIX_FMT_CUDA)
    assert len(got) == n + 1 and lib.hbcu_frames_alive() == 0 and cuda_filters.buffers_alive() == 0
    clip = clip_of(fmt, w, h, n, seed=4)
    g = cuda_filters.run([ROT, DOWN], [settings, None], clip, FORMATS[fmt][0], w, h)
    assert np.array_equal(g.frames, rotate_clip(clip, fmt, w, h, settings))


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["yuv420p", "nv12", "p010le", "yuv444p10le"])
@pytest.mark.parametrize("device", [False, True])
def test_round_trips_are_identity(cuda_filters, fmt, device):
    """90 then 270, 180 twice, each flip twice and each _flip transpose twice"""
    w, h = 1921, 1081
    clip = clip_of(fmt, w, h, 2, seed=5)
    for pair in (("angle=90:hflip=0", "angle=270:hflip=0"), ("angle=180:hflip=0",) * 2, ("angle=0:hflip=1",) * 2,
                 ("angle=180:hflip=1",) * 2, ("angle=90:hflip=1",) * 2, ("angle=270:hflip=1",) * 2):
        chain = [ROT, ROT] if not device else [UP, ROT, ROT, DOWN]
        sets = list(pair) if not device else [None, *pair, None]
        g = cuda_filters.run(chain, sets, clip, FORMATS[fmt][0], w, h, par=(8, 9))
        assert np.array_equal(g.frames, clip) and (g.width, g.height, g.par) == (w, h, (8, 9)), pair
    assert core().hbcu_frames_alive() == 0 and cuda_filters.buffers_alive() == 0


@pytest.mark.gpu
def test_passthrough_and_refusals(cuda_filters):
    check_passthrough_and_refusals(cuda_filters.lib, device=True, launches=core().hbcu_kernel_launches)
    assert core().hbcu_frames_alive() == 0 and cuda_filters.buffers_alive() == 0


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(CHAIN_CASES)))
def test_chain_matches_reference(rref, cuda_filters, case):
    """rotate -> NLMeans -> lapsharp on host and on device frames: the reference's NLMeans -> lapsharp on the rotated
    input"""
    fmt, w, h, settings = CHAIN_CASES[case]
    r = chain_ref(rref, fmt, w, h, settings)
    clip = chain_inputs(fmt, w, h)
    for chain, sets in (([ROT] + product(CHAIN[0]), [settings] + CHAIN[1]),
                        ([UP, ROT] + product(CHAIN[0]) + [DOWN], [None, settings] + CHAIN[1] + [None])):
        g = cuda_filters.run(chain, sets, clip, FORMATS[fmt][0], w, h)
        assert g.init_failed == 0 and np.array_equal(g.frames, r.frames), chain
    assert core().hbcu_frames_alive() == 0 and cuda_filters.buffers_alive() == 0


@pytest.mark.gpu
def test_nv12_surfaces_chain_matches_reference(rref, cuda_filters, monkeypatch):
    """wrapped NV12 surfaces (the upload adapter playing NVDEC) -> rotate angle=90 -> format=yuv420p -> NLMeans ->
    download: the reference's NLMeans on the rotated, de-interleaved input; every surface goes back to its owner"""
    r = nv12_chain_ref(rref)
    w, h, clip = nv12_chain_inputs()
    monkeypatch.setenv("HBCU_UPLOAD_EXTERNAL", "1")
    cuda_filters.lib.hbcu_test_surfaces_returned.restype = C.c_long
    before = cuda_filters.lib.hbcu_test_surfaces_returned()
    g = cuda_filters.run([UP, ROT, FMT] + product(NV12_CHAIN[0]) + [DOWN],
                         [None, "angle=90:hflip=0", "format=yuv420p"] + NV12_CHAIN[1] + [None], to_nv12(clip, w, h), 23, w, h)
    assert g.init_failed == 0 and np.array_equal(g.frames, r.frames)
    assert cuda_filters.lib.hbcu_test_surfaces_returned() - before == len(clip)
    assert core().hbcu_frames_alive() == 0 and cuda_filters.buffers_alive() == 0


@pytest.mark.gpu
def test_surfaces_return_before_the_nlmeans_window_moves_on(cuda_filters):
    """wrapped NV12 surfaces -> rotate angle=90 -> format -> NLMeans frame-count=4 at the C-ABI: a surface goes back to
    its owner as soon as it is released behind the queued rotation, before NLMeans has even taken the frame, while
    NLMeans holds 4 frames; the denoised frames equal those of the numpy-rotated planar host input"""
    import torch
    lib = core()
    flt = cuda_filters.lib
    w, h, n = 640, 360, 10
    ow, oh = h, w
    planar = synth.progressive_clip(synth.PIX_FMT_YUV420P, w, h, n, seed=12)
    semi = to_nv12(planar, w, h)
    cfg = NlmConfig()
    flt.hb_parse_filter_settings.restype = C.c_void_p
    flt.hb_parse_filter_settings.argtypes = [C.c_char_p]
    flt.hb_nlmeans_cuda_build_config.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(NlmConfig), C.c_void_p, C.c_void_p, C.c_void_p]
    assert flt.hb_nlmeans_cuda_build_config(flt.hb_parse_filter_settings(b"y-strength=6:frame-count=4"), 0, ow, oh,
                                            C.byref(cfg), None, None, None) == 0
    cfg.device, cfg.ring_frames, cfg.out_slots = 0, 12, 4
    from test_format_gpu import FormatConfig
    rcfg = config_of("nv12", w, h, "angle=90:hflip=0")
    fcfg = FormatConfig(ow, oh, 8, 0, 0, 6)
    nl, rt, fm = C.c_void_p(), C.c_void_p(), C.c_void_p()
    assert lib.hbcu_nlmeans_create(C.byref(nl), C.byref(cfg)) == 0, lib.hbcu_last_error()
    assert lib.hbcu_rotate_create(C.byref(rt), C.byref(rcfg)) == 0, lib.hbcu_last_error()
    assert lib.hbcu_format_create(C.byref(fm), C.byref(fcfg)) == 0, lib.hbcu_last_error()
    released, keep, outs = [], [], []
    rel = REL(lambda opaque: released.append(int(opaque or 0)))
    side = torch.cuda.Stream()

    def pooled(fmt):
        shapes = byte_shapes(fmt, ow, oh)
        fr = C.c_void_p()
        rb = (C.c_int * 3)(*[s[0] for s in shapes]); rows = (C.c_int * 3)(*[s[1] for s in shapes])
        st = (C.c_int * 3)(*[(s[0] + 63) // 64 * 64 for s in shapes])
        assert lib.hbcu_frame_alloc(C.byref(fr), 0, rb, rows, st) == 0, lib.hbcu_last_error()
        return fr

    for t in range(n):
        fin, surf, _ = wrap_torch(lib, torch, "nv12", w, h, 1024, 0, side, semi[t], rel, t + 1)
        keep.append(surf)
        frot, fpl = pooled("nv12"), pooled("yuv420p")
        assert lib.hbcu_rotate_frame(rt, C.c_int64(t), fin, None, None, frot, None, None) == 0, lib.hbcu_last_error()
        lib.hbcu_frame_release(fin)                      # what rotate_cuda.c does once the rotation is queued
        assert released[-1:] == [t + 1], "the surface went back before the frame reached NLMeans"
        assert lib.hbcu_format_convert(fm, C.c_int64(t), frot, None, None, fpl, None, None) == 0, lib.hbcu_last_error()
        lib.hbcu_frame_release(frot)
        assert lib.hbcu_nlmeans_upload_frame(nl, C.c_int64(t), fpl) == 0, lib.hbcu_last_error()
        lib.hbcu_frame_release(fpl)
        if t >= 3:
            k = t - 3
            dims = synth.plane_dims(ow, oh)
            o = [np.zeros((ph, pw), np.uint8) for pw, ph in dims]
            ptrs = (C.c_void_p * 3)(*[a.ctypes.data for a in o]); ost = (C.c_int * 3)(*[pw for pw, _ in dims])
            assert lib.hbcu_nlmeans_filter(nl, C.c_int64(k), 4, ptrs, ost) == 0, lib.hbcu_last_error()
            assert lib.hbcu_nlmeans_wait(nl, C.c_int64(k)) == 0
            outs.append(np.concatenate([a.ravel() for a in o]))
    assert sorted(released) == list(range(1, n + 1))
    lib.hbcu_format_destroy(fm)
    lib.hbcu_rotate_destroy(rt)
    lib.hbcu_nlmeans_destroy(nl)
    want = cuda_filters.run("hb_filter_nlmeans_cuda", "y-strength=6:frame-count=4",
                            rotate_clip(planar, "yuv420p", w, h, "angle=90:hflip=0"), 0, ow, oh)
    assert np.array_equal(np.stack(outs), want.frames[: len(outs)])
    assert lib.hbcu_frames_alive() == 0
