"""Semi-planar 4:2:0 frames (NV12, P010, P016: what NVDEC decodes into) through the shim, the device frames, hb_blend_cuda
and the framerate shaper, against the reference's own blend.c (its *bi* functions) and vfr.c.

  - the shim: FFmpeg's descriptors, plane counts and linesizes; packed frames and guard bands round-trip per plane;
  - the planar-only CUDA filters refuse the formats in init(); hb_filter_vfr_cuda takes NV12 in every mode and P010 /
    P016 in mode 0 only;
  - hb_blend_cuda on NV12 / P010 / P016 with YUVA 4:2:0 (plain path) and YUVA 4:4:4 (subsample path, every chroma
    location) overlays, on the geometry set of tests/test_blend_gpu.py, on host frames with guard bands and on device
    frames;
  - two-plane device frames: host -> device -> host, a torch-allocated NV12 surface at a decoder pitch wrapped with
    hbcu_frame_wrap, and a hardware-decoder-like chain (wrapped surfaces -> vfr -> render_sub -> download).

The reference's results are stored in tests/golden/blend_semiplanar_ref_digests.json.  On a machine without a GPU the
host objects over the plain-C restatements, extended to semi-planar frames (oracle/semiplanar.mk,
oracle/_ref/libhostlogic_semiplanar.so), must reproduce each of them.  `HBCU_RECORD_REF=1` with the reference built (oracle/blend.mk, oracle/vfr.mk) re-records them through the CPU
tests, which make every reference call the GPU tests make."""
import ctypes as C
import json
from pathlib import Path

import numpy as np
import pytest

from golden_ref import REPO, GoldenRef, RecordedResult, _h, result_digest
from handbrake_b200 import LIBHBCU, synth
from handbrake_b200.hblib import FilterLib, RENDER_SUB
from test_blend_gpu import OVERLAY_FMTS, REF_BLEND_SO, assert_same, geometry_spec, overlays_of
from test_vfr_gpu import REF_VFR_SO, luma, timestamps

STORE = Path(__file__).resolve().parent / "golden" / "blend_semiplanar_ref_digests.json"
# built by oracle/semiplanar.mk: the host filters, hb_blend_cuda and hb_filter_vfr_cuda over the restatements, with
# two-plane device frames and blend.c's semi-planar functions
HOSTLOGIC_SEMI_SO = REPO / "oracle" / "_ref" / "libhostlogic_semiplanar.so"
UP, DOWN = "hb_filter_hbcu_upload", "hb_filter_hbcu_download"
# the shim's enum AVPixelFormat (FFmpeg's values): (pix_fmt, depth); samples sit in the high bits of 16-bit words
SEMI = {"nv12": (synth.PIX_FMT_NV12, 8), "p010": (synth.PIX_FMT_P010, 10), "p016": (synth.PIX_FMT_P016, 16)}
NTSC, FILM = (30000, 1001), (24000, 1001)
LOC_CENTER = 2


def chroma_dims(w, h):
    return -((-w) >> 1), -((-h) >> 1)


def semi_frame(fmt, y, rng):
    """a packed semi-planar frame: luma y (h, w) of depth-bit values, random Cb/Cr pairs"""
    depth = SEMI[fmt][1]
    h, w = y.shape
    cw, ch = chroma_dims(w, h)
    c = rng.integers(0, 1 << depth, (ch, 2 * cw))
    if depth == 8:
        return np.concatenate([y.astype(np.uint8).ravel(), c.astype(np.uint8).ravel()])
    up = 16 - depth
    return np.concatenate([(y.astype(np.uint16) << up).ravel(), (c.astype(np.uint16) << up).ravel()]).view(np.uint8)


def semi_frames(fmt, w, h, n, seed):
    rng = np.random.default_rng(seed)
    return np.stack([semi_frame(fmt, rng.integers(0, 1 << SEMI[fmt][1], (h, w)), rng) for _ in range(n)])


# ---------------------------------------------------------------------------------------------------------- cases
def build_cases():
    cases = []
    for fmt in SEMI:
        for ofmt in ("yuva420p", "yuva444p"):
            for w, h in ((128, 96), (333, 211)):
                cases.append(dict(id=f"{fmt}-{ofmt}-{w}x{h}", fmt=fmt, ofmt=ofmt, w=w, h=h, loc=LOC_CENTER, n=4,
                                  spec=geometry_spec(w, h, 4)))
    for fmt in ("nv12", "p010"):
        for loc in range(7):
            w, h = 97, 63
            spec = [(0, 3, 5, 40, 30, "glyph"), (0, 20, 16, 50, 33, "noise"), (0, -3, -1, 17, 11, "ramp")]
            cases.append(dict(id=f"loc{loc}-{fmt}", fmt=fmt, ofmt="yuva444p", w=w, h=h, loc=loc, n=1, spec=spec))
    return cases


CASES = build_cases()


def case_inputs(c):
    frames = semi_frames(c["fmt"], c["w"], c["h"], c["n"], seed=c["w"] + c["n"] + len(c["id"]))
    return frames, overlays_of(c["spec"], c["ofmt"], seed=len(c["id"]) * 7 + c["w"])


def chain_inputs():
    """NVDEC-like NV12 1080p at 29.97 with 3:2-like repeats, shaped to 23.976 CFR, then an SSA-like band per frame"""
    w, h, n = 1920, 1080, 20
    rng = np.random.default_rng(41)
    frames, base = [], None
    for i in range(n):
        base = luma("scene", 8, w, h, rng) if i % 5 in (0, 3) or base is None else luma("jitter", 8, w, h, rng, base=base)
        frames.append(semi_frame("nv12", base, np.random.default_rng(100 + i)))
    start, stop = timestamps(n, NTSC)
    spec = [(f, 160 + 2 * f, 900 - f, 1600, 120, "glyph") for f in range(n)]
    return w, h, np.stack(frames), start, stop, overlays_of(spec, "yuva444p", seed=17)


CHAIN_SETTINGS = "mode=1:rate=24000/1001"


# ---------------------------------------------------------------------------------------------------------- reference
class SemiRef(GoldenRef):
    """GoldenRef over this file's own store: the reference's hb_blend and hb_filter_vfr on semi-planar frames"""

    def __init__(self):
        super().__init__()
        self.store = json.loads(STORE.read_text()) if STORE.exists() else {}
        if self.recording:
            self.blend_lib, self.vfr_lib = FilterLib(REF_BLEND_SO), FilterLib(REF_VFR_SO)
        self.host = FilterLib(HOSTLOGIC_SEMI_SO)

    def _save(self):
        STORE.write_text(json.dumps(dict(sorted(self.store.items())), indent=0) + "\n")

    def _want(self, key, what):
        if key not in self.store:
            raise KeyError(f"no stored reference result for {what} ({key}): record it with HBCU_RECORD_REF=1 where the "
                           "reference is built")
        return self.store[key]

    def blend(self, overlays, ofmt, frames, fmt, w, h, loc=LOC_CENTER, guard=(0, 0)):
        """the reference's hb_blend through the render_sub stand-in; checked against the CPU restatement"""
        pix, opix = SEMI[fmt][0], OVERLAY_FMTS[ofmt][0]
        key = _h("blend-semi", pix, w, h, np.ascontiguousarray(frames), opix, loc,
                 [(o[0], o[1], o[2], o[3], o[4], _h(o[5])) for o in overlays], tuple(guard))
        kw = dict(chroma_location=loc, guard=guard)
        if self.recording:
            r, _ = self.blend_lib.run_blend("hb_blend", overlays, opix, [RENDER_SUB], [None], frames, pix, w, h, **kw)
            self.store[key] = result_digest(r)
            self._save()
            return r
        want = self._want(key, f"blend {fmt} {w}x{h}")
        r, _ = self.host.run_blend("hb_blend_cuda", overlays, opix, [RENDER_SUB], [None], frames, pix, w, h, **kw)
        assert result_digest(r) == want, f"the CPU restatement of the {fmt} {w}x{h} blend no longer reproduces the reference"
        return r

    def vfr_then_blend(self):
        """the reference's vfr, then its hb_blend on vfr's output (vfr hands frames on untouched): per-frame digests and
        timestamps of the NV12 chain"""
        w, h, frames, start, stop, ov = chain_inputs()
        pix, opix = SEMI["nv12"][0], OVERLAY_FMTS["yuva444p"][0]
        key = _h("vfr-blend-semi", CHAIN_SETTINGS, pix, w, h, frames, start, stop,
                 [(o[0], o[1], o[2], o[3], o[4], _h(o[5])) for o in ov])
        vfr_kw = dict(start=start, stop=stop, vrate=NTSC)
        if self.recording:
            vlib, blib, vname, bname = self.vfr_lib, self.blend_lib, "hb_filter_vfr", "hb_blend"
        else:
            vlib, blib, vname, bname = self.host, self.host, "hb_filter_vfr_cuda", "hb_blend_cuda"
        v = vlib.run(vname, CHAIN_SETTINGS, frames, pix, w, h, **vfr_kw)
        r, _ = blib.run_blend(bname, ov, opix, [RENDER_SUB], [None], v.frames, pix, w, h, start=v.start, stop=v.stop)
        got = RecordedResult.record(r)
        if self.recording:
            self.store[key] = got
            self._save()
        else:
            assert got == self._want(key, "the NV12 vfr -> blend chain"), "the CPU restatement no longer reproduces the chain"
        return RecordedResult(got)


@pytest.fixture(scope="module")
def sref():
    return SemiRef()


# ---------------------------------------------------------------------------------------------------------- CPU tests
class Comp(C.Structure):
    _fields_ = [("plane", C.c_int), ("step", C.c_int), ("offset", C.c_int), ("shift", C.c_int), ("depth", C.c_int)]


class Desc(C.Structure):
    _fields_ = [("name", C.c_char_p), ("nb_components", C.c_uint8), ("log2_chroma_w", C.c_uint8),
                ("log2_chroma_h", C.c_uint8), ("flags", C.c_uint64), ("comp", Comp * 4)]


def shim():
    lib = FilterLib(HOSTLOGIC_SEMI_SO).lib
    lib.av_pix_fmt_desc_get.restype = C.POINTER(Desc)
    return lib


@pytest.mark.parametrize("fmt", list(SEMI))
def test_descriptors_planes_and_linesizes(fmt):
    lib = shim()
    pix, depth = SEMI[fmt]
    d = lib.av_pix_fmt_desc_get(pix).contents
    bytes_ = 1 if depth == 8 else 2
    assert d.name.decode() == {"nv12": "nv12", "p010": "p010le", "p016": "p016le"}[fmt]
    assert (d.nb_components, d.log2_chroma_w, d.log2_chroma_h) == (3, 1, 1)
    comps = [(c.plane, c.step, c.offset, c.shift, c.depth) for c in d.comp[:3]]
    shift = 6 if fmt == "p010" else 0
    assert comps == [(0, bytes_, 0, shift, depth), (1, 2 * bytes_, 0, shift, depth), (1, 2 * bytes_, bytes_, shift, depth)]
    assert lib.av_pix_fmt_count_planes(pix) == 2
    for w in (1, 2, 333, 1920):
        cw = (w + 1) // 2
        assert [lib.av_image_get_linesize(pix, w, p) for p in range(4)] == [w * bytes_, 2 * cw * bytes_, 0, 0]
        assert lib.hb_harness_frame_bytes(pix, w, 211) == (w * 211 + 2 * cw * 106) * bytes_


def test_planar_linesizes_unchanged():
    lib = shim()
    for pix, bps, cws in ((0, 1, 1), (62, 2, 1), (5, 1, 0), (79, 1, 0)):
        assert [lib.av_image_get_linesize(pix, 333, p) for p in range(3)] == [333 * bps] + [(333 + cws) // (1 + cws) * bps] * 2
    assert lib.av_pix_fmt_count_planes(0) == 3 and lib.av_pix_fmt_count_planes(79) == 4


@pytest.mark.parametrize("fmt", list(SEMI))
def test_packed_frames_round_trip(fmt):
    """packed -> hb_frame_buffer_init's two planes -> packed, alone, through the host stand-ins of the device frames,
    and through the render_sub stand-in with guard bands (no overlays: nothing may change, no guard byte either)"""
    w, h = 333, 211
    pix = SEMI[fmt][0]
    frames = semi_frames(fmt, w, h, 3, seed=8)
    lib = FilterLib(HOSTLOGIC_SEMI_SO)
    assert np.array_equal(lib.run([], [], frames, pix, w, h).frames, frames)
    assert np.array_equal(lib.run([UP, DOWN], [None, None], frames, pix, w, h).frames, frames)
    r, st = lib.run_blend("hb_blend_cuda", [], OVERLAY_FMTS["yuva444p"][0], [RENDER_SUB], [None], frames, pix, w, h, guard=(5, 3))
    assert np.array_equal(r.frames, frames) and st["guard_damaged"] == 0 and st["frames"] == 3
    assert lib.buffers_alive() == 0


PLANAR_ONLY = ["hb_filter_nlmeans_cuda", "hb_filter_comb_detect_cuda", "hb_filter_decomb_cuda", "hb_filter_lapsharp_cuda",
               "hb_filter_unsharp_cuda", "hb_filter_chroma_smooth_cuda", "hb_filter_denoise_cuda", "hb_filter_detelecine_cuda"]


@pytest.mark.parametrize("fmt", list(SEMI))
@pytest.mark.parametrize("name", PLANAR_ONLY)
def test_planar_filters_refuse_semiplanar(fmt, name):
    w, h = 64, 48
    frames = semi_frames(fmt, w, h, 2, seed=3)
    r = FilterLib(HOSTLOGIC_SEMI_SO).run([name], [None], frames, SEMI[fmt][0], w, h)
    assert r.init_failed == 1 and np.array_equal(r.frames, frames)


@pytest.mark.parametrize("fmt", list(SEMI))
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_vfr_formats_per_mode(fmt, mode):
    """the metric reads plane 0: NV12 in every mode; P010 / P016 would index the gamma table with 16-bit samples"""
    w, h, n = 64, 48, 10
    frames = semi_frames(fmt, w, h, n, seed=4)
    start, stop = timestamps(n, NTSC)
    r = FilterLib(HOSTLOGIC_SEMI_SO).run("hb_filter_vfr_cuda", f"mode={mode}:rate=24000/1001", frames, SEMI[fmt][0], w, h,
                                        start=start, stop=stop, vrate=NTSC)
    refused = mode > 0 and fmt != "nv12"
    assert r.init_failed == int(refused)
    assert r.saw_eof and r.frames.shape[0] > 0


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_restatement_reproduces_reference(sref, case):
    c = case
    frames, ov = case_inputs(c)
    r = sref.blend(ov, c["ofmt"], frames, c["fmt"], c["w"], c["h"], loc=c["loc"], guard=(c["w"], c["h"]))
    assert r.frames.shape[0] == c["n"]


def test_restatement_reproduces_reference_vfr_chain(sref):
    r = sref.vfr_then_blend()
    assert r.saw_eof and 0 < r.shape[0] < 20


def test_restatement_pfr_below_peak(sref):
    w, h, n, frames, ov = pfr_inputs()
    sref.blend(ov, "yuva420p", frames, "nv12", w, h)


def test_restatement_wrapped_surface_case(sref):
    w, h, frames, ov = wrap_inputs()
    sref.blend(ov, "yuva444p", frames, "nv12", w, h)


def wrap_inputs():
    w, h = 640, 360
    ov_spec = [(0, 100, 280, 440, 60, "glyph"), (0, -7, -5, 120, 90, "noise")]
    return w, h, semi_frames("nv12", w, h, 1, seed=31), overlays_of(ov_spec, "yuva444p", seed=2)


def pfr_inputs():
    w, h, n = 320, 180, 12
    return w, h, n, semi_frames("nv12", w, h, n, seed=12), overlays_of([(f, 20, 120, 280, 40, "glyph") for f in range(n)], "yuva420p", seed=5)


# ---------------------------------------------------------------------------------------------------------- GPU tests
def core():
    lib = C.CDLL(str(LIBHBCU))
    lib.hbcu_frames_alive.restype = C.c_long
    lib.hbcu_last_error.restype = C.c_char_p
    lib.hbcu_motion_metric_waits.restype = C.c_uint64
    lib.hbcu_frame_plane.restype = C.c_void_p
    lib.hbcu_frame_plane.argtypes = [C.c_void_p, C.c_int]
    lib.hbcu_frame_stride.argtypes = [C.c_void_p, C.c_int]
    lib.hbcu_frame_release.argtypes = [C.c_void_p]
    return lib


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_semiplanar_blend_matches_reference(sref, cuda_filters, case):
    c = case
    frames, ov = case_inputs(c)
    guard = (c["w"], c["h"])
    r = sref.blend(ov, c["ofmt"], frames, c["fmt"], c["w"], c["h"], loc=c["loc"], guard=guard)
    pix, opix = SEMI[c["fmt"]][0], OVERLAY_FMTS[c["ofmt"]][0]
    g, st = cuda_filters.run_blend("hb_blend_cuda", ov, opix, [RENDER_SUB], [None], frames, pix, c["w"], c["h"],
                                   chroma_location=c["loc"], guard=guard)
    assert g.init_failed == 0
    assert_same(r, g)
    assert st["guard_damaged"] == 0, "the CUDA blend wrote outside the picture"
    d, _ = cuda_filters.run_blend("hb_blend_cuda", ov, opix, [UP, RENDER_SUB, DOWN], [None] * 3, frames, pix, c["w"], c["h"],
                                  chroma_location=c["loc"])
    assert_same(r, d)
    assert core().hbcu_frames_alive() == 0 and cuda_filters.buffers_alive() == 0


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", list(SEMI))
def test_two_plane_frames_round_trip(cuda_filters, fmt):
    w, h = 333, 211
    frames = semi_frames(fmt, w, h, 4, seed=21)
    g = cuda_filters.run([UP, DOWN], [None, None], frames, SEMI[fmt][0], w, h)
    assert np.array_equal(g.frames, frames)
    assert core().hbcu_frames_alive() == 0 and cuda_filters.buffers_alive() == 0


class BlendConfig(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("depth", C.c_int), ("chroma_shift_w", C.c_int),
                ("chroma_shift_h", C.c_int), ("overlay_shift_w", C.c_int), ("overlay_shift_h", C.c_int),
                ("device", C.c_int), ("chroma_coeffs", C.c_uint32 * 8), ("interleaved_chroma", C.c_int)]


class BlendOverlay(C.Structure):
    _fields_ = [("x", C.c_int), ("y", C.c_int), ("width", C.c_int), ("height", C.c_int),
                ("planes", C.c_void_p * 4), ("strides", C.c_int * 4)]


@pytest.mark.gpu
def test_torch_nv12_surface_wrapped(sref, cuda_filters):
    """an NV12 surface another allocator (torch) owns, at a decoder-like pitch, written on its own stream: wrapped with
    hbcu_frame_wrap (two planes), blended into a pooled frame, downloaded; the reference's bytes, one release"""
    import torch
    lib = core()
    w, h, frames, ov = wrap_inputs()
    pitch = 768
    cw, ch = chroma_dims(w, h)
    want = sref.blend(ov, "yuva444p", frames, "nv12", w, h)

    rows_alloc = 368 + 184                    # decoder surfaces: heights aligned up, chroma after the aligned luma
    side = torch.cuda.Stream()
    surf = torch.zeros(rows_alloc * pitch + 4096, dtype=torch.uint8, device="cuda")
    with torch.cuda.stream(side):
        y_dev = surf[: h * pitch].view(h, pitch)
        uv_dev = surf[368 * pitch: 368 * pitch + ch * pitch].view(ch, pitch)
        y_dev[:, :w].copy_(torch.from_numpy(frames[0, : w * h].reshape(h, w)), non_blocking=False)
        uv_dev[:, : 2 * cw].copy_(torch.from_numpy(frames[0, w * h:].reshape(ch, 2 * cw)), non_blocking=False)
    released = []
    REL = C.CFUNCTYPE(None, C.c_void_p)
    rel = REL(lambda opaque: released.append(1))
    fin = C.c_void_p()
    dplanes = (C.c_void_p * 3)(surf.data_ptr(), surf.data_ptr() + 368 * pitch, None)
    row_bytes, rows = (C.c_int * 3)(w, 2 * cw, 0), (C.c_int * 3)(h, ch, 0)
    strides = (C.c_int * 3)(pitch, pitch, 0)
    assert lib.hbcu_frame_wrap(C.byref(fin), 0, dplanes, row_bytes, rows, strides, C.c_size_t(4096),
                               C.c_void_p(side.cuda_stream), rel, None) == 0, lib.hbcu_last_error()
    assert lib.hbcu_frame_plane(fin, 2) is None and lib.hbcu_frame_stride(fin, 2) == 0

    cfg = BlendConfig(w, h, 8, 1, 1, 0, 0, 0)
    cfg.interleaved_chroma = 1
    coeff = (C.c_uint32 * 8)()
    cuda_filters.lib.hb_compute_chroma_smoothing_coefficient(coeff, SEMI["nv12"][0], LOC_CENTER)
    cfg.chroma_coeffs[:] = list(coeff)
    hnd = C.c_void_p()
    assert lib.hbcu_blend_create(C.byref(hnd), C.byref(cfg)) == 0, lib.hbcu_last_error()
    arr, keep = (BlendOverlay * len(ov))(), []
    for i, (_, x, y, ow, oh, yuva) in enumerate(ov):
        o = arr[i]
        o.x, o.y, o.width, o.height = x, y, ow, oh
        off = 0
        for p in range(4):
            a = np.ascontiguousarray(yuva[off: off + ow * oh])
            keep.append(a)
            o.planes[p], o.strides[p] = a.ctypes.data, ow
            off += ow * oh
    assert lib.hbcu_blend_set_overlays(hnd, arr, len(ov), 1) == 0
    out_strides = (C.c_int * 3)(640, 640, 0)
    fout = C.c_void_p()
    assert lib.hbcu_frame_alloc(C.byref(fout), 0, row_bytes, rows, out_strides) == 0, lib.hbcu_last_error()
    assert lib.hbcu_blend_frames(hnd, fin, None, None, fout, None, None) == 0, lib.hbcu_last_error()
    lib.hbcu_frame_release(fin)                # the caller's reference goes; the queued blend still reads the surface
    x = C.c_void_p()
    assert lib.hbcu_xfer_create(C.byref(x), 0, 4) == 0
    got_y, got_uv = np.zeros((h, 640), np.uint8), np.zeros((ch, 640), np.uint8)
    hp = (C.c_void_p * 3)(got_y.ctypes.data, got_uv.ctypes.data, None)
    assert lib.hbcu_xfer_download(x, C.c_int64(0), fout, hp, out_strides) == 0, lib.hbcu_last_error()
    assert lib.hbcu_xfer_wait(x, C.c_int64(0)) == 0
    lib.hbcu_xfer_destroy(x)
    lib.hbcu_frame_release(fout)
    lib.hbcu_blend_destroy(hnd)
    got = np.concatenate([got_y[:, :w].ravel(), got_uv[:, : 2 * cw].ravel()])
    assert np.array_equal(got, want.frames[0])
    assert released == [1], "the surface's release callback must run exactly once"
    assert lib.hbcu_frames_alive() == 0


@pytest.mark.gpu
def test_decoder_surfaces_vfr_cfr_then_blend(sref, cuda_filters, monkeypatch):
    """wrapped NV12 surfaces (the upload adapter playing NVDEC) -> hb_filter_vfr_cuda 29.97 -> 23.976 CFR ->
    render_sub(hb_blend_cuda) -> download: the reference's vfr-then-blend frames and timestamps"""
    want = sref.vfr_then_blend()
    w, h, frames, start, stop, ov = chain_inputs()
    monkeypatch.setenv("HBCU_UPLOAD_EXTERNAL", "1")
    cuda_filters.lib.hbcu_test_surfaces_returned.restype = C.c_long
    before = cuda_filters.lib.hbcu_test_surfaces_returned()
    g, _ = cuda_filters.run_blend("hb_blend_cuda", ov, OVERLAY_FMTS["yuva444p"][0], [UP, "hb_filter_vfr_cuda", RENDER_SUB, DOWN],
                                  [None, CHAIN_SETTINGS, None, None], frames, SEMI["nv12"][0], w, h,
                                  start=start, stop=stop, vrate=NTSC)
    assert g.init_failed == 0 and g.saw_eof and g.frames.shape == want.shape
    assert np.array_equal(g.start, want.start) and np.array_equal(g.stop, want.stop)
    bad = want.frames_differing(g.frames)
    assert not bad, f"frames {bad} differ from the reference's vfr -> blend"
    assert cuda_filters.lib.hbcu_test_surfaces_returned() - before == len(frames)
    assert core().hbcu_frames_alive() == 0 and cuda_filters.buffers_alive() == 0


@pytest.mark.gpu
def test_pfr_below_peak_adds_no_metric_wait(sref, cuda_filters, monkeypatch):
    """23.976 into a 30 fps peak: every frame passes, no metric result is read, the blend is the reference's"""
    w, h, n, frames, ov = pfr_inputs()
    want = sref.blend(ov, "yuva420p", frames, "nv12", w, h)
    monkeypatch.setenv("HBCU_UPLOAD_EXTERNAL", "1")
    lib = core()
    w0 = lib.hbcu_motion_metric_waits()
    start, stop = timestamps(n, FILM)
    g, _ = cuda_filters.run_blend("hb_blend_cuda", ov, OVERLAY_FMTS["yuva420p"][0], [UP, "hb_filter_vfr_cuda", RENDER_SUB, DOWN],
                                  [None, "mode=2:rate=30/1", None, None], frames, SEMI["nv12"][0], w, h,
                                  start=start, stop=stop, vrate=FILM)
    assert g.init_failed == 0 and np.array_equal(g.frames, want.frames)
    assert lib.hbcu_motion_metric_waits() == w0
    assert lib.hbcu_frames_alive() == 0 and cuda_filters.buffers_alive() == 0
