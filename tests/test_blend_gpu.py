"""hb_blend_cuda, the CUDA twin of libhb's subtitle overlay blend (blend.c), against the reference's hb_blend.

Both objects are driven by the harness's render_sub stand-in (hb_filter_render_sub_harness), which hands each frame its
overlay list the way rendersub.c does.  Every result must equal the reference's bit for bit inside the picture:
  - frame formats 8/10/12/16-bit 4:2:0, 8/10-bit 4:2:2, 8/10-bit 4:4:4; YUVA 4:4:4 overlays on all of them (the
    subsample path on 4:2:0 / 4:2:2), YUVA 4:2:0 on 4:2:0 and YUVA 4:2:2 on 4:2:2 (the plain path);
  - every chroma location on the subsample path;
  - overlays inside, at the origin, touching and crossing every edge at even and odd offsets, larger than the frame,
    1x1, overlapping (list order decides), on odd frame sizes;
  - alpha 0, 255, ramps, noise and anti-aliased glyph masks.
Frames get guard bands (spare rows and columns around the picture) where the reference writes outside the picture; the
CUDA object must leave them untouched.

The reference's results are stored in tests/golden/blend_ref_digests.json.  On a machine without a GPU the host object
over the plain-C restatement (oracle/port/blend_port.c, oracle/_ref/libhostlogic_blend.so) must reproduce each of them.
`HBCU_RECORD_REF=1` with the reference's blend built (oracle/blend.mk, oracle/_ref/libhbref_blend.so) re-records them,
through the CPU tests, which make every reference call the GPU tests make."""
import ctypes as C
import json
import os
from pathlib import Path

import numpy as np
import pytest

import handbrake_b200
from golden_ref import GoldenRef, RecordedResult, _h, result_digest
from handbrake_b200 import LIBHBCU, synth
from handbrake_b200.hblib import RENDER_SUB

STORE = Path(__file__).resolve().parent / "golden" / "blend_ref_digests.json"
REPO = Path(__file__).resolve().parent.parent
# built by oracle/blend.mk: the reference's filters with its hb_blend, and the host filters with hb_blend_cuda over the
# plain-C restatement
REF_BLEND_SO = REPO / "oracle" / "_ref" / "libhbref_blend.so"
HOSTLOGIC_BLEND_SO = REPO / "oracle" / "_ref" / "libhostlogic_blend.so"
UP, DOWN = "hb_filter_hbcu_upload", "hb_filter_hbcu_download"

# the shim's enum AVPixelFormat: frame formats (depth, chroma shifts) and overlay formats (chroma shifts)
FRAME_FMTS = {"420p": (0, 8, 1, 1), "420p10": (62, 10, 1, 1), "420p12": (123, 12, 1, 1), "420p16": (47, 16, 1, 1),
              "422p": (4, 8, 1, 0), "422p10": (64, 10, 1, 0), "444p": (5, 8, 0, 0), "444p10": (68, 10, 0, 0)}
OVERLAY_FMTS = {"yuva420p": (33, 1, 1), "yuva422p": (78, 1, 0), "yuva444p": (79, 0, 0)}
LOC_CENTER = 2


def plane_dims(w, h, sw, sh, n):
    cw, ch = -((-w) >> sw), -((-h) >> sh)
    return [(w, h), (cw, ch), (cw, ch), (w, h)][:n]


def make_frames(fmt, w, h, n, seed):
    pix, depth, sw, sh = FRAME_FMTS[fmt]
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        parts = []
        for pw, ph in plane_dims(w, h, sw, sh, 3):
            if depth == 8:
                parts.append(rng.integers(0, 256, pw * ph, dtype=np.uint8))
            else:
                parts.append(rng.integers(0, 1 << depth, pw * ph, dtype=np.uint16).view(np.uint8))
        out.append(np.concatenate(parts))
    return np.stack(out)


def alpha_mask(kind, w, h, rng):
    yy, xx = np.mgrid[0:h, 0:w]
    if kind == "zero":
        return np.zeros((h, w), np.uint8)
    if kind == "full":
        return np.full((h, w), 255, np.uint8)
    if kind == "ramp":
        return ((xx * 255 // max(1, w - 1) + yy * 97) % 256).astype(np.uint8)
    if kind == "noise":
        return rng.integers(0, 256, (h, w), dtype=np.uint8)
    # "glyph": anti-aliased strokes -- rings and a diagonal bar with soft 1.5-sample edges, as libass renders text
    cx, cy = w / 2.0, h / 2.0
    r = np.hypot(xx + 0.5 - cx, yy + 0.5 - cy)
    ring = np.clip(1.5 - np.abs(r - min(w, h) * 0.3), 0, 1)
    bar = np.clip(1.5 - np.abs((xx - yy * w / max(1, h)) * 0.7), 0, 1)
    return np.round(255 * np.maximum(ring, bar)).astype(np.uint8)


def make_overlay(ofmt, w, h, alpha, seed):
    _, sw, sh = OVERLAY_FMTS[ofmt]
    rng = np.random.default_rng(seed)
    parts = [rng.integers(0, 256, pw * ph, dtype=np.uint8) for pw, ph in plane_dims(w, h, sw, sh, 3)]
    parts.append(alpha_mask(alpha, w, h, rng).ravel())
    return np.concatenate(parts)


def overlays_of(spec, ofmt, seed):
    """spec: (frame, x, y, w, h, alpha kind) -> the stand-in's overlay tuples"""
    return [(f, x, y, w, h, make_overlay(ofmt, w, h, a, seed * 131 + i)) for i, (f, x, y, w, h, a) in enumerate(spec)]


# ---------------------------------------------------------------------------------------------------------- cases
def geometry_spec(w, h, n_frames=2):
    """overlays on every frame: inside, at the origin, touching the right / bottom edges exactly, crossing left / top at
    even and odd negative offsets, crossing right / bottom, larger than the frame, 1x1, odd positions, overlapping"""
    per_frame = [
        [(17, 11, 40, 30, "glyph"), (0, 0, 21, 13, "ramp"), (w - 25, h - 19, 25, 19, "noise"), (29, 23, 40, 30, "full")],
        [(-6, -4, 30, 20, "noise"), (-7, -5, 31, 21, "glyph"), (w - 20, h - 12, 37, 29, "ramp"), (w // 2, -3, 9, 8, "full"),
         (-3, h // 2 + 1, 9, 7, "noise")],
        [(-5, -9, w + 13, h + 11, "ramp"), (33, 21, 1, 1, "full"), (34, 21, 1, 1, "noise"), (w - 1, h - 1, 1, 1, "full"),
         (13, 7, 19, 17, "zero"), (14, 8, 19, 17, "glyph")],
        [(5, 3, 60, 40, "noise"), (6, 4, 60, 40, "glyph"), (7, 5, 60, 40, "ramp"), (-2, 1, w + 5, 4, "noise")],
    ]
    return [(f,) + o for f in range(n_frames) for o in per_frame[f % len(per_frame)]]


def build_cases():
    cases = []
    combos = [("420p", "yuva444p"), ("420p10", "yuva444p"), ("420p12", "yuva444p"), ("420p16", "yuva444p"),
              ("422p", "yuva444p"), ("422p10", "yuva444p"), ("444p", "yuva444p"), ("444p10", "yuva444p"),
              ("420p", "yuva420p"), ("420p10", "yuva420p"), ("420p12", "yuva420p"), ("420p16", "yuva420p"),
              ("422p", "yuva422p"), ("422p10", "yuva422p")]
    for fmt, ofmt in combos:
        for w, h in ((128, 96), (333, 211)):
            cases.append(dict(id=f"{fmt}-{ofmt}-{w}x{h}", fmt=fmt, ofmt=ofmt, w=w, h=h, loc=LOC_CENTER, n=4,
                              spec=geometry_spec(w, h, 4), guard=(w, h)))
    # chroma locations (unspecified, left, center, topleft, top, bottomleft, bottom) on the subsample path
    for fmt in ("420p", "422p", "420p10"):
        for loc in range(7):
            w, h = 97, 63
            spec = [(0, 3, 5, 40, 30, "glyph"), (0, 20, 16, 50, 33, "noise"), (0, -3, -1, 17, 11, "ramp")]
            cases.append(dict(id=f"loc{loc}-{fmt}", fmt=fmt, ofmt="yuva444p", w=w, h=h, loc=loc, n=1, spec=spec, guard=(w, h)))
    return cases


CASES = build_cases()


def case_overlays(c):
    return overlays_of(c["spec"], c["ofmt"], seed=len(c["id"]) * 7 + c["w"])


# ---------------------------------------------------------------------------------------------------------- reference
class BlendRef(GoldenRef):
    """GoldenRef over this file's own store: the reference's hb_blend through the stand-in, keyed by the whole call
    (chain, frames, overlays, changed flags, guard bands)"""

    def __init__(self):
        from handbrake_b200.hblib import FilterLib
        super().__init__()
        self.store = json.loads(STORE.read_text()) if STORE.exists() else {}
        if self.recording:
            self.lib = FilterLib(REF_BLEND_SO)
        self.host = FilterLib(HOSTLOGIC_BLEND_SO)

    def _save(self):
        STORE.write_text(json.dumps(dict(sorted(self.store.items())), indent=0) + "\n")

    def run_blend(self, overlays, ofmt, filters, settings, frames, fmt, w, h, loc=LOC_CENTER, changed=None, guard=(0, 0),
                  digest_only=False):
        pix, opix = FRAME_FMTS[fmt][0], OVERLAY_FMTS[ofmt][0]
        key = _h("blend", list(filters), list(settings), pix, w, h, np.ascontiguousarray(frames), opix, loc,
                 [(o[0], o[1], o[2], o[3], o[4], _h(o[5])) for o in overlays], list(changed or []), tuple(guard))
        kw = dict(chroma_location=loc, changed=changed, guard=guard)
        if self.recording:
            r, _ = self.lib.run_blend("hb_blend", overlays, opix, filters, settings, frames, pix, w, h, **kw)
            self.store[key] = RecordedResult.record(r) if digest_only else result_digest(r)
            self._save()
            return RecordedResult(self.store[key]) if digest_only else r
        want = self.store.get(key)
        if want is None:
            raise KeyError(f"no stored reference result for blend call {filters} {fmt} {w}x{h} ({key}): "
                           "record it with HBCU_RECORD_REF=1 where the reference is built")
        if digest_only:
            return RecordedResult(want)
        names = [f if f == RENDER_SUB else f + "_cuda" for f in filters]
        r, _ = self.host.run_blend("hb_blend_cuda", overlays, opix, names, settings, frames, pix, w, h, **kw)
        assert result_digest(r) == want, f"the CPU restatement of the blend call {filters} {fmt} {w}x{h} no longer reproduces the reference's result"
        return r

    def chroma_coeffs(self):
        """the reference's hb_compute_chroma_smoothing_coefficient for every frame format's subsampling and location"""
        if self.recording:
            self.store["chroma_coeffs"] = coeff_table(self.lib.lib)
            self._save()
        return self.store["chroma_coeffs"]


def coeff_table(lib):
    fn = lib.hb_compute_chroma_smoothing_coefficient
    fn.argtypes = [C.c_void_p, C.c_int, C.c_int]
    out = {}
    for fmt in ("420p", "422p", "444p"):
        for loc in range(7):
            c = (C.c_uint32 * 8)()
            fn(C.addressof(c), FRAME_FMTS[fmt][0], loc)
            out[f"{fmt}-{loc}"] = list(c)
    return out


@pytest.fixture(scope="module")
def bref():
    return BlendRef()


def assert_same(r, g):
    assert g.saw_eof and r.saw_eof
    assert g.frames.shape == r.frames.shape, (g.frames.shape, r.frames.shape)
    assert np.array_equal(g.start, r.start)
    if not np.array_equal(g.frames, r.frames):
        d = g.frames != r.frames
        raise AssertionError(f"{np.count_nonzero(d)} bytes differ in frames {np.argwhere(d.any(axis=1)).ravel()[:8]}")


def core():
    lib = C.CDLL(str(LIBHBCU))
    lib.hbcu_kernel_launches.restype = C.c_uint64
    lib.hbcu_blend_uploads.restype = C.c_uint64
    lib.hbcu_frames_alive.restype = C.c_long
    return lib


CHANGED = [1, 0, 0, 1, 0]


def changed_inputs():
    w, h, fmt, ofmt = 160, 90, "420p10", "yuva444p"
    frames = make_frames(fmt, w, h, len(CHANGED), seed=5)
    ov = overlays_of([(f, 10, 50, 120, 30, "glyph") for f in range(len(CHANGED))], ofmt, seed=9)
    # the renderer's list is the same subtitle while changed == 0: the same planes
    for f in range(1, len(CHANGED)):
        if not CHANGED[f]:
            ov[f] = (f,) + ov[f - 1][1:]
    return w, h, fmt, ofmt, frames, ov


CHAIN_SETTINGS = ["y-strength=6", None, "y-strength=0.2:y-kernel=isolap"]


def chain_inputs():
    w, h, fmt, ofmt = 1920, 1080, "420p10", "yuva444p"
    frames = make_frames(fmt, w, h, 3, seed=77)
    spec = [(f, 160 + 4 * f, 900, 1600, 120, "glyph") for f in range(3)] + [(f, 161, 50 - f, 1600, 120, "noise") for f in range(3)]
    spec.sort(key=lambda o: o[0])
    return w, h, fmt, ofmt, frames, overlays_of(spec, ofmt, seed=3)


def ref_chain(bref):
    w, h, fmt, ofmt, frames, ov = chain_inputs()
    return bref.run_blend(ov, ofmt, ["hb_filter_nlmeans", RENDER_SUB, "hb_filter_lapsharp"],
                          [CHAIN_SETTINGS[0] + ":threads=2", None, CHAIN_SETTINGS[2]], frames, fmt, w, h, digest_only=True)


# ---------------------------------------------------------------------------------------------------------- CPU tests
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_restatement_reproduces_reference(bref, case):
    c = case
    frames = make_frames(c["fmt"], c["w"], c["h"], c["n"], seed=c["w"] + c["n"])
    r = bref.run_blend(case_overlays(c), c["ofmt"], [RENDER_SUB], [None], frames, c["fmt"], c["w"], c["h"], loc=c["loc"],
                       guard=c["guard"])
    assert r.frames.shape[0] == c["n"]


def test_restatement_changed_sequence(bref):
    """the host object over the restatement uploads a list only when it changed, and still matches the reference"""
    w, h, fmt, ofmt, frames, ov = changed_inputs()
    before = C.CDLL(str(bref.host.path)).oracle_hbcu_blend_uploads
    before.restype = C.c_uint64
    n0 = before()
    bref.run_blend(ov, ofmt, [RENDER_SUB], [None], frames, fmt, w, h, changed=CHANGED)
    if not bref.recording:
        assert before() - n0 == sum(CHANGED)


def test_reference_chain_recorded(bref):
    """the 1080p device-chain reference (NLMeans, blend, lapsharp) is stored; the GPU test compares with it"""
    r = ref_chain(bref)
    assert r.shape[0] == 3 and r.saw_eof


def test_chroma_coefficients_match_reference(bref):
    want = bref.chroma_coeffs()
    assert coeff_table(bref.host.lib) == want


def test_blend_cuda_exported_and_refused_without_gpu():
    flt = handbrake_b200.filters()
    assert flt.filter_object("hb_blend_cuda")
    if core().hbcu_device_count() > 0:
        return
    w, h = 64, 48
    frames = make_frames("420p", w, h, 2, seed=1)
    ov = overlays_of([(0, 3, 4, 20, 10, "full")], "yuva444p", seed=1)
    r, st = flt.run_blend("hb_blend_cuda", ov, OVERLAY_FMTS["yuva444p"][0], [RENDER_SUB], [None], frames, 0, w, h)
    assert r.init_failed == 1 and np.array_equal(r.frames, frames) and st["frames"] == 0


@pytest.mark.parametrize("fmt,ofmt", [("444p", "yuva420p"), ("420p", "yuva422p"), ("422p", "yuva420p"), ("444p10", "yuva422p")])
def test_unsupported_combinations_refused(bref, fmt, ofmt):
    w, h = 64, 48
    frames = make_frames(fmt, w, h, 2, seed=2)
    ov = overlays_of([(0, 3, 4, 20, 10, "full")], ofmt, seed=2)
    r, _ = bref.host.run_blend("hb_blend_cuda", ov, OVERLAY_FMTS[ofmt][0], [RENDER_SUB], [None], frames, FRAME_FMTS[fmt][0], w, h)
    assert r.init_failed == 1 and np.array_equal(r.frames, frames)


def test_restatement_zero_overlays_return_the_input(bref):
    w, h = 64, 48
    frames = make_frames("420p", w, h, 3, seed=3)
    r, st = bref.host.run_blend("hb_blend_cuda", [], OVERLAY_FMTS["yuva444p"][0], [RENDER_SUB], [None], frames, 0, w, h)
    assert np.array_equal(r.frames, frames) and st["same_buffer"] == 3
    r, st = bref.host.run_blend("hb_blend_cuda", [], OVERLAY_FMTS["yuva444p"][0], [UP, RENDER_SUB, DOWN], [None] * 3, frames, 0, w, h)
    assert np.array_equal(r.frames, frames) and st["same_buffer"] == 3


# ---------------------------------------------------------------------------------------------------------- GPU tests
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_blend_matches_reference(bref, cuda_filters, case):
    c = case
    frames = make_frames(c["fmt"], c["w"], c["h"], c["n"], seed=c["w"] + c["n"])
    ov = case_overlays(c)
    r = bref.run_blend(ov, c["ofmt"], [RENDER_SUB], [None], frames, c["fmt"], c["w"], c["h"], loc=c["loc"], guard=c["guard"])
    pix, opix = FRAME_FMTS[c["fmt"]][0], OVERLAY_FMTS[c["ofmt"]][0]
    g, st = cuda_filters.run_blend("hb_blend_cuda", ov, opix, [RENDER_SUB], [None], frames, pix, c["w"], c["h"],
                                   chroma_location=c["loc"], guard=c["guard"])
    assert g.init_failed == 0
    assert_same(r, g)
    assert st["guard_damaged"] == 0, "the CUDA blend wrote outside the picture"
    # the same frames as device frames: a new device frame per frame, the same result
    d, _ = cuda_filters.run_blend("hb_blend_cuda", ov, opix, [UP, RENDER_SUB, DOWN], [None] * 3, frames, pix, c["w"], c["h"],
                                  chroma_location=c["loc"])
    assert_same(r, d)
    assert core().hbcu_frames_alive() == 0 and cuda_filters.buffers_alive() == 0


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_unchanged_overlays_are_not_uploaded_again(bref, cuda_filters, device):
    w, h, fmt, ofmt, frames, ov = changed_inputs()
    r = bref.run_blend(ov, ofmt, [RENDER_SUB], [None], frames, fmt, w, h, changed=CHANGED)
    lib = core()
    n0 = lib.hbcu_blend_uploads()
    chain = [UP, RENDER_SUB, DOWN] if device else [RENDER_SUB]
    g, _ = cuda_filters.run_blend("hb_blend_cuda", ov, OVERLAY_FMTS[ofmt][0], chain, [None] * len(chain), frames,
                                  FRAME_FMTS[fmt][0], w, h, changed=CHANGED)
    assert lib.hbcu_blend_uploads() - n0 == sum(CHANGED)
    assert_same(r, g)


@pytest.mark.gpu
def test_zero_overlays_no_gpu_work(cuda_filters):
    w, h = 160, 90
    frames = make_frames("420p10", w, h, 4, seed=4)
    lib = core()
    k0 = lib.hbcu_kernel_launches()
    g, st = cuda_filters.run_blend("hb_blend_cuda", [], OVERLAY_FMTS["yuva444p"][0], [RENDER_SUB], [None], frames, 62, w, h)
    assert lib.hbcu_kernel_launches() == k0
    assert st["same_buffer"] == 4 and np.array_equal(g.frames, frames)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_launches_do_not_depend_on_overlay_count(cuda_filters, device):
    w, h, n = 320, 180, 3
    frames = make_frames("420p", w, h, n, seed=6)
    lib = core()
    chain = [UP, RENDER_SUB, DOWN] if device else [RENDER_SUB]
    counts = []
    for per_frame in (1, 12):
        spec = [(f, 7 + 19 * i, 5 + 11 * i, 40, 24, "glyph") for f in range(n) for i in range(per_frame)]
        k0 = lib.hbcu_kernel_launches()
        cuda_filters.run_blend("hb_blend_cuda", overlays_of(spec, "yuva444p", seed=per_frame), OVERLAY_FMTS["yuva444p"][0],
                               chain, [None] * len(chain), frames, 0, w, h)
        counts.append(lib.hbcu_kernel_launches() - k0)
    if device:
        assert counts[0] == counts[1]
    else:
        assert counts == [n, n]


@pytest.mark.gpu
def test_1080p10_device_chain(bref, cuda_filters):
    """upload -> NLMeans -> blend -> lapsharp -> download, frames in HBM throughout, against the reference's
    NLMeans -> hb_blend -> lapsharp on host frames"""
    w, h, fmt, ofmt, frames, ov = chain_inputs()
    want = ref_chain(bref)
    names = [UP, "hb_filter_nlmeans_cuda", RENDER_SUB, "hb_filter_lapsharp_cuda", DOWN]
    g, _ = cuda_filters.run_blend("hb_blend_cuda", ov, OVERLAY_FMTS[ofmt][0], names, [None] + CHAIN_SETTINGS + [None], frames,
                                  FRAME_FMTS[fmt][0], w, h)
    assert g.init_failed == 0 and g.frames.shape == want.shape
    assert np.array_equal(g.start, want.start)
    bad = want.frames_differing(g.frames)
    assert not bad, f"frames {bad} differ from the reference chain"
    assert core().hbcu_frames_alive() == 0 and cuda_filters.buffers_alive() == 0
