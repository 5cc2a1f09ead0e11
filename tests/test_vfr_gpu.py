"""hb_filter_vfr_cuda, the CUDA twin of libhb's framerate shaper (vfr.c) and its motion metric (motion_metric.c).

Two tables of the reference's results, stored in tests/golden/vfr_ref_digests.json:
  - metrics: the float bits hb_motion_metric returns for pairs of frames at 8, 10 and 12 bits, on sizes either side of the
    fast path's 1920 / 1080 bound (each bound alone), at 4K and at sizes that are not multiples of 16 or 64, with padded
    pitches; identical frames, small noise, full-scale black / white cuts (whose 16x16 block sums wrap in uint32) and the
    largest sample value (the gamma table's top entry);
  - shaper cases: every output of hb_filter_vfr (frame digest, start, stop, new_chap) plus the vrate / cfr init() leaves
    and the info() text, for modes 0 / 1 / 2, the usual rate conversions, telecine-like repeats, ties, input gaps,
    non-monotonic stops, a chapter mark on a duplicated frame, short clips (the EOF flush) and 4:2:0 / 4:2:2 / 4:4:4.
On a machine without a GPU the shaper over the plain-C restatement of the metric (oracle/_ref/libhostlogic_vfr.so) must
reproduce each shaper case, and a numpy restatement of the metric each metric.  `HBCU_RECORD_REF=1` with the reference's
vfr built (oracle/vfr.mk, oracle/_ref/libhbref_vfr.so) re-records them through the CPU tests."""
import ctypes as C
import json
import math
from pathlib import Path

import numpy as np
import pytest

import handbrake_b200
from golden_ref import GoldenRef, _h, frame_digests
from handbrake_b200 import LIBHBCU

STORE = Path(__file__).resolve().parent / "golden" / "vfr_ref_digests.json"
REPO = Path(__file__).resolve().parent.parent
REF_VFR_SO = REPO / "oracle" / "_ref" / "libhbref_vfr.so"
HOSTLOGIC_VFR_SO = REPO / "oracle" / "_ref" / "libhostlogic_vfr.so"
UP, DOWN = "hb_filter_hbcu_upload", "hb_filter_hbcu_download"

# the shim's enum AVPixelFormat: (pix_fmt, depth, chroma shift w, chroma shift h)
FMTS = {"420p": (0, 8, 1, 1), "420p10": (62, 10, 1, 1), "420p12": (123, 12, 1, 1), "420p16": (47, 16, 1, 1),
        "422p": (4, 8, 1, 0), "422p10": (64, 10, 1, 0), "444p": (5, 8, 0, 0), "444p10": (68, 10, 0, 0)}


# ---------------------------------------------------------------------------------------------------------- content
def luma(kind, depth, w, h, rng, base=None):
    maxv = (1 << depth) - 1
    if kind == "black":
        return np.zeros((h, w), np.int64)
    if kind == "white":
        return np.full((h, w), maxv, np.int64)
    if kind == "checker":            # full-scale 16x16 checkerboard: every block of a black / white cut wraps
        yy, xx = np.mgrid[0:h, 0:w]
        return np.where(((yy // 16) + (xx // 16)) % 2 == 0, maxv, 0).astype(np.int64)
    if kind == "max":
        return np.where(rng.random((h, w)) < 0.5, maxv, maxv - 1 - rng.integers(0, 3, (h, w))).astype(np.int64)
    if kind == "scene":              # smooth gradients plus texture
        yy, xx = np.mgrid[0:h, 0:w]
        ph = rng.random() * 6.28
        v = (np.sin(xx / (7 + 20 * rng.random()) + ph) + np.cos(yy / (5 + 15 * rng.random()) - ph)) * 0.22 + 0.5
        return np.clip(v * maxv + rng.integers(-(maxv // 32), maxv // 32 + 1, (h, w)), 0, maxv).astype(np.int64)
    if kind == "jitter":             # base with small noise
        return np.clip(base + rng.integers(-(maxv // 128) - 1, maxv // 128 + 2, base.shape), 0, maxv).astype(np.int64)
    raise ValueError(kind)


def pack(fmt, y, rng):
    """a packed planar frame (luma y, random chroma)"""
    _, depth, sw, sh = FMTS[fmt]
    h, w = y.shape
    cw, ch = -((-w) >> sw), -((-h) >> sh)
    dt = np.uint8 if depth == 8 else np.uint16
    parts = [y.astype(dt).ravel(), rng.integers(0, 1 << depth, 2 * cw * ch).astype(dt)]
    return np.concatenate(parts).view(np.uint8)


def luma_of(fmt, frame, w, h):
    depth = FMTS[fmt][1]
    bps = 1 if depth == 8 else 2
    raw = frame[: w * h * bps]
    return (raw if bps == 1 else raw.view(np.uint16)).reshape(h, w).astype(np.int64)


# ---------------------------------------------------------------------------------------------------------- metric
def gamma_lut(depth):
    """motion_metric.c build_gamma_lut: 4095 * pow((float)i / (float)(max - 1), 2.2f), truncated"""
    maxv = (1 << depth) - 1
    den, e = np.float32(maxv - 1), float(np.float32(2.2))
    return np.array([int(4095 * math.pow(float(np.float32(i) / den), e)) for i in range(maxv + 1)], dtype=np.int64)


def reduce4(x):
    h4, w4 = x.shape[0] // 4, x.shape[1] // 4
    s = x[: h4 * 4, : w4 * 4].reshape(h4, 4, w4, 4)

    def ap(a, b, c, d):
        return (((a + b + 1) >> 1) + ((c + d + 1) >> 1) + 1) >> 1
    return ap(ap(s[:, 0, :, 0], s[:, 1, :, 0], s[:, 0, :, 1], s[:, 1, :, 1]),
              ap(s[:, 0, :, 2], s[:, 1, :, 2], s[:, 0, :, 3], s[:, 1, :, 3]),
              ap(s[:, 2, :, 0], s[:, 3, :, 0], s[:, 2, :, 1], s[:, 3, :, 1]),
              ap(s[:, 2, :, 2], s[:, 3, :, 2], s[:, 2, :, 3], s[:, 3, :, 3]))


def is_fast(w, h):
    return w >= 1920 or h >= 1080


def metric_sum(a, b, depth, fast):
    """the uint64 sum of the x86 motion metric: per 16x16 block a wrapping uint32, whole blocks only"""
    lut = gamma_lut(depth)
    if fast:
        a, b = reduce4(a), reduce4(b)
        if depth > 8:
            # the reduced images are packed, and above 8 bits the reference walks them with half the pitch
            h4, w4 = a.shape
            yy, xx = np.mgrid[0:(h4 // 16) * 16, 0:(w4 // 16) * 16]
            idx = yy * (w4 // 2) + xx
            a, b = a.ravel()[idx], b.ravel()[idx]
    bh, bw = a.shape[0] // 16, a.shape[1] // 16
    d = lut[a[: bh * 16, : bw * 16]] - lut[b[: bh * 16, : bw * 16]]
    return int(((d * d).reshape(bh, 16, bw, 16).sum(axis=(1, 3)) & 0xFFFFFFFF).sum())


def metric_bits(s, w, h, fast):
    """(float)sum / (width * height) on the (reduced) geometry, as float32 bits"""
    if fast:
        w, h = w // 4, h // 4
    return int(np.array([np.float32(np.float32(s) / np.float32(w * h))], np.float32).view(np.uint32)[0])


METRIC_SIZES = [(1918, 1078), (1920, 1078), (1918, 1080), (3840, 2160), (333, 211), (200, 120), (1000, 700)]


def build_metric_cases():
    cases = []
    for w, h in METRIC_SIZES:
        for fmt in ("420p", "420p10", "420p12"):
            if (w, h) == (3840, 2160) and fmt == "420p12":
                continue
            for kind in ("same", "noise", "cut", "max", "scene"):
                cases.append(dict(id=f"{fmt}-{w}x{h}-{kind}", fmt=fmt, w=w, h=h, kind=kind, pad=0))
    for fmt, pad in (("420p", 64), ("420p10", 40), ("420p", 7)):
        for w, h in ((333, 211), (1920, 1080)):
            cases.append(dict(id=f"{fmt}-{w}x{h}-pad{pad}", fmt=fmt, w=w, h=h, kind="noise", pad=pad))
    return cases


METRIC_CASES = build_metric_cases()


def metric_pair(c):
    depth = FMTS[c["fmt"]][1]
    rng = np.random.default_rng(len(c["id"]) * 1009 + c["w"] + c["h"])
    kind = c["kind"]
    if kind == "cut":
        return luma("checker", depth, c["w"], c["h"], rng), luma("black", depth, c["w"], c["h"], rng)
    if kind == "max":
        return luma("max", depth, c["w"], c["h"], rng), luma("black", depth, c["w"], c["h"], rng)
    a = luma("scene", depth, c["w"], c["h"], rng)
    if kind == "same":
        return a, a.copy()
    if kind == "noise":
        return a, luma("jitter", depth, c["w"], c["h"], rng, base=a)
    return a, luma("scene", depth, c["w"], c["h"], rng)


def luma_bytes(fmt, y):
    return np.ascontiguousarray(y.astype(np.uint8 if FMTS[fmt][1] == 8 else np.uint16)).view(np.uint8).ravel()


# ---------------------------------------------------------------------------------------------------------- shaper
def analysis_depth(in_rate, out_rate):
    """vfr.c hb_vfr_init: frame_analysis_depth"""
    depth = 2
    if in_rate > out_rate:
        f = in_rate / out_rate
        if 1.0 < f < 2.0:
            f = 1 / (f - 1)
        depth = min(math.ceil(f) + 1, 10)
    return depth


def timestamps(n, rate, gaps=(), backs=()):
    """frame i from floor(i * 90000 / rate); a gap index skips one frame's time, a back index ends before its
    predecessor"""
    t = [int(i * 90000 * rate[1] // rate[0]) for i in range(n + len(gaps) + 1)]
    start, stop, k = [], [], 0
    for i in range(n):
        if i in gaps:
            k += 1
        start.append(t[k])
        stop.append(t[k + 1])
        k += 1
    for i in backs:
        start[i], stop[i] = start[i - 1] - 10, stop[i - 1] - 5
    return np.array(start, np.int64), np.array(stop, np.int64)


def shaper_clip(fmt, w, h, n, content, seed):
    """content: 'distinct' frames; 'telecine' (new frames followed by repeats with slight noise, 3:2 then 2:3:3 from the
    middle); 'ties' (exact repeats of a 2:2 pattern: equal metrics); 'static' (every frame the same)"""
    depth = FMTS[fmt][1]
    rng = np.random.default_rng(seed)
    frames, base = [], None
    if content == "telecine":
        pattern = [3, 2] * 40
        half = [2, 3, 3] * 40
        reps = []
        for r in pattern:
            reps += [True] + [False] * (r - 1)
            if len(reps) >= n // 2:
                break
        while len(reps) < n:
            r = half[len(reps) % 3]
            reps += [True] + [False] * (r - 1)
    elif content == "ties":
        reps = [i % 2 == 0 for i in range(n)]
    elif content == "static":
        reps = [i == 0 for i in range(n)]
    else:
        reps = [True] * n
    for i in range(n):
        if reps[i] or base is None:
            base = luma("scene", depth, w, h, rng)
            y = base
        else:
            y = base if content in ("ties", "static") else luma("jitter", depth, w, h, rng, base=base)
        frames.append(pack(fmt, y, np.random.default_rng(seed + i if content not in ("ties", "static") else seed)))
    return np.stack(frames)


NTSC, FILM, PAL = (30000, 1001), (24000, 1001), (25, 1)


def build_shaper_cases():
    cs = []

    def add(id, settings, n=36, rate=NTSC, fmt="420p", w=64, h=48, content="telecine", cfr=0, gaps=(), backs=(), chap=None):
        cs.append(dict(id=id, settings=settings, n=n, rate=rate, fmt=fmt, w=w, h=h, content=content, cfr=cfr,
                       gaps=tuple(gaps), backs=tuple(backs), chap=chap))

    add("mode0", "mode=0")
    add("mode0-rate", "mode=0:rate=24000/1001")
    add("init-cfr1", None, cfr=1)
    add("init-cfr2-rate", "rate=24000/1001", cfr=2)
    add("cfr-2997-23976", "mode=1:rate=24000/1001")
    add("cfr-2997-23976-shift", "mode=1:rate=24000/1001", n=60)
    add("cfr-5994-23976", "mode=1:rate=24000/1001", rate=(60000, 1001), n=40)
    add("cfr-120-24", "mode=1:rate=24/1", rate=(120, 1), n=48, content="distinct")
    add("cfr-25-24", "mode=1:rate=24/1", rate=PAL, n=60, content="distinct")
    add("cfr-240-24", "mode=1:rate=24/1", rate=(240, 1), n=60, content="distinct")
    add("pfr-23976-30", "mode=2:rate=30/1", rate=FILM, n=30, content="distinct")
    add("pfr-2997-23976", "mode=2:rate=24000/1001")
    add("pfr-5994-30", "mode=2:rate=30/1", rate=(60000, 1001), n=40)
    add("cfr-up-23976-2997", "mode=1:rate=30000/1001", rate=FILM, n=20, content="distinct",
        chap=[0, 0, 0, 0, 0, 7, 0, 0, 0, 0, 0, 0, 0, 9, 0, 0, 0, 0, 0, 0])
    add("cfr-ties", "mode=1:rate=24000/1001", content="ties")
    add("cfr-static", "mode=1:rate=24000/1001", content="static", n=20)
    add("cfr-gaps", "mode=1:rate=24000/1001", n=40, gaps=(6, 7, 20, 31))
    add("mode0-gaps", "mode=0", n=24, gaps=(5, 12))
    add("cfr-backwards", "mode=1:rate=24000/1001", n=30, backs=(9, 17))
    add("pfr-backwards-gaps", "mode=2:rate=30/1", rate=FILM, n=30, gaps=(4,), backs=(15,), content="distinct")
    for n in (1, 2, 3, 4, 5, 7):        # depth 6 at 29.97 -> 23.976 (see below): 5 and 7 are depth -/+ 1
        add(f"cfr-eof-{n}", "mode=1:rate=24000/1001", n=n)
    for n in (1, 2, 3):
        add(f"pfr-eof-{n}", "mode=2:rate=30/1", rate=FILM, n=n, content="distinct")
    for fmt in ("422p", "444p", "420p10", "422p10", "444p10", "420p12", "420p16"):
        add(f"cfr-{fmt}", "mode=1:rate=24000/1001", fmt=fmt, n=24)
    add("cfr-odd-size", "mode=1:rate=24000/1001", w=333, h=211, n=24)
    add("cfr-1080p-fast", "mode=1:rate=24000/1001", w=1920, h=1080, n=16)
    return cs


SHAPER_CASES = build_shaper_cases()
SHAPER_4K = [dict(id=f"cfr-4k-{fmt}", settings="mode=1:rate=24000/1001", n=12, rate=NTSC, fmt=fmt, w=3840, h=2160,
                  content="telecine", cfr=0, gaps=(), backs=(), chap=None) for fmt in ("420p", "420p10")]


def shaper_inputs(c):
    frames = shaper_clip(c["fmt"], c["w"], c["h"], c["n"], c["content"], seed=len(c["id"]) * 31 + c["n"])
    start, stop = timestamps(c["n"], c["rate"], c["gaps"], c["backs"])
    chap = np.array(c["chap"] if c["chap"] is not None else range(c["n"]), np.int32)
    return frames, start, stop, chap


def shaper_record(r):
    return dict(n=int(r.frames.shape[0]), d=_h(frame_digests(r.frames), [int(v) for v in r.start], [int(v) for v in r.stop],
                                              [int(v) for v in r.new_chap], tuple(r.vrate), int(r.cfr), r.info,
                                              bool(r.saw_eof), int(r.init_failed)))


# ---------------------------------------------------------------------------------------------------------- reference
class VfrRef(GoldenRef):
    """GoldenRef over this file's own store: the reference's vfr and motion metric (oracle/_ref/libhbref_vfr.so)"""

    def __init__(self):
        from handbrake_b200.hblib import FilterLib
        super().__init__()
        self.store = json.loads(STORE.read_text()) if STORE.exists() else {}
        if self.recording:
            self.lib = FilterLib(REF_VFR_SO)
        self.host = FilterLib(HOSTLOGIC_VFR_SO)

    def _save(self):
        STORE.write_text(json.dumps(dict(sorted(self.store.items())), indent=0) + "\n")

    def _get(self, key, what):
        if self.recording:
            return None
        if key not in self.store:
            raise KeyError(f"no stored reference result for {what} ({key}): record it with HBCU_RECORD_REF=1 where the "
                           "reference is built")
        return self.store[key]

    def metric(self, c, a, b):
        """the reference's hb_motion_metric on luma a, b: float32 bits"""
        key = _h("metric", c["fmt"], c["w"], c["h"], c["pad"], luma_bytes(c["fmt"], a), luma_bytes(c["fmt"], b))
        want = self._get(key, f"metric {c['id']}")
        if want is not None:
            return want
        fn = self.lib.lib.hb_harness_motion_metric
        fn.restype = C.c_float
        fn.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        la, lb = luma_bytes(c["fmt"], a), luma_bytes(c["fmt"], b)
        v = fn(self.lib.filter_object("hb_motion_metric"), FMTS[c["fmt"]][0], c["w"], c["h"], c["pad"], la.ctypes.data, lb.ctypes.data)
        self.store[key] = int(np.array([v], np.float32).view(np.uint32)[0])
        self._save()
        return self.store[key]

    def shaper(self, c):
        """the reference's vfr on the case's clip: its stored record"""
        frames, start, stop, chap = shaper_inputs(c)
        key = _h("vfr", c["settings"], FMTS[c["fmt"]][0], c["w"], c["h"], frames, start, stop, chap, c["rate"], c["cfr"])
        want = self._get(key, f"vfr case {c['id']}")
        if want is not None:
            return want
        r = self.lib.run("hb_filter_vfr", c["settings"], frames, FMTS[c["fmt"]][0], c["w"], c["h"], **run_kw(c, start, stop, chap))
        self.store[key] = shaper_record(r)
        self._save()
        return self.store[key]

    def template_digest(self):
        key = "template:hb_filter_vfr"
        if self.recording:
            class Head(C.Structure):
                _fields_ = [("pad", C.c_byte * 96), ("settings_template", C.c_char_p)]
            self.store[key] = _h(Head.in_dll(self.lib.lib, "hb_filter_vfr").settings_template.decode())
            self._save()
        return self.store[key]


def run_kw(c, start, stop, chap):
    return dict(start=start, stop=stop, new_chap=chap, vrate=c["rate"], cfr=c["cfr"], info=True)


@pytest.fixture(scope="module")
def vref():
    return VfrRef()


def core():
    lib = C.CDLL(str(LIBHBCU))
    lib.hbcu_motion_metric_waits.restype = C.c_uint64
    lib.hbcu_motion_metric_launches.restype = C.c_uint64
    lib.hbcu_frames_alive.restype = C.c_long
    lib.hbcu_last_error.restype = C.c_char_p
    lib.hbcu_motion_metric_create.argtypes = [C.c_void_p, C.c_void_p]
    lib.hbcu_motion_metric_enqueue.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    lib.hbcu_motion_metric_result.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    lib.hbcu_motion_metric_destroy.argtypes = [C.c_void_p]
    lib.hbcu_frame_release.argtypes = [C.c_void_p]
    return lib


def run_product(lib, c, chain):
    frames, start, stop, chap = shaper_inputs(c)
    sets = [c["settings"] if f.startswith("hb_filter_vfr") else None for f in chain]
    return lib.run(chain, sets, frames, FMTS[c["fmt"]][0], c["w"], c["h"], **run_kw(c, start, stop, chap))


# ---------------------------------------------------------------------------------------------------------- CPU tests
@pytest.mark.parametrize("case", METRIC_CASES, ids=[c["id"] for c in METRIC_CASES])
def test_metric_restatement_reproduces_reference(vref, case):
    a, b = metric_pair(case)
    want = vref.metric(case, a, b)
    depth, fast = FMTS[case["fmt"]][1], is_fast(case["w"], case["h"])
    assert metric_bits(metric_sum(a, b, depth, fast), case["w"], case["h"], fast) == want
    if case["kind"] == "same":
        assert want == 0


def test_block_sums_wrap_in_the_cut_cases():
    """a full-scale 16x16 block exceeds 2^32 at every depth: the cut cases exercise the reference's wrap"""
    for depth in (8, 10, 12):
        lut = gamma_lut(depth)
        assert 256 * int(lut[-1]) ** 2 > 2 ** 32
    assert [gamma_lut(d)[-1] for d in (8, 10, 12)] == [4130, 4103, 4097]


@pytest.mark.parametrize("case", SHAPER_CASES + SHAPER_4K, ids=[c["id"] for c in SHAPER_CASES + SHAPER_4K])
def test_shaper_restatement_reproduces_reference(vref, case):
    want = vref.shaper(case)
    if vref.recording:
        return
    r = run_product(vref.host, case, ["hb_filter_vfr_cuda"])
    assert shaper_record(r) == want, f"the CPU restatement no longer reproduces the reference's vfr for {case['id']}"


def test_analysis_depth_restatement():
    """29.97 / 23.976 is 1.25 exactly, but in doubles 1 / (factor - 1) comes out just above 4: depth 6, not 5"""
    assert [analysis_depth(a[0] / a[1], b[0] / b[1]) for a, b in
            ((NTSC, FILM), ((60000, 1001), FILM), ((120, 1), (24, 1)), (PAL, (24, 1)), ((240, 1), (24, 1)), (FILM, (30, 1)))] \
        == [6, 4, 6, 10, 10, 2]


def test_vfr_cuda_exported_with_reference_id_and_template(vref):
    flt = handbrake_b200.filters()

    class FilterObject(C.Structure):
        _fields_ = [("id", C.c_int), ("enforce_order", C.c_int), ("skip", C.c_int), ("aliased", C.c_int),
                    ("name", C.c_char_p), ("short_name", C.c_char_p), ("settings", C.c_void_p),
                    ("init", C.c_void_p), ("init_thread", C.c_void_p), ("post_init", C.c_void_p),
                    ("work", C.c_void_p), ("work_thread", C.c_void_p), ("close", C.c_void_p), ("info", C.c_void_p),
                    ("settings_template", C.c_char_p)]
    obj = FilterObject.in_dll(flt.lib, "hb_filter_vfr_cuda")
    assert obj.id == 11 and obj.short_name == b"vfr" and obj.enforce_order == 1 and obj.info
    assert _h(obj.settings_template.decode()) == vref.template_digest()
    flt.lib.hb_filter_get.restype = C.c_void_p
    assert flt.lib.hb_filter_get(11) == flt.filter_object("hb_filter_vfr_cuda")


def test_without_gpu_modes_1_2_refused_mode_0_matches(vref):
    if core().hbcu_device_count() > 0:
        pytest.skip("a GPU is present")
    flt = handbrake_b200.filters()
    by_id = {c["id"]: c for c in SHAPER_CASES}
    for cid in ("cfr-2997-23976", "pfr-23976-30", "init-cfr1"):
        r = run_product(flt, by_id[cid], ["hb_filter_vfr_cuda"])
        assert r.init_failed == 1 and r.frames.shape[0] == by_id[cid]["n"]
    for cid in ("mode0", "mode0-rate", "mode0-gaps"):
        assert shaper_record(run_product(flt, by_id[cid], ["hb_filter_vfr_cuda"])) == vref.shaper(by_id[cid])


# ---------------------------------------------------------------------------------------------------------- GPU tests
class MMConfig(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("depth", C.c_int), ("fast", C.c_int), ("device", C.c_int),
                ("slots", C.c_int), ("results", C.c_int), ("gamma_lut", C.c_void_p)]


def cuda_metric(lib, c, a, b, device_frames):
    """the CUDA handle's metric of b against a: host luma (with the case's padding) or torch-owned pitched device
    memory wrapped as frames"""
    depth, fast = FMTS[c["fmt"]][1], is_fast(c["w"], c["h"])
    w, h = c["w"], c["h"]
    lut = np.ascontiguousarray(gamma_lut(depth).astype(np.uint32))
    cfg = MMConfig(w, h, depth, int(fast), 0, 4, 2, lut.ctypes.data)
    hdl = C.c_void_p()
    assert lib.hbcu_motion_metric_create(C.byref(hdl), C.byref(cfg)) == 0, lib.hbcu_last_error()
    keep = []
    try:
        for slot, y in ((0, a), (1, b)):
            raw = luma_bytes(c["fmt"], y).reshape(h, -1)
            row = raw.shape[1]
            if device_frames:
                import torch
                pitch = (row + c["pad"] + 255) // 256 * 256
                t = torch.zeros((h + 2) * pitch, dtype=torch.uint8, device="cuda")
                t[: h * pitch].view(h, pitch)[:, :row] = torch.from_numpy(np.ascontiguousarray(raw)).cuda()
                torch.cuda.synchronize()
                f = C.c_void_p()
                planes = (C.c_void_p * 3)(t.data_ptr(), t.data_ptr(), t.data_ptr())
                rb, rows, st = (C.c_int * 3)(row, row // 2, row // 2), (C.c_int * 3)(h, h // 2, h // 2), (C.c_int * 3)(pitch, pitch, pitch)
                assert lib.hbcu_frame_wrap(C.byref(f), 0, planes, rb, rows, st, C.c_size_t(2 * pitch), None, None, None) == 0, lib.hbcu_last_error()
                keep += [t, f]
                rc = lib.hbcu_motion_metric_enqueue(hdl, slot, slot - 1, 0, f, None, 0)
            else:
                host = np.zeros((h, row + c["pad"]), np.uint8)
                host[:, :row] = raw
                rc = lib.hbcu_motion_metric_enqueue(hdl, slot, slot - 1, 0, None, host.ctypes.data, row + c["pad"])
                del host                                         # copied before the call returned
            assert rc == 0, lib.hbcu_last_error()
        s = C.c_uint64()
        assert lib.hbcu_motion_metric_result(hdl, 0, C.byref(s)) == 0, lib.hbcu_last_error()
    finally:
        lib.hbcu_motion_metric_destroy(hdl)
        for k in keep:
            if isinstance(k, C.c_void_p):
                lib.hbcu_frame_release(k)
    return metric_bits(s.value, w, h, fast)


@pytest.mark.gpu
@pytest.mark.parametrize("device_frames", [False, True], ids=["host", "device"])
def test_cuda_metric_matches_reference(vref, cuda_filters, device_frames):
    lib = core()
    bad = []
    for c in METRIC_CASES:
        a, b = metric_pair(c)
        want = vref.metric(c, a, b)
        got = cuda_metric(lib, c, a, b, device_frames)
        if got != want:
            bad.append((c["id"], hex(got), hex(want)))
    assert not bad, bad
    assert lib.hbcu_frames_alive() == 0


@pytest.mark.gpu
@pytest.mark.parametrize("case", SHAPER_CASES + SHAPER_4K, ids=[c["id"] for c in SHAPER_CASES + SHAPER_4K])
def test_vfr_cuda_matches_reference(vref, cuda_filters, case):
    want = vref.shaper(case)
    g = run_product(cuda_filters, case, ["hb_filter_vfr_cuda"])
    assert g.init_failed == 0 and shaper_record(g) == want
    alive = cuda_filters.buffers_alive()
    d = run_product(cuda_filters, case, [UP, "hb_filter_vfr_cuda", DOWN])
    assert d.init_failed == 0 and shaper_record(d) == want
    assert cuda_filters.buffers_alive() == alive and core().hbcu_frames_alive() == 0


@pytest.mark.gpu
def test_peak_rate_adds_no_host_wait(cuda_filters):
    """23.976 under a 30 fps peak: no drop is ever due, so no metric is ever read -- no blocking wait"""
    c = next(c for c in SHAPER_CASES if c["id"] == "pfr-23976-30")
    lib = core()
    w0, l0 = lib.hbcu_motion_metric_waits(), lib.hbcu_motion_metric_launches()
    d = run_product(cuda_filters, c, [UP, "hb_filter_vfr_cuda", DOWN])
    assert d.frames.shape[0] == c["n"]
    assert lib.hbcu_motion_metric_waits() == w0
    assert lib.hbcu_motion_metric_launches() - l0 == c["n"] - 1


@pytest.mark.gpu
def test_constant_rate_waits_at_most_once_per_drop(cuda_filters):
    c = next(c for c in SHAPER_CASES if c["id"] == "cfr-2997-23976-shift")
    lib = core()
    w0 = lib.hbcu_motion_metric_waits()
    d = run_product(cuda_filters, c, [UP, "hb_filter_vfr_cuda", DOWN])
    drops = c["n"] - d.frames.shape[0]
    assert drops > 0 and lib.hbcu_motion_metric_waits() - w0 <= drops


@pytest.mark.gpu
def test_1080p10_device_chain_equals_host_chain(cuda_filters):
    """upload -> decomb -> vfr CFR -> NLMeans -> download equals the same filters on host frames"""
    c = dict(id="chain-1080p10", settings="mode=1:rate=24000/1001", n=12, rate=NTSC, fmt="420p10", w=1920, h=1080,
             content="telecine", cfr=0, gaps=(), backs=(), chap=None)
    frames, start, stop, chap = shaper_inputs(c)
    names = ["hb_filter_decomb_cuda", "hb_filter_vfr_cuda", "hb_filter_nlmeans_cuda"]
    sets = [None, c["settings"], "y-strength=6"]
    kw = run_kw(c, start, stop, chap)
    host = cuda_filters.run(names, sets, frames, 62, 1920, 1080, **kw)
    alive = cuda_filters.buffers_alive()
    dev = cuda_filters.run([UP] + names + [DOWN], [None] + sets + [None], frames, 62, 1920, 1080, **kw)
    assert host.init_failed == 0 and dev.init_failed == 0
    assert 0 < dev.frames.shape[0] < c["n"]
    assert np.array_equal(host.start, dev.start) and np.array_equal(host.stop, dev.stop)
    assert np.array_equal(host.frames, dev.frames)
    assert cuda_filters.buffers_alive() == alive and core().hbcu_frames_alive() == 0
