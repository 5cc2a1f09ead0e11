"""NLMeans across its parameter space: search ranges 1-27, frame counts up to 32, patch sizes 1-31, the strengths at the
limits of the fast kernels' table trick, 8/10/12-bit, the v3 prefilter variant and every shipping preset x tune.

`select_kernels` in handbrake_b200/csrc/nlmeans.cu chooses between about ten kernels from the patch size, range, frame
count, strength (through wfact), bit depth and prefilter of each plane, and from whether all planes fit one launch.
CASES names, for each job, the kernel class it is meant to reach; `test_dispatch_coverage` restates that choice in
Python and checks every claim, and that the 8-bit and 10-bit cases that reach the v3 kernels run every group shape
those kernels are built with (V3_GROUP_SHAPES in nlmeans_v3.cuh).

Each case runs twice: without a GPU, the plain-C restatement (through the host filters) must reproduce the stored
digest of the reference's result; on the GPU, hb_filter_nlmeans_cuda must reproduce the reference's frames bit for bit.
The reference's results are stored in tests/golden/nlmeans_params_ref_digests.json; `HBCU_RECORD_REF=1` with the
reference built re-records them from the CPU tests of this file."""
import ctypes as C
import json
import re
from collections import namedtuple
from pathlib import Path

import numpy as np
import pytest

from golden_ref import GoldenRef
from handbrake_b200 import synth
from oracle_port import PORT_SO

FMT8, FMT10, FMT12 = synth.PIX_FMT_YUV420P, synth.PIX_FMT_YUV420P10, synth.PIX_FMT_YUV420P12
HERE = Path(__file__).resolve().parent
STORE = HERE / "golden" / "nlmeans_params_ref_digests.json"
V3_HEADER = HERE.parent / "handbrake_b200" / "csrc" / "nlmeans_v3.cuh"

# nlmeans.cu: tile halo, displacements per v3 group, deepest window of the tiled kernels, the plane border
K_HALO, K_GROUP, K_MAX_TILED_FRAMES, K_BORDER = 8, 3, 8, 16


class ParamsRef(GoldenRef):
    """GoldenRef over this file's own store of reference digests"""

    def __init__(self):
        super().__init__()
        self.store = json.loads(STORE.read_text()) if STORE.exists() else {}

    def _save(self):
        STORE.write_text(json.dumps(dict(sorted(self.store.items())), indent=0) + "\n")


@pytest.fixture(scope="module")
def ref():
    return ParamsRef()


# ------------------------------------------------------------------------------------------------------------ clips
def clip_noise(fmt, w, h, n, seed):
    """the moving 8x8 pattern with +-8 noise (synth.progressive_clip)"""
    return synth.progressive_clip(fmt, w, h, n, seed=seed)


def _samples(fmt, w, h, frames):
    dt = np.uint16 if synth.depth_of(fmt) > 8 else np.uint8
    return np.stack([np.asarray(f, dt) for f in frames]).view(np.uint8).reshape(len(frames), -1)


def clip_extreme(fmt, w, h, n, seed):
    """full-range noise, flat 0, flat max, 0/max noise, repeating (the largest patch distances)"""
    m = synth.frame_bytes(fmt, w, h) // (2 if synth.depth_of(fmt) > 8 else 1)
    top = (1 << synth.depth_of(fmt)) - 1
    rng = np.random.default_rng(seed)
    kinds = [lambda: rng.integers(0, top + 1, m), lambda: np.zeros(m, np.int64), lambda: np.full(m, top),
             lambda: rng.integers(0, 2, m) * top]
    return _samples(fmt, w, h, [kinds[t % 4]() for t in range(n)])


def clip_band(fmt, w, h, n, seed, lo, hi):
    """uniform noise in [lo, hi]: bounds the largest patch distance (p^2 (hi-lo)^2)"""
    m = synth.frame_bytes(fmt, w, h) // (2 if synth.depth_of(fmt) > 8 else 1)
    rng = np.random.default_rng(seed)
    return _samples(fmt, w, h, [rng.integers(lo, hi + 1, m) for _ in range(n)])


def clip_step(fmt, w, h, n, seed, v, c):
    """flat frames, frame t = v + t*c: every temporal patch distance between neighbours is exactly p^2 c^2"""
    m = synth.frame_bytes(fmt, w, h) // (2 if synth.depth_of(fmt) > 8 else 1)
    return _samples(fmt, w, h, [np.full(m, v + t * c) for t in range(n)])


CLIPS = {"noise": clip_noise, "extreme": clip_extreme, "band": clip_band, "step": clip_step}

# ------------------------------------------------------------------------------------------------------------ cases
Case = namedtuple("Case", "id settings fmt w h n clip cls threads")
# clip: (kind, seed, *args) of CLIPS; cls: the kernel class the first output frame is meant to reach (dispatch())
CLASSES = ("v3 fused", "v3 planes", "v3 pre", "v3w fused", "fast16 fused", "tiled8", "tiled16", "generic")


def plane_settings(patch, rng, frames=2, strength=6, prefix="y"):
    return f"{prefix}-strength={strength}:{prefix}-patch-size={patch}:{prefix}-range={rng}:{prefix}-frame-count={frames}"


def case(cid, settings, fmt, wh, n, clip, cls, threads=2):
    return Case(cid, settings, fmt, wh[0], wh[1], n, clip, cls, threads)


# 257x130: 3 tile columns (128 wide) x 2 tile rows (120 high), chroma 129x65; 136x122 (chroma 68x61) for the costly ones
G_WIDE, G_SMALL, G_TINY = (257, 130), (136, 122), (48, 40)
BITS = {FMT8: "8", FMT10: "10", FMT12: "12"}


def _halo_edge(patch):
    """the largest range whose patch/search window fits the tile halo: n/2 + r/2 == K_HALO"""
    return 2 * (K_HALO - patch // 2) + 1


def _sweep():
    """every odd range up to the halo edge and one past it (the generic kernel), luma and chroma the same"""
    out = []
    for patch in (3, 5, 7, 9):
        edge = _halo_edge(patch)
        for rng in range(1, edge + 3, 2):
            # range 1 splits into no v3 group shape: one generic launch per plane
            cls = "v3 fused" if 1 < rng <= edge else "generic"
            out.append(case(f"sweep8-p{patch}-r{rng}", plane_settings(patch, rng), FMT8, G_WIDE if rng <= 7 else G_SMALL,
                            2, ("noise", 10 * patch + rng), cls))
    for patch in (3, 5, 7):
        edge = _halo_edge(patch)
        for rng in [1] + list(range(9, edge + 1, 2)) + ([edge + 2] if patch == 3 else []):
            cls = "fast16 fused" if rng == 1 else "v3w fused" if rng <= edge else "generic"
            out.append(case(f"sweep10-p{patch}-r{rng}", plane_settings(patch, rng), FMT10, G_SMALL, 2,
                            ("noise", 100 + 10 * patch + rng), cls))
    out.append(case("sweep10-p5-r11-extreme", plane_settings(5, 11, strength=4), FMT10, G_SMALL, 4, ("extreme", 9),
                    "v3w fused"))
    # chroma at another range than luma: one launch, two decompositions of the displacement rows
    out.append(case("split8-r5-r11-same-patch", plane_settings(5, 5) + ":" + plane_settings(5, 11, strength=4, prefix="cb"),
                    FMT8, G_SMALL, 2, ("noise", 71), "v3 fused"))
    # another patch size: one launch per plane
    out.append(case("split8-p3r13-p5r9", plane_settings(3, 13) + ":" + plane_settings(5, 9, strength=4, prefix="cb"),
                    FMT8, G_SMALL, 2, ("noise", 72), "v3 planes"))
    return out


def _frame_counts():
    """windows deeper than the tiled kernels take (9-32) and clips shorter and longer than the window: at the end of
    the stream the window shrinks, across 9 -> 8 where the kernel changes"""
    out = []
    for fmt in (FMT8, FMT10):
        fused = "v3 fused" if fmt == FMT8 else "v3w fused"
        for fc, n, rng in ((5, 7, 5), (8, 10, 5), (9, 11, 5), (16, 12, 5), (32, 34, 3)):
            cls = fused if min(fc, n) <= K_MAX_TILED_FRAMES else "generic"
            out.append(case(f"frames{BITS[fmt]}-fc{fc}-n{n}", plane_settings(3, rng, frames=fc), fmt, G_SMALL, n,
                            ("noise", 200 + fc), cls))
    out.append(case("frames8-luma8-chroma9", plane_settings(3, 5, frames=8) + ":cb-frame-count=9", FMT8, G_SMALL, 11,
                    ("noise", 231), "v3 planes"))
    return out


def _patch_edges():
    out = [case("patch1-r3", plane_settings(1, 3), FMT8, G_WIDE, 3, ("noise", 301), "generic"),
           case("patch1-r15", plane_settings(1, 15), FMT8, G_SMALL, 2, ("noise", 302), "generic"),
           case("patch11-r3", plane_settings(11, 3), FMT8, G_SMALL, 2, ("noise", 303), "generic"),
           case("patch13-r5", plane_settings(13, 5), FMT8, G_SMALL, 2, ("noise", 304), "generic")]
    # patch/2 + range/2 == K_BORDER: the largest search the 16-pixel plane border allows
    out.append(case("border-p7-r27", plane_settings(7, 27), FMT8, G_TINY, 2, ("noise", 305), "generic"))
    out.append(case("border-p31-r3-10bit", plane_settings(31, 3, strength=3), FMT10, G_TINY, 2, ("noise", 306), "generic"))
    return out


# strengths just inside and just outside the window 1e-5 < wfact < 0.99 of the fast kernels' saturating table, found
# by bisection over oracle_nlmeans_table; test_dispatch_coverage checks the side each one is on
STRENGTH_EDGES = {
    # (depth, patch): {edge: (strength inside, strength outside)}
    # the outside strength puts wfact exactly on the limit (float32(0.99) / float32(1e-5)), which the kernels refuse
    (8, 3): {0.99: (1.374781092455386, 1.3747810924553858), 1e-5: (432.56476012919757, 432.5647601291976)},
    (8, 7): {0.99: (0.589191896766594, 0.5891918967665939), 1e-5: (185.38489719822752, 185.38489719822755)},
    (10, 3): {0.99: (0.3436952731138465, 0.34369527311384646), 1e-5: (108.14119003229939, 108.1411900322994)},
    (10, 7): {0.99: (0.1472979741916485, 0.14729797419164847), 1e-5: (46.34622429955688, 46.34622429955689)},
}
# flat two-frame clips whose temporal patch distance n^2 c^2 is exactly diff_max - 1 (still weighted) or diff_max (not):
# (depth, patch, base, c): {diff_max: strength}
DIFF_MAX_EDGES = {
    (8, 3, 100, 10): {900: 3.62817, 901: 3.63019},
    (8, 7, 60, 4): {784: 1.45133, 785: 1.45225},
    (10, 3, 400, 40): {14400: 3.62723, 14401: 3.62735},
    (10, 7, 300, 12): {7056: 1.08819, 7057: 1.08827},
}


def _strength_edges():
    out = []
    for (depth, patch), edges in STRENGTH_EDGES.items():
        fmt = FMT8 if depth == 8 else FMT10
        top = (1 << depth) - 1
        for edge, (s_in, s_out) in edges.items():
            # 0.99: distances below diff_max (~129) need near-equal patches; 1e-5: a bounded distance keeps the
            # reference's table index below 128
            lo, hi = ((top + 1) // 2, (top + 1) // 2 + 3) if edge == 0.99 else ((top + 1) // 4, (top + 1) // 4 + (top + 1) // 8)
            for side, s in (("in", s_in), ("out", s_out)):
                cls = ("v3 fused" if depth == 8 else "v3w fused") if side == "in" else ("tiled8" if depth == 8 else "tiled16")
                out.append(case(f"wfact{depth}-p{patch}-{edge:g}-{side}", plane_settings(patch, 5, strength=s), fmt, G_SMALL,
                                3, ("band", 400 + patch, lo, hi), cls))
    for (depth, patch, v, c), edges in DIFF_MAX_EDGES.items():
        fmt = FMT8 if depth == 8 else FMT10
        for dmax, s in edges.items():
            tag = "at" if dmax == patch * patch * c * c else "below"
            out.append(case(f"diffmax{depth}-p{patch}-{tag}", plane_settings(patch, 5, strength=s), fmt, G_SMALL, 2,
                            ("step", 0, v, c), "v3 fused" if depth == 8 else "v3w fused"))
    return out


def _twelve_bit():
    out = []
    for patch in (3, 5, 7, 9):
        for rng in (3, 9):
            out.append(case(f"12bit-p{patch}-r{rng}-noise", plane_settings(patch, rng), FMT12, G_SMALL, 2,
                            ("noise", 500 + patch + rng), "tiled16"))
            out.append(case(f"12bit-p{patch}-r{rng}-extreme", plane_settings(patch, rng, strength=4), FMT12, G_SMALL, 2,
                            ("extreme", 500 + patch + rng), "tiled16"))
    # the 12-bit patch distance of the reference is an int: 11^2 * 4095^2 still fits it, 13^2 * 4095^2 does not
    out.append(case("12bit-p11-r3-extreme", plane_settings(11, 3), FMT12, G_SMALL, 2, ("extreme", 520), "generic"))
    return out


def _prefilter():
    """the v3 kernel's prefilter variant (patch distances on the pre-denoised planes); the reference races on
    frame[0].image_pre with more than one worker, so it runs with one"""
    out = []
    for mode in (1, 4):
        for patch in (3, 5):
            for rng in (5, 9, 13):
                out.append(case(f"prefilter{mode}-p{patch}-r{rng}", plane_settings(patch, rng) + f":y-prefilter={mode}", FMT8,
                                G_SMALL, 3, ("noise", 600 + patch + rng), "v3 pre", threads=1))
    return out


# the nlmeans presets x tunes of HandBrake's libhb/param.c (generate_nlmeans_settings, lines 408-574): per tune the
# medium values of luma and chroma, then the ultralight / light / strong overrides; cr inherits cb.
# (strength, origin tune, patch size, range, frame count) per plane.
TUNE_MEDIUM = {
    "none":       ((6, 1, 7, 3, 2),      (6, 1, 7, 3, 2)),        # param.c:410-415
    "film":       ((6, 0.8, 7, 3, 2),    (8, 0.8, 7, 3, 2)),      # param.c:431-436
    "grain":      ((0, 0.8, 7, 3, 2),    (6, 0.8, 7, 3, 2)),      # param.c:455-460
    "highmotion": ((6, 0.8, 7, 3, 2),    (6, 0.7, 7, 5, 1)),      # param.c:479-484
    "animation":  ((5, 0.15, 5, 7, 4),   (4, 0.15, 5, 7, 4)),     # param.c:503-508
    "tape":       ((3, 0.8, 3, 5, 2),    (6, 0.8, 5, 5, 2)),      # param.c:526-531
    "sprite":     ((3, 0.15, 5, 5, 2),   (4, 0.5, 5, 9, 4)),      # param.c:552-557
}
# preset -> tune -> {field: (luma, chroma)}; fields: 0 strength, 1 origin tune, 2 patch size, 3 range, 4 frame count
TUNE_OVERRIDES = {
    "ultralight": {"none": {0: (1.5, 1.5)},                                              # param.c:416-419
                   "film": {0: (1.5, 2.4), 1: (0.9, 0.9)},                               # param.c:437-441
                   "grain": {0: (0, 2.4), 1: (0.9, 0.9)},                                # param.c:461-465
                   "highmotion": {0: (1.5, 2.4), 1: (0.9, 0.9)},                         # param.c:485-489
                   "animation": {0: (2.5, 2), 4: (2, 2)},                                # param.c:509-513
                   "tape": {0: (1.5, 5), 1: (0.9, 0.9), 4: (1, 1)},                      # param.c:532-537
                   "sprite": {0: (1.5, 3), 3: (5, 7), 4: (1, 2)}},                       # param.c:558-563
    "light": {"none": {0: (3, 3)},                                                       # param.c:420-423
              "film": {0: (3, 4), 1: (0.9, 0.9)},                                        # param.c:442-446
              "grain": {0: (0, 3.5), 1: (0.9, 0.9)},                                     # param.c:466-470
              "highmotion": {0: (3, 3.25), 1: (0.9, 0.8)},                               # param.c:490-494
              "animation": {0: (3, 2.25), 4: (3, 3)},                                    # param.c:514-518
              "tape": {0: (2, 6), 1: (0.9, 0.9)},                                        # param.c:538-542
              "sprite": {0: (2, 4), 4: (2, 2)}},                                         # param.c:564-568
    "medium": {},
    "strong": {"none": {0: (10, 10)},                                                    # param.c:424-427
               "film": {0: (8, 10), 1: (0.6, 0.6)},                                      # param.c:447-451
               "grain": {0: (0, 8), 1: (0.6, 0.6)},                                      # param.c:471-475
               "highmotion": {0: (8, 6.75), 1: (0.6, 0.5)},                              # param.c:495-499
               "animation": {0: (10, 8)},                                                # param.c:519-522
               "tape": {0: (3.5, 8), 1: (0.6, 0.6), 2: (5, 5)},                          # param.c:543-548
               "sprite": {0: (3, 4), 3: (7, 11)}},                                       # param.c:569-573
}


def preset_settings(preset, tune):
    """the settings generate_nlmeans_settings() writes (param.c:581-594), in its key order"""
    planes = [list(v) for v in TUNE_MEDIUM[tune]]
    for field, (y, c) in TUNE_OVERRIDES[preset].get(tune, {}).items():
        planes[0][field], planes[1][field] = y, c
    s = []
    for prefix, (st, org, patch, rng, fc) in zip(("y", "cb"), planes):
        s.append(f"{prefix}-strength={st:g}:{prefix}-origin-tune={org:g}:{prefix}-patch-size={patch}:{prefix}-range={rng}:"
                 f"{prefix}-frame-count={fc}:{prefix}-prefilter=0")
    return ":".join(s)


def _presets():
    out = []
    for fmt in (FMT8, FMT10):
        for preset in TUNE_OVERRIDES:
            for tune in TUNE_MEDIUM:
                # tape (but strong) filters luma with patch 3 and chroma with patch 5: one launch per plane
                split = tune == "tape" and preset != "strong"
                cls = ("v3 planes" if split else "v3 fused") if fmt == FMT8 else ("tiled16" if split else "v3w fused")
                out.append(case(f"preset{BITS[fmt]}-{preset}-{tune}", preset_settings(preset, tune), fmt, G_SMALL, 3,
                                ("noise", 700), cls))
    return out


CASES = _sweep() + _frame_counts() + _patch_edges() + _strength_edges() + _twelve_bit() + _prefilter() + _presets()


def make_clip(c):
    kind, seed, *args = c.clip
    return CLIPS[kind](c.fmt, c.w, c.h, c.n, seed, *args)


def ref_run(ref, c, clip):
    return ref.run("hb_filter_nlmeans", c.settings + f":threads={c.threads}", clip, c.fmt, c.w, c.h)


# ------------------------------------------------------------------------------------------------ kernel dispatch
def v3_group_shapes():
    """the (displacements, (12 + dx0) & 3, origin slot or None) the v3 kernels are built with, read from V3_GROUP_SHAPES"""
    m = re.search(r"#define V3_GROUP_SHAPES\(X\)((?:.*\\\n)*.*)", V3_HEADER.read_text())
    shapes = {(int(a), int(b), None if o == "kOrgNone" else int(o))
              for a, b, o in re.findall(r"X\((\d+),\s*(\d+),\s*(\w+)\)", m.group(1))}
    assert len(shapes) == 11, shapes
    return shapes


def v3_groups(r_half):
    """range_splits: a displacement row cut into groups of K_GROUP, the remainder last -> (dx0, ng, (12 + dx0) & 3)"""
    for dx0 in range(-r_half, r_half + 1, K_GROUP):
        ng = min(K_GROUP, r_half - dx0 + 1)
        yield dx0, ng, (12 + dx0) & 3


def v3_known(r_half, known):
    """range_splits: every group of the range, and its origin variant, is a built shape"""
    return all((ng, ob, None) in known and (not dx0 <= 0 < dx0 + ng or (ng, ob, -dx0) in known)
               for dx0, ng, ob in v3_groups(r_half))


def v3_launch_shapes(planes, sym_ok):
    """the group shapes one v3 launch runs (nlmeans_v3_kernel's frame loop): frame 0's row dy == 0 runs the group
    holding dx = 0 in its origin variant; with range 3 in every plane (and patch <= 7, 8-bit) frame 0 is the V3Sym
    march instead and runs no group"""
    sym = sym_ok and all(p["r_half"] == 1 for p in planes)
    out = set()
    for p in planes:
        for f in range(p["nf"]):
            if f == 0 and sym:
                continue
            for dy in range(-p["r_half"], p["r_half"] + 1):
                for dx0, ng, ob in v3_groups(p["r_half"]):
                    out.add((ng, ob, -dx0 if f == 0 and dy == 0 and dx0 <= 0 < dx0 + ng else None))
    return out


_PORT = None


def nlmeans_table(strength, patch, depth):
    """(wfact, diff_max) of the reference's table for these settings, from the restatement (oracle_nlmeans_table)"""
    global _PORT
    if _PORT is None:
        _PORT = C.CDLL(str(PORT_SO))
        _PORT.oracle_nlmeans_table.argtypes = [C.c_double, C.c_int, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_int),
                                               C.POINTER(C.c_float)]
    wf, dm, tab = C.c_float(), C.c_int(), (C.c_float * 128)()
    _PORT.oracle_nlmeans_table(float(strength), int(patch), int(depth), C.byref(wf), C.byref(dm), tab)
    return np.float32(wf.value), dm.value


def plane_params(settings, depth):
    """hb_nlmeans_cuda_build_config: per-plane settings with cb inheriting y and cr inheriting cb, defaults, sanitising"""
    kv = dict(s.split("=") for s in settings.split(":"))
    keys = {"strength": float, "origin-tune": float, "patch-size": int, "range": int, "frame-count": int, "prefilter": int}
    defaults = {"strength": 6, "origin-tune": 1, "patch-size": 7, "range": 3, "frame-count": 2, "prefilter": 0}
    out, prev = [], {}
    for prefix in ("y", "cb", "cr"):
        p = {k: t(kv[f"{prefix}-{k}"]) if f"{prefix}-{k}" in kv else prev.get(k) for k, t in keys.items()}
        prev = p
        p = {k: defaults[k] if v is None else v for k, v in p.items()}
        p["patch-size"] = max(1, p["patch-size"] - (p["patch-size"] % 2 == 0))
        p["range"] = max(1, p["range"] - (p["range"] % 2 == 0))
        p["frame-count"] = min(32, max(1, p["frame-count"]))
        out.append(p)
    return out


def dispatch(c):
    """the kernel class of the first output frame and the v3 / v3w group shapes it runs, as select_kernels() and
    plane_kernel() choose them (HBCU_NLMEANS_IMPL unset)"""
    depth = synth.depth_of(c.fmt)
    params = plane_params(c.settings, depth)
    navail = min(max(p["frame-count"] for p in params), c.n)
    known = v3_group_shapes()
    planes = []
    for p in params:
        if p["strength"] == 0 or p["prefilter"] & 2048:
            continue
        wfact, _ = nlmeans_table(p["strength"], p["patch-size"], depth)
        k = dict(n_half=(p["patch-size"] - 1) // 2, r_half=(p["range"] - 1) // 2, nf=min(navail, p["frame-count"]),
                 pre=(p["prefilter"] & 63) != 0, window=np.float32(1e-5) < wfact < np.float32(0.99))
        k["tiled"] = not k["pre"] and 1 <= k["n_half"] <= 4 and k["n_half"] + k["r_half"] <= K_HALO and k["nf"] <= K_MAX_TILED_FRAMES
        k["known"] = v3_known(k["r_half"], known)
        planes.append(k)
    same_nh = len({k["n_half"] for k in planes}) == 1
    shapes = {"v3": set(), "v3w": set()}
    if depth > 8:
        if planes and same_nh and all(depth <= 10 and k["tiled"] and k["n_half"] <= 3 and k["window"] for k in planes):
            if all(k["known"] for k in planes):
                shapes["v3w"] = v3_launch_shapes(planes, sym_ok=False)
                return "v3w fused", shapes
            return "fast16 fused", shapes
        return ("tiled16" if any(k["tiled"] for k in planes) else "generic"), shapes
    if len(planes) > 1 and same_nh and all(k["tiled"] and k["window"] and k["known"] for k in planes):
        shapes["v3"] = v3_launch_shapes(planes, sym_ok=planes[0]["n_half"] <= 3)
        return "v3 fused", shapes
    kinds = set()
    for k in planes:
        if k["pre"] and 1 <= k["n_half"] <= 3 and k["n_half"] + k["r_half"] <= K_HALO and k["nf"] <= K_MAX_TILED_FRAMES \
                and k["window"] and k["known"]:
            kinds.add("v3 pre")
        elif k["tiled"] and k["window"] and k["known"]:
            shapes["v3"] |= v3_launch_shapes([k], sym_ok=k["n_half"] <= 3)
            kinds.add("v3 planes")
        elif k["tiled"] and not k["window"]:
            kinds.add("tiled8")
        else:
            kinds.add("generic")
    return next(cls for cls in ("v3 pre", "v3 planes", "tiled8", "generic") if cls in kinds), shapes


def test_dispatch_coverage():
    """every case reaches the kernel class it claims; together they reach every class and, at 8 and at 10 bits, every
    group shape of the v3 kernels"""
    known = v3_group_shapes()
    reached = {"v3": set(), "v3w": set()}
    for c in CASES:
        cls, shapes = dispatch(c)
        assert cls == c.cls, f"{c.id}: reaches {cls}, claims {c.cls}"
        for k in reached:
            reached[k] |= shapes[k]
    assert {c.cls for c in CASES} == set(CLASSES)
    assert reached["v3"] == known, f"8-bit v3 shapes never run: {sorted(known - reached['v3'], key=str)}"
    assert reached["v3w"] == known, f"10-bit v3w shapes never run: {sorted(known - reached['v3w'], key=str)}"


def test_edge_cases_lie_where_they_claim():
    """the strength cases sit just inside / just outside 1e-5 < wfact < 0.99; the flat-step cases put the temporal
    patch distance exactly at diff_max - 1 or diff_max; wherever wfact is small, the largest possible patch distance
    keeps the reference's table index (int)(diff * wfact) at or below 127"""
    for (depth, patch), edges in STRENGTH_EDGES.items():
        for edge, (s_in, s_out) in edges.items():
            w_in, w_out = nlmeans_table(s_in, patch, depth)[0], nlmeans_table(s_out, patch, depth)[0]
            e = np.float32(edge)
            assert np.float32(1e-5) < w_in < np.float32(0.99), (depth, patch, edge, w_in)
            assert (w_out >= e) if edge == 0.99 else (w_out <= e), (depth, patch, edge, w_out)
            assert abs(w_in / e - 1) < 1e-5 and abs(w_out / e - 1) < 1e-5, (depth, patch, edge, w_in, w_out)
    for (depth, patch, v, c), edges in DIFF_MAX_EDGES.items():
        d = patch * patch * c * c
        assert sorted(edges) == [d, d + 1]
        for dmax, s in edges.items():
            wfact, got = nlmeans_table(s, patch, depth)
            assert got == dmax
            assert int(np.float32(d) * wfact) <= 127
    for c in CASES:
        clip = make_clip(c)
        depth = synth.depth_of(c.fmt)
        samples = clip.view(np.uint16) if depth > 8 else clip
        spread = int(samples.max()) - int(samples.min())
        for p in plane_params(c.settings, depth):
            if p["strength"] == 0:
                continue
            wfact, dmax = nlmeans_table(p["strength"], p["patch-size"], depth)
            if wfact < np.float32(1.5e-5):
                assert int(np.float32(min(p["patch-size"] ** 2 * spread ** 2, dmax - 1)) * wfact) <= 127, c.id


@pytest.mark.parametrize("c", CASES, ids=[c.id for c in CASES])
def test_restatement_matches_reference(ref, c):
    """the plain-C restatement reproduces the reference's stored result for every case"""
    r = ref_run(ref, c, make_clip(c))
    assert r.saw_eof and r.frames.shape == (c.n, synth.frame_bytes(c.fmt, c.w, c.h))
    assert ref.buffers_alive() == 0


@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES, ids=[c.id for c in CASES])
def test_cuda_matches_reference(ref, cuda_filters, c):
    clip = make_clip(c)
    r = ref_run(ref, c, clip)
    g = cuda_filters.run("hb_filter_nlmeans_cuda", c.settings, clip, c.fmt, c.w, c.h)
    assert not g.init_failed
    assert g.saw_eof and r.saw_eof
    assert g.frames.shape == r.frames.shape
    assert np.array_equal(g.start, r.start)
    if not np.array_equal(g.frames, r.frames):
        d = np.abs(g.frames.astype(np.int32) - r.frames.astype(np.int32))
        bad = np.argwhere(d.max(axis=1) > 0).ravel()
        raise AssertionError(f"mismatch: max abs {d.max()}, {np.count_nonzero(d)} bytes differ, frames {bad[:8]}")
    assert cuda_filters.buffers_alive() == 0 and ref.buffers_alive() == 0


@pytest.mark.gpu
@pytest.mark.parametrize("patch,rng", [(7, 29), (3, 33), (9, 27)])
def test_search_past_the_border_is_refused(cuda_filters, patch, rng):
    """patch/2 + range/2 == 17 reaches past the 16-pixel border (the reference reads outside its planes there)"""
    w, h = G_TINY
    clip = clip_noise(FMT8, w, h, 2, 1)
    g = cuda_filters.run("hb_filter_nlmeans_cuda", plane_settings(patch, rng), clip, FMT8, w, h)
    assert g.init_failed == 1
