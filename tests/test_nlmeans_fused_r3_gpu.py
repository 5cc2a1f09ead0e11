"""GPU parity of the one-march 8-bit NLMeans kernel (nlmeans_v3f_kernel: range 3, one or two frames, patch 3/5/7, no
prefilter): frame 0 by the symmetric march, frame 1's nine displacements in the same row step, every pixel finished in
registers.  Bit-exact against the reference's hb_filter_nlmeans on geometries that end just before, at and just after
the kernel's strip and tile heights, on flat, striped, checkerboard, saturated and noisy content, and in launches that
must keep the accumulating v3 kernel (range 5 chroma, three frames).  Every case runs with the kernel on and with
HBCU_NLMEANS_V3_FUSED=0, which keeps the accumulating kernel.

The reference's results of these calls are stored in tests/golden/fused_r3_ref_digests.json; `HBCU_RECORD_REF=1` with
the reference built re-records them from the CPU test of this file."""
import json
from collections import namedtuple
from pathlib import Path

import numpy as np
import pytest

from golden_ref import GoldenRef
from handbrake_b200 import synth

FMT8 = synth.PIX_FMT_YUV420P
STORE = Path(__file__).resolve().parent / "golden" / "fused_r3_ref_digests.json"

# nlmeans.cu: kV3Fused, 12 warps x 20 rows per warp
STRIP, TILE = 20, 240


class FusedR3Ref(GoldenRef):
    """GoldenRef over this file's own store of reference digests"""

    def __init__(self):
        super().__init__()
        self.store = json.loads(STORE.read_text()) if STORE.exists() else {}

    def _save(self):
        STORE.write_text(json.dumps(dict(sorted(self.store.items())), indent=0) + "\n")


@pytest.fixture(scope="module")
def ref():
    return FusedR3Ref()


# ------------------------------------------------------------------------------------------------------------ clips
def clip_noise(w, h, n, seed):
    """the moving 8x8 pattern with +-8 noise (synth.progressive_clip)"""
    return synth.progressive_clip(FMT8, w, h, n, seed=seed)


def clip_content(w, h, n, seed):
    """flat 128, 0/255 stripes, 0/255 checkerboard, full-range noise, 0/255 noise, flat 0, flat 255 (the largest patch
    distances saturate the table index; flat frames give every displacement the same weight)"""
    fb = synth.frame_bytes(FMT8, w, h)
    idx = np.arange(fb)
    rng = np.random.default_rng(seed)
    kinds = [np.full(fb, 128, np.uint8),
             np.where((idx // 3) % 2 == 0, 255, 0).astype(np.uint8),
             np.where(((idx % w) + (idx // w)) % 2 == 0, 255, 0).astype(np.uint8),
             rng.integers(0, 256, fb, dtype=np.uint8),
             (rng.integers(0, 2, fb) * 255).astype(np.uint8),
             np.zeros(fb, np.uint8),
             np.full(fb, 255, np.uint8)]
    return np.stack([kinds[t % len(kinds)] for t in range(n)])


CLIPS = {"noise": clip_noise, "content": clip_content}

# ------------------------------------------------------------------------------------------------------------ cases
# cls: the kernel the first output frame runs (dispatch()): "v3f" nlmeans_v3f_kernel, "v3 sym" the accumulating v3 kernel
# with its symmetric frame-0 march, "v3" the accumulating kernel's group marches only
Case = namedtuple("Case", "id settings w h n clip cls")


def planes(patch, frames, strength=6, origin=None, rng=3, which=("y", "cb", "cr")):
    s = []
    for c in which:
        s.append(f"{c}-strength={strength}:{c}-patch-size={patch}:{c}-range={rng}:{c}-frame-count={frames}")
        if origin is not None:
            s.append(f"{c}-origin-tune={origin}")
    return ":".join(s)


def _patch_and_frames():
    return [Case(f"p{p}-nf{nf}", planes(p, nf), 257, 121, 4, ("noise", 100 + p), "v3f") for p in (3, 5, 7) for nf in (1, 2)]


def _edges():
    """heights one below, at and one above the strip and the tile, for luma (h) and chroma ((h + 1) / 2)"""
    hs = sorted({e + d for e in (STRIP, TILE) for d in (-1, 0, 1)} | {2 * e + d for e in (STRIP, TILE) for d in (-3, -1, 1)})
    return [Case(f"edge-{w}x{h}", planes(7, 2), w, h, 3, ("noise", 7 * w + h), "v3f") for w in (127, 128, 129, 257) for h in hs]


def _content():
    out = []
    for p in (3, 5, 7):
        for strength, origin in ((3, 0.05), (10, 0.8), (6, 1.0), (1.5, 2.5)):
            out.append(Case(f"content-p{p}-s{strength}-o{origin}", planes(p, 2, strength, origin), 161, 123, 8, ("content", p), "v3f"))
    return out


def _launches():
    luma_only = "y-strength=7:y-patch-size={}:y-range=3:y-frame-count={}:cb-strength=0:cr-strength=0"
    return [
        Case("luma-only-nf2", luma_only.format(7, 2), 190, 250, 4, ("noise", 43), "v3f"),
        Case("luma-only-nf1-p5", luma_only.format(5, 1), 190, 250, 3, ("noise", 44), "v3f"),
        # two frames in luma, one in chroma: nf per plane inside one launch
        Case("luma-nf2-chroma-nf1", planes(5, 2, which=("y",)) + ":" + planes(5, 1, strength=4, which=("cb", "cr")),
             203, 131, 4, ("noise", 45), "v3f"),
        # range 5 chroma: the whole launch keeps the accumulating kernel
        Case("luma-r3-chroma-r5", planes(5, 2, which=("y",)) + ":" + planes(5, 2, strength=5, rng=5, which=("cb", "cr")),
             203, 131, 4, ("noise", 31), "v3"),
        # three frames: the accumulating kernel with the symmetric frame-0 march; the stream's last frames have fewer
        Case("r3-nf3", planes(7, 3), 203, 249, 5, ("noise", 32), "v3 sym"),
    ]


CASES = _patch_and_frames() + _edges() + _content() + _launches()


def make_clip(c):
    kind, seed = c.clip
    return CLIPS[kind](c.w, c.h, c.n, seed)


def ref_run(ref, c, clip):
    return ref.run("hb_filter_nlmeans", c.settings + ":threads=2", clip, FMT8, c.w, c.h)


# ------------------------------------------------------------------------------------------------ kernel dispatch
def plane_params(settings):
    """range, patch and frame count of the filtered planes (cb inherits y, cr inherits cb; defaults as the filter's)"""
    kv = dict(s.split("=") for s in settings.split(":"))
    out, prev = [], {}
    for prefix in ("y", "cb", "cr"):
        p = {k: float(kv[f"{prefix}-{k}"]) if f"{prefix}-{k}" in kv else prev.get(k)
             for k in ("strength", "patch-size", "range", "frame-count")}
        prev = p
        defaults = {"strength": 6, "patch-size": 7, "range": 3, "frame-count": 2}
        p = {k: defaults[k] if v is None else v for k, v in p.items()}
        if p["strength"] != 0:
            out.append(dict(n_half=int(p["patch-size"]) // 2, r_half=int(p["range"]) // 2, frames=int(p["frame-count"])))
    return out


def dispatch(c):
    """the kernel of the first output frame, as run_filter() / launch_v3_nh() choose it for 8-bit planes of one patch
    size: nlmeans_v3f_kernel when every plane has range 3 and at most two frames, the symmetric frame-0 march of the
    accumulating kernel when every plane has range 3, its group marches otherwise"""
    ps = plane_params(c.settings)
    assert len({p["n_half"] for p in ps}) == 1 and all(1 <= p["n_half"] <= 3 for p in ps), c.id
    navail = min(max(p["frames"] for p in ps), c.n)
    nf = [min(navail, p["frames"]) for p in ps]
    if all(p["r_half"] == 1 for p in ps):
        return "v3f" if max(nf) <= 2 else "v3 sym"
    return "v3"


def test_dispatch():
    """every case reaches the kernel it claims, all three are reached, and the heights straddle the strip and the tile
    in luma and in chroma"""
    for c in CASES:
        assert dispatch(c) == c.cls, c.id
    assert {c.cls for c in CASES} == {"v3f", "v3 sym", "v3"}
    luma = {c.h for c in CASES}
    chroma = {(h + 1) // 2 for h in luma}
    for edge in (STRIP, TILE):
        assert {edge - 1, edge, edge + 1} <= luma and {edge - 1, edge, edge + 1} <= chroma, edge


def test_shape_matches_kernel():
    """STRIP and TILE restate kV3Fused in nlmeans.cu"""
    src = (Path(__file__).resolve().parent.parent / "handbrake_b200" / "csrc" / "nlmeans.cu").read_text()
    assert f"constexpr V3Shape kV3Fused = {{ {TILE // STRIP}, {STRIP} }};" in src


@pytest.mark.parametrize("c", CASES, ids=[c.id for c in CASES])
def test_restatement_matches_reference(ref, c):
    """the plain-C restatement reproduces the reference's stored result for every case"""
    r = ref_run(ref, c, make_clip(c))
    assert r.saw_eof and r.frames.shape == (c.n, synth.frame_bytes(FMT8, c.w, c.h))


@pytest.mark.gpu
@pytest.mark.parametrize("fused", ["1", "0"], ids=["fused", "accumulating"])
@pytest.mark.parametrize("c", CASES, ids=[c.id for c in CASES])
def test_cuda_matches_reference(ref, cuda_filters, monkeypatch, c, fused):
    monkeypatch.setenv("HBCU_NLMEANS_V3_FUSED", fused)
    clip = make_clip(c)
    r = ref_run(ref, c, clip)
    g = cuda_filters.run("hb_filter_nlmeans_cuda", c.settings, clip, FMT8, c.w, c.h)
    assert not g.init_failed
    assert g.saw_eof and r.saw_eof
    assert g.frames.shape == r.frames.shape
    assert np.array_equal(g.start, r.start)
    if not np.array_equal(g.frames, r.frames):
        d = np.abs(g.frames.astype(np.int32) - r.frames.astype(np.int32))
        bad = np.argwhere(d.max(axis=1) > 0).ravel()
        raise AssertionError(f"mismatch: max abs {d.max()}, {np.count_nonzero(d)} bytes differ, frames {bad[:8]}")
