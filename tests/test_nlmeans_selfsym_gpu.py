"""GPU parity of the symmetric frame-0 march of the 8-bit v3 NLMeans kernel (range 3, no prefilter): frame 0 is compared
with itself there, and its eight weights come from four displacements read at shifted pixels.  Bit-exact against the
reference's hb_filter_nlmeans on geometries that end inside a tile and inside a 10-row strip, on flat and saturating
content, and in a fused launch whose chroma planes keep the general path.

The reference's results of these calls are stored in tests/golden/selfsym_ref_digests.json and answered the same way
as the suite's other reference calls (tests/golden_ref.py); `HBCU_RECORD_REF=1` with the reference built re-records
them into that file."""
import json
from pathlib import Path

import numpy as np
import pytest

from golden_ref import GoldenRef
from handbrake_b200 import synth

pytestmark = pytest.mark.gpu

FMT8 = synth.PIX_FMT_YUV420P
STORE = Path(__file__).resolve().parent / "golden" / "selfsym_ref_digests.json"


class SelfSymRef(GoldenRef):
    """GoldenRef over this file's own store of reference digests"""

    def __init__(self):
        super().__init__()
        self.store = json.loads(STORE.read_text()) if STORE.exists() else {}

    def _save(self):
        STORE.write_text(json.dumps(dict(sorted(self.store.items())), indent=0) + "\n")


@pytest.fixture(scope="module")
def ref():
    return SelfSymRef()


def run_both(ref, cuda, settings, clip, w, h):
    r = ref.run("hb_filter_nlmeans", settings + ":threads=2", clip, FMT8, w, h)
    g = cuda.run("hb_filter_nlmeans_cuda", settings, clip, FMT8, w, h)
    return r, g


def assert_same(r, g):
    assert g.saw_eof and r.saw_eof
    assert g.frames.shape == r.frames.shape
    assert np.array_equal(g.start, r.start)
    if not np.array_equal(g.frames, r.frames):
        d = np.abs(g.frames.astype(np.int32) - r.frames.astype(np.int32))
        bad = np.argwhere(d.max(axis=1) > 0).ravel()
        raise AssertionError(f"mismatch: max abs {d.max()}, {np.count_nonzero(d)} bytes differ, frames {bad[:8]}")


def range3(patch, frames, strength=6, origin=None):
    """the same patch size, range 3 and frame count in all three planes (one fused launch)"""
    s = []
    for c in ("y", "cb", "cr"):
        s.append(f"{c}-strength={strength}:{c}-patch-size={patch}:{c}-range=3:{c}-frame-count={frames}")
        if origin is not None:
            s.append(f"{c}-origin-tune={origin}")
    return ":".join(s)


@pytest.mark.parametrize("frames", [1, 2, 3])
@pytest.mark.parametrize("patch", [3, 5, 7])
def test_patch_and_frame_count(ref, cuda_filters, patch, frames):
    w, h = 257, 121
    clip = synth.progressive_clip(FMT8, w, h, 5, seed=101 + patch)
    r, g = run_both(ref, cuda_filters, range3(patch, frames), clip, w, h)
    assert_same(r, g)


@pytest.mark.parametrize("h", [119, 120, 121])
@pytest.mark.parametrize("w", [127, 128, 129, 257])
def test_tile_and_strip_edges(ref, cuda_filters, w, h):
    """widths around the 128-pixel tile, heights around the 120-row tile; odd widths and heights give odd chroma planes"""
    clip = synth.progressive_clip(FMT8, w, h, 3, seed=7 * w + h)
    r, g = run_both(ref, cuda_filters, range3(7, 2), clip, w, h)
    assert_same(r, g)


@pytest.mark.parametrize("patch", [3, 5, 7])
def test_flat_and_saturating_content(ref, cuda_filters, patch):
    """flat frames (every weight the same), 0/255 stripes and checkerboards (the largest patch distances: saturated
    table index), full-range noise, at several origin-tune values"""
    w, h = 161, 123
    fb = synth.frame_bytes(FMT8, w, h)
    idx = np.arange(fb)
    rng = np.random.default_rng(patch)
    clip = np.stack([np.full(fb, 128, np.uint8),
                     np.where((idx // 3) % 2 == 0, 255, 0).astype(np.uint8),
                     np.where(((idx % w) + (idx // w)) % 2 == 0, 255, 0).astype(np.uint8),
                     rng.integers(0, 256, fb, dtype=np.uint8),
                     np.zeros(fb, np.uint8)])
    for strength, origin in ((3, 0.05), (10, 0.8), (6, 1.0), (1.5, 2.5)):
        r, g = run_both(ref, cuda_filters, range3(patch, 2, strength, origin), clip, w, h)
        assert_same(r, g)


def test_fused_range3_luma_range5_chroma(ref, cuda_filters):
    """one launch over the three planes: luma at range 3, chroma at range 5 (the general path for every plane)"""
    w, h = 203, 131
    clip = synth.progressive_clip(FMT8, w, h, 4, seed=31)
    s = ("y-strength=6:y-patch-size=5:y-range=3:y-frame-count=2:"
         "cb-strength=5:cb-patch-size=5:cb-range=5:cb-frame-count=2:"
         "cr-strength=4:cr-patch-size=5:cr-range=5:cr-frame-count=2")
    r, g = run_both(ref, cuda_filters, s, clip, w, h)
    assert_same(r, g)


def test_luma_only_launch(ref, cuda_filters):
    """one plane per launch (the chroma planes are left as they are)"""
    w, h = 190, 250
    clip = synth.progressive_clip(FMT8, w, h, 4, seed=43)
    s = "y-strength=7:y-patch-size=7:y-range=3:y-frame-count=2:cb-strength=0:cr-strength=0"
    r, g = run_both(ref, cuda_filters, s, clip, w, h)
    assert_same(r, g)
