"""The 45-row shape of the one-march 8-bit NLMeans kernel (nlmeans_v3f_kernel at 12 warps x 45 rows, a 540-row tile that
arrives in three TMA boxes of 188 rows) and the rule that picks a shape per handle.

Bit-exact against the reference's hb_filter_nlmeans with the 45-row shape forced (HBCU_NLMEANS_V3F_RS=45; on their own,
frames this small take the 20-row shape): patch 3/5/7 with one and two frames, heights one below, at and one above a box
edge, the 45-row strip and the 540-row tile in luma and in chroma, widths that leave partial lanes, and flat, saturated,
striped and noisy content.  The same cases also run with the shape the handle picks.

The reference's results of these calls are stored in tests/golden/v3f_tall_ref_digests.json; `HBCU_RECORD_REF=1` with
the reference built re-records them from the CPU test of this file."""
import json
import re
from collections import namedtuple
from pathlib import Path

import numpy as np
import pytest

from golden_ref import GoldenRef
from handbrake_b200 import synth
from test_nlmeans_fused_r3_gpu import clip_content, clip_noise, planes

FMT8 = synth.PIX_FMT_YUV420P
STORE = Path(__file__).resolve().parent / "golden" / "v3f_tall_ref_digests.json"
NLMEANS_CU = Path(__file__).resolve().parent.parent / "handbrake_b200" / "csrc" / "nlmeans.cu"

# nlmeans.cu: kV3Fused (12 warps x 20 rows), kV3FusedTall (12 x 30), kV3FusedTaller (12 x 45), kV3FusedWarmRows
WARPS, SHORT, TALL, TALLER, WARM = 12, 20, 30, 45, 7
HALO = 8                                          # kHalo: tile row t is output row t - HALO
STRIP, TILE = TALLER, WARPS * TALLER
LOADS = -(-(TILE + 2 * HALO) // 256)              # V3FusedLayout::kLoads: a TMA box has at most 256 rows
BOX = (-(-(TILE + 2 * HALO) // LOADS) + 3) // 4 * 4   # V3FusedLayout::kBoxRows
BOX_EDGE = BOX - HALO                             # the first output row of the second box


class TallRef(GoldenRef):
    """GoldenRef over this file's own store of reference digests"""

    def __init__(self):
        super().__init__()
        self.store = json.loads(STORE.read_text()) if STORE.exists() else {}

    def _save(self):
        STORE.write_text(json.dumps(dict(sorted(self.store.items())), indent=0) + "\n")


@pytest.fixture(scope="module")
def ref():
    return TallRef()


CLIPS = {"noise": clip_noise, "content": clip_content}
Case = namedtuple("Case", "id settings w h n clip")


def _patch_and_frames():
    return [Case(f"p{p}-nf{nf}", planes(p, nf), 257, TILE + BOX + 5, 3, ("noise", 300 + p)) for p in (3, 5, 7) for nf in (1, 2)]


def _edges():
    """heights one below, at and one above a box edge, the strip and the tile, in luma (h) and in chroma ((h + 1) / 2);
    widths whose last lane holds 3 or 1 pixels, or ends a tile"""
    edges = (BOX_EDGE, STRIP, TILE)
    hs = sorted({e + d for e in edges for d in (-1, 0, 1)} | {2 * e + d for e in edges for d in (-3, -1, 1)})
    return [Case(f"edge-{w}x{h}", planes(7, 2), w, h, 3, ("noise", 13 * w + h)) for w in (127, 129, 256) for h in hs]


def _content():
    return [Case(f"content-p{p}-nf{nf}", planes(p, nf), 161, TILE + 3, 7, ("content", 10 + p)) for p in (3, 5, 7) for nf in (1, 2)]


CASES = _patch_and_frames() + _edges() + _content()


def make_clip(c):
    kind, seed = c.clip
    return CLIPS[kind](c.w, c.h, c.n, seed)


def ref_run(ref, c, clip):
    return ref.run("hb_filter_nlmeans", c.settings + ":threads=2", clip, FMT8, c.w, c.h)


# ---------------------------------------------------------------------------------------------------------- shape rule
def tiles(w, h, rs):
    """CTAs of one 4:2:0 frame (three planes) at strips of rs rows"""
    dims = [(w, h), ((w + 1) // 2, (h + 1) // 2), ((w + 1) // 2, (h + 1) // 2)]
    return sum(-(-pw // 128) * -(-ph // (WARPS * rs)) for pw, ph in dims)


def sm_rows(w, h, rs):
    return tiles(w, h, rs) * (rs + WARM)


def pick_rs(w, h, sms):
    """v3f_pick_rs: a taller shape only with at least one CTA per SM; of 30 and 45 the fewer CTAs x (RS + WARM)"""
    if tiles(w, h, TALLER) >= sms and sm_rows(w, h, TALLER) < sm_rows(w, h, TALL):
        return TALLER
    return TALL if tiles(w, h, TALL) >= sms else SHORT


def test_shape_rule():
    """the rule for an H100 SXM (132 SMs): 20 rows below 4K, 45 from 4K up and on a letterboxed 4K frame"""
    sms = 132
    assert [tiles(1920, 1080, rs) for rs in (SHORT, TALL, TALLER)] == [123, 77, 46]
    assert [tiles(3840, 2160, rs) for rs in (SHORT, TALL, TALLER)] == [420, 270, 180]
    assert [tiles(3840, 1600, rs) for rs in (SHORT, TALL, TALLER)] == [330, 240, 150]
    assert [tiles(7680, 4320, rs) for rs in (SHORT, TALL, TALLER)] == [1620, 1080, 720]
    assert pick_rs(640, 360, sms) == SHORT
    assert pick_rs(1920, 1080, sms) == SHORT
    assert pick_rs(3840, 2160, sms) == TALLER
    assert pick_rs(3840, 1600, sms) == TALLER
    assert pick_rs(7680, 4320, sms) == TALLER


def test_shapes_match_kernel():
    """WARPS, SHORT, TALL, TALLER and WARM restate nlmeans.cu"""
    src = NLMEANS_CU.read_text()
    assert f"constexpr V3Shape kV3Fused = {{ {WARPS}, {SHORT} }};" in src
    assert f"constexpr V3Shape kV3FusedTall = {{ {WARPS}, {TALL} }};" in src
    assert f"constexpr V3Shape kV3FusedTaller = {{ {WARPS}, {TALLER} }};" in src
    assert f"constexpr int kV3FusedWarmRows = {WARM};" in src
    assert "long v3f_sm_rows(const PlaneGeom *g, int rs) { return (long)v3f_tiles(g, rs) * (rs + kV3FusedWarmRows); }" in src
    assert re.search(r"if \(v3f_tiles\(g, kV3FusedTaller\.rs\) >= sms && v3f_sm_rows\(g, kV3FusedTaller\.rs\) < "
                     r"v3f_sm_rows\(g, kV3FusedTall\.rs\)\) return kV3FusedTaller\.rs;", src)


def test_cases_straddle_the_tall_shape():
    luma = {c.h for c in CASES}
    chroma = {(h + 1) // 2 for h in luma}
    assert (LOADS, BOX) == (3, 188)
    for edge in (BOX_EDGE, STRIP, TILE):
        assert {edge - 1, edge, edge + 1} <= luma and {edge - 1, edge, edge + 1} <= chroma, edge
    assert {c.w % 128 for c in CASES} >= {127, 1, 0}


# ------------------------------------------------------------------------------------------------------------- parity
@pytest.mark.parametrize("c", CASES, ids=[c.id for c in CASES])
def test_restatement_matches_reference(ref, c):
    """the plain-C restatement reproduces the reference's stored result for every case"""
    r = ref_run(ref, c, make_clip(c))
    assert r.saw_eof and r.frames.shape == (c.n, synth.frame_bytes(FMT8, c.w, c.h))


@pytest.mark.gpu
@pytest.mark.parametrize("rs", [str(TALLER), ""], ids=["taller", "picked"])
@pytest.mark.parametrize("c", CASES, ids=[c.id for c in CASES])
def test_cuda_matches_reference(ref, cuda_filters, monkeypatch, c, rs):
    if rs:
        monkeypatch.setenv("HBCU_NLMEANS_V3F_RS", rs)
    else:
        monkeypatch.delenv("HBCU_NLMEANS_V3F_RS", raising=False)
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
