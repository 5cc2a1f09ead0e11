"""Generates tests/golden/ref_lib_golden.json from the reference itself (oracle/_ref/libhbref.so, built by oracle/Makefile
from the HandBrake sources): what the tests that call the reference's library directly, rather than its filter objects,
compare with -- digests of the settings templates of the filter objects (test_abi.py) and the EEDI2 corner-filter stages
(test_oracle.py).  python tests/golden/make_ref_lib_golden.py"""
import ctypes as C
import json
import sys
from pathlib import Path

import numpy as np

TESTS = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(TESTS))
sys.path.insert(0, str(TESTS.parent))

from golden_ref import REF_SO, _h  # noqa: E402
from handbrake_b200.hblib import FilterLib  # noqa: E402
import test_oracle as T  # noqa: E402


class Head(C.Structure):
    _fields_ = [("pad", C.c_byte * 96), ("settings_template", C.c_char_p)]


def main():
    ref = FilterLib(REF_SO)
    out = {"templates": {}, "eedi2_stages": {}, "eedi2_chain_luma": {}}
    for name in ("nlmeans", "comb_detect", "decomb", "lapsharp", "unsharp", "chroma_smooth", "denoise", "detelecine"):
        out["templates"]["hb_filter_" + name] = _h(Head.in_dll(ref.lib, "hb_filter_" + name).settings_template.decode())
    P = lambda a: a.ctypes.data_as(C.c_void_p)
    for depth in (8, 10):
        sfx = "16" if depth > 8 else "8"
        for w, h, pitch in T.EEDI2_PP_GEOMETRY:
            src = T._pp_planes(depth, w, h, pitch, 3)
            g = {}
            ra, rt = src.copy(), np.zeros_like(src)
            getattr(ref.lib, "eedi2_gaussian_blur1_" + sfx)(P(ra), pitch, P(rt), pitch, P(ra), pitch, h, w)
            g["blur1"] = _h(ra, rt)
            rd = [np.zeros((h + 2, pitch), np.int32) for _ in range(3)]
            getattr(ref.lib, "eedi2_calc_derivatives_" + sfx)(P(ra), pitch, h, w, P(rd[0]), P(rd[1]), P(rd[2]), depth)
            g["derivatives"] = _h(*rd)
            g["blur_sqrt2"] = []
            for a in rd:
                rtmp = np.zeros_like(a)
                getattr(ref.lib, "eedi2_gaussian_blur_sqrt2_" + sfx)(P(a), P(rtmp), P(a), pitch, h, w)
                g["blur_sqrt2"].append(_h(a, rtmp))
            H = 2 * h
            msk = T._pp_mask(depth, w, H, pitch, src.dtype)
            g["corner"] = []
            for field in (0, 1):
                rdst = T._pp_planes(depth, w, H, pitch, 5)
                getattr(ref.lib, "eedi2_post_process_corner_" + sfx)(P(rd[0]), P(rd[1]), P(rd[2]), pitch, P(msk), pitch, P(rdst), pitch, H, w, field, depth)
                g["corner"].append(_h(rdst))
            out["eedi2_stages"][f"{depth}_{w}x{h}_{pitch}"] = g
        libc = C.CDLL(None)
        w, h = T.EEDI2_CHAIN_GEOMETRY
        clip, flags, _ = T.decomb_inputs(depth, w, h, 4, seed=13)
        for pp in (2, 3):
            libc.mallopt(-3, 4096)                     # M_MMAP_THRESHOLD: every sizeable malloc is a fresh zeroed mapping
            try:
                r = ref.run("hb_filter_decomb", f"mode=24:postproc={pp}", clip, T.FMT[depth], w, h, flags=flags)
            finally:
                libc.mallopt(-3, 128 * 1024)
            out["eedi2_chain_luma"][f"{depth}_{pp}"] = _h(np.ascontiguousarray(r.frames[:, T.eedi2_chain_rows(depth, w, h)]))
    (Path(__file__).parent / "ref_lib_golden.json").write_text(json.dumps(out, indent=1) + "\n")


if __name__ == "__main__":
    main()
