"""CPU tests of the drop-in boundary: the C-ABI library loads without a GPU and exports every
function include/hbcu.h declares; the filter library exports the hb_filter_object_t drop-ins with
the reference's ids / settings templates; without a GPU, init() fails (no CPU fallback)."""
import ctypes as C
import re
from pathlib import Path

import numpy as np
import pytest

import handbrake_b200
from handbrake_b200 import synth

REPO = Path(__file__).resolve().parent.parent


def declared_functions():
    text = (REPO / "include" / "hbcu.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(hbcu_[a-z0-9_]+)\s*\(", text)))


def test_every_declared_symbol_is_exported():
    lib = C.CDLL(str(handbrake_b200.LIBHBCU))
    names = declared_functions()
    assert len(names) > 40
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, missing
    assert lib.hbcu_abi_version() == 6


def test_filter_objects_exported_with_reference_ids():
    flt = handbrake_b200.filters()

    class FilterObject(C.Structure):       # head of hb_filter_object_t (handbrake/common.h:1670-1680)
        _fields_ = [("id", C.c_int), ("enforce_order", C.c_int), ("skip", C.c_int), ("aliased", C.c_int),
                    ("name", C.c_char_p), ("short_name", C.c_char_p), ("settings", C.c_void_p),
                    ("init", C.c_void_p), ("init_thread", C.c_void_p), ("post_init", C.c_void_p),
                    ("work", C.c_void_p), ("work_thread", C.c_void_p), ("close", C.c_void_p), ("info", C.c_void_p),
                    ("settings_template", C.c_char_p)]

    expect = {"hb_filter_nlmeans_cuda": (16, b"nlmeans"), "hb_filter_comb_detect_cuda": (4, b"comb-detect"),
              "hb_filter_decomb_cuda": (6, b"decomb"), "hb_filter_lapsharp_cuda": (24, b"lapsharp"),
              "hb_filter_unsharp_cuda": (26, b"unsharp"), "hb_filter_chroma_smooth_cuda": (17, b"chromasmooth"),
              "hb_filter_denoise_cuda": (14, b"hqdn3d"), "hb_filter_detelecine_cuda": (3, b"detelecine")}
    for sym, (fid, short) in expect.items():
        obj = FilterObject.in_dll(flt.lib, sym)
        assert obj.id == fid and obj.short_name == short and obj.enforce_order == 1
        assert obj.init and obj.work and obj.close and obj.settings_template


def test_templates_match_reference():
    """same settings_template strings as the reference objects (the job engine validates settings against them; the
    digests of the reference's strings are stored in tests/golden/ref_lib_golden.json)"""
    from golden_ref import _h
    from test_oracle import ref_lib_golden
    flt = handbrake_b200.filters()
    want = ref_lib_golden()["templates"]

    class Head(C.Structure):
        _fields_ = [("pad", C.c_byte * 96), ("settings_template", C.c_char_p)]

    for a, b in (("hb_filter_nlmeans_cuda", "hb_filter_nlmeans"), ("hb_filter_comb_detect_cuda", "hb_filter_comb_detect"),
                 ("hb_filter_decomb_cuda", "hb_filter_decomb"), ("hb_filter_lapsharp_cuda", "hb_filter_lapsharp"),
                 ("hb_filter_unsharp_cuda", "hb_filter_unsharp"), ("hb_filter_chroma_smooth_cuda", "hb_filter_chroma_smooth"),
                 ("hb_filter_denoise_cuda", "hb_filter_denoise"), ("hb_filter_detelecine_cuda", "hb_filter_detelecine")):
        assert _h(Head.in_dll(flt.lib, a).settings_template.decode()) == want[b], a


def test_no_cpu_fallback_without_gpu():
    """no usable device -> init() != 0 -> the harness (like libhb, work.c:1861-1868) drops the filter"""
    lib = C.CDLL(str(handbrake_b200.LIBHBCU))
    if lib.hbcu_device_count() > 0:
        pytest.skip("a GPU is present")
    flt = handbrake_b200.filters()
    w, h = 64, 48
    clip = synth.progressive_clip(synth.PIX_FMT_YUV420P, w, h, 2)
    for name in ("hb_filter_nlmeans_cuda", "hb_filter_comb_detect_cuda", "hb_filter_decomb_cuda", "hb_filter_lapsharp_cuda",
                 "hb_filter_unsharp_cuda", "hb_filter_chroma_smooth_cuda", "hb_filter_denoise_cuda", "hb_filter_detelecine_cuda",
                 "hb_filter_hbcu_upload"):
        g = flt.run(name, None, clip, synth.PIX_FMT_YUV420P, w, h)
        assert g.init_failed == 1 and np.array_equal(g.frames, clip)
    lib.hbcu_last_error.restype = C.c_char_p


def test_oracle_is_not_linked_into_the_product():
    import subprocess
    for so in (handbrake_b200.LIBHBCU, handbrake_b200.LIBHBCU_FILTERS):
        out = subprocess.run(["nm", "-D", str(so)], capture_output=True, text=True).stdout
        assert "oracle_" not in out


def test_product_filter_library_carries_no_libhb_stand_in():
    """VERDICT r1 hygiene: libhbcu_filters.so is the filter objects alone.  What libhb provides (hb_buffer_*, hb_dict_*,
    hb_log ...) is UNDEFINED in it and, outside a HandBrake build, resolved by the separate test scaffolding libhbshim.so;
    the harness and the bench driver live there too."""
    import subprocess
    nm = subprocess.run(["nm", "-D", str(handbrake_b200.LIBHBCU_FILTERS)], capture_output=True, text=True).stdout.splitlines()
    defined = {l.split()[-1] for l in nm if len(l.split()) == 3 and l.split()[1] in "TDBR"}
    undefined = {l.split()[-1] for l in nm if l.split()[0] == "U"}
    assert {"hb_filter_nlmeans_cuda", "hb_filter_decomb_cuda", "hb_filter_get"} <= defined
    for sym in ("hb_buffer_init", "hb_frame_buffer_init", "hb_buffer_close", "hb_dict_extract_int", "hb_log"):
        assert sym in undefined and sym not in defined, sym
    assert not [s for s in defined if s.startswith(("hb_harness_", "hb_bench_", "hb_shim_"))]
    shim = handbrake_b200.LIB_DIR / "libhbshim.so"
    sh = subprocess.run(["nm", "-D", str(shim)], capture_output=True, text=True).stdout
    assert " T hb_harness_run_chain" in sh and " T hb_bench_stream" in sh and " T hb_buffer_init" in sh
    assert "hbcu_" not in "\n".join(l for l in sh.splitlines() if " U " in l)      # the stand-in knows nothing of the product

