"""ctypes binding of hb_harness.h: run libhb-style filter objects over numpy frames.

`FilterLib(path)` wraps any shared library that exports `hb_filter_*` objects and
the harness (`hb_harness_run_chain`): the product's libhbcu_filters.so, or -- from
tests only -- the reference build oracle/_ref/libhbref.so.
"""
import ctypes as C
import numpy as np

from . import synth


class HarnessIO(C.Structure):
    _fields_ = [
        ("pix_fmt", C.c_int), ("width", C.c_int), ("height", C.c_int),
        ("n_in", C.c_int),
        ("in_", C.c_void_p), ("in_flags", C.c_void_p), ("in_combed", C.c_void_p),
        ("out", C.c_void_p), ("out_capacity", C.c_int),
        ("out_combed", C.c_void_p), ("out_flags", C.c_void_p),
        ("out_start", C.c_void_p), ("out_stop", C.c_void_p), ("out_duration", C.c_void_p),
        ("n_out", C.c_int), ("n_dropped", C.c_int), ("saw_eof", C.c_int),
        ("init_failed", C.c_int), ("vrate_num_out", C.c_int), ("vrate_den_out", C.c_int),
        ("in_start", C.c_void_p), ("in_stop", C.c_void_p), ("in_new_chap", C.c_void_p),
        ("vrate_num", C.c_int), ("vrate_den", C.c_int), ("cfr", C.c_int), ("collect_info", C.c_int),
        ("out_new_chap", C.c_void_p), ("cfr_out", C.c_int), ("info_text", C.c_char * 128),
        ("par_num", C.c_int), ("par_den", C.c_int),
        ("par_num_out", C.c_int), ("par_den_out", C.c_int), ("width_out", C.c_int), ("height_out", C.c_int),
    ]


class HarnessOverlay(C.Structure):
    _fields_ = [("frame", C.c_int), ("x", C.c_int), ("y", C.c_int), ("width", C.c_int), ("height", C.c_int),
                ("yuva", C.c_void_p)]


class HarnessBlend(C.Structure):
    _fields_ = [("blend", C.c_void_p), ("overlay_pix_fmt", C.c_int), ("chroma_location", C.c_int),
                ("n_overlays", C.c_int), ("overlays", C.c_void_p), ("n_changed", C.c_int), ("changed", C.c_void_p),
                ("guard_x", C.c_int), ("guard_y", C.c_int),
                ("guard_damaged", C.c_int), ("same_buffer", C.c_int), ("frames", C.c_int)]


# the render_sub stand-in of the harness (hb_harness.h): put it in a chain with run_blend()
RENDER_SUB = "hb_filter_render_sub_harness"


class FilterResult:
    def __init__(self):
        self.frames = None
        self.combed = None
        self.flags = None
        self.start = None
        self.stop = None
        self.duration = None
        self.saw_eof = False
        self.init_failed = 0
        self.vrate = (0, 0)
        self.n_dropped = 0
        self.new_chap = None
        self.cfr = 0
        self.info = ""
        self.width = self.height = 0          # the output geometry and PAR (init->geometry after every init())
        self.par = (1, 1)


class FilterLib:
    def __init__(self, path):
        self.path = str(path)
        self.lib = C.CDLL(self.path, mode=C.RTLD_LOCAL)
        self.lib.hb_harness_run_chain.restype = C.c_int
        self.lib.hb_harness_run_chain.argtypes = [C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_char_p), C.POINTER(HarnessIO)]
        self.lib.hb_harness_frame_bytes.restype = C.c_size_t
        self.lib.hb_harness_frame_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
        self.lib.hb_shim_buffers_alive.restype = C.c_long
        self.lib.hb_shim_set_log_level.argtypes = [C.c_int]
        self.lib.hb_shim_set_cpu_count.argtypes = [C.c_int]
        self.lib.hb_shim_set_log_level(-1)

    def filter_object(self, name):
        """address of the exported hb_filter_object_t `name` (e.g. 'hb_filter_nlmeans')"""
        return C.addressof(C.c_char.in_dll(self.lib, name))

    def run_blend(self, blend, overlays, overlay_pix_fmt, filters, settings, frames, pix_fmt, width, height,
                  chroma_location=2, changed=None, guard=(0, 0), **kw):
        """run a chain holding RENDER_SUB, which burns `overlays` into the frames through the exported blend object
        `blend` ('hb_blend', 'hb_blend_cuda').  overlays: (frame, x, y, width, height, yuva) in list order, yuva the
        overlay's planes Y, Cb, Cr, A packed at their widths (uint8); changed: per-frame flags (default 1);
        guard: (columns, rows) of spare samples around host frames while the blend object works on them.
        Returns (FilterResult, dict(guard_damaged, same_buffer, frames))."""
        keep = [np.ascontiguousarray(o[5], dtype=np.uint8) for o in overlays]
        arr = (HarnessOverlay * max(1, len(overlays)))()
        for i, (o, data) in enumerate(zip(overlays, keep)):
            arr[i] = HarnessOverlay(int(o[0]), int(o[1]), int(o[2]), int(o[3]), int(o[4]), data.ctypes.data)
        ch = np.ascontiguousarray(changed if changed is not None else [], dtype=np.int32)
        cfg = HarnessBlend()
        cfg.blend = self.filter_object(blend)
        cfg.overlay_pix_fmt, cfg.chroma_location = int(overlay_pix_fmt), int(chroma_location)
        cfg.n_overlays, cfg.overlays = len(overlays), C.addressof(arr)
        cfg.n_changed, cfg.changed = len(ch), ch.ctypes.data
        cfg.guard_x, cfg.guard_y = int(guard[0]), int(guard[1])
        self.lib.hb_harness_set_blend.argtypes = [C.c_void_p]
        self.lib.hb_harness_set_blend(C.addressof(cfg))
        try:
            r = self.run(filters, settings, frames, pix_fmt, width, height, **kw)
        finally:
            self.lib.hb_harness_set_blend(None)
        return r, dict(guard_damaged=cfg.guard_damaged, same_buffer=cfg.same_buffer, frames=cfg.frames)

    def buffers_alive(self):
        return int(self.lib.hb_shim_buffers_alive())

    def set_cpu_count(self, n):
        self.lib.hb_shim_set_cpu_count(int(n))

    def run(self, filters, settings, frames, pix_fmt, width, height, flags=None, combed=None,
            max_out=None, out_scale=1, start=None, stop=None, new_chap=None, vrate=None, cfr=0, info=False, par=None):
        """filters: list of exported object names; settings: list of 'k=v:k=v' strings (or None).
        frames: (n, frame_bytes) uint8 array.  start / stop / new_chap: per-frame input times and chapter marks
        (default i*3003, (i+1)*3003, i); vrate: (num, den) of the input (default 30000/1001); cfr: init->cfr;
        info: fill FilterResult.info with the last info() text; par: (num, den) of the input (default 1:1).
        Returns FilterResult, whose width / height / par are the output's."""
        if isinstance(filters, str):
            filters, settings = [filters], [settings]
        frames = np.ascontiguousarray(frames, dtype=np.uint8)
        n_in = frames.shape[0]
        fb = int(self.lib.hb_harness_frame_bytes(pix_fmt, width, height))     # any format the shim knows
        assert frames.shape[1] == fb, (frames.shape, fb)
        cap = max_out if max_out is not None else (n_in * 2 * out_scale + 8)
        out = np.zeros((cap, fb), dtype=np.uint8)
        o_combed = np.zeros(cap, dtype=np.uint8)
        o_flags = np.zeros(cap, dtype=np.uint16)
        o_start = np.zeros(cap, dtype=np.int64)
        o_stop = np.zeros(cap, dtype=np.int64)
        o_dur = np.zeros(cap, dtype=np.float64)
        io = HarnessIO()
        io.pix_fmt, io.width, io.height, io.n_in = pix_fmt, width, height, n_in
        io.in_ = frames.ctypes.data
        keep = [frames]
        if flags is not None:
            fl = np.ascontiguousarray(flags, dtype=np.uint16); keep.append(fl)
            io.in_flags = fl.ctypes.data
        if combed is not None:
            cb = np.ascontiguousarray(combed, dtype=np.uint8); keep.append(cb)
            io.in_combed = cb.ctypes.data
        for name, arr, dt in (("in_start", start, np.int64), ("in_stop", stop, np.int64), ("in_new_chap", new_chap, np.int32)):
            if arr is not None:
                a = np.ascontiguousarray(arr, dtype=dt); keep.append(a)
                assert a.shape == (n_in,), (name, a.shape)
                setattr(io, name, a.ctypes.data)
        if vrate is not None:
            io.vrate_num, io.vrate_den = int(vrate[0]), int(vrate[1])
        io.cfr, io.collect_info = int(cfr), int(bool(info))
        if par is not None:
            io.par_num, io.par_den = int(par[0]), int(par[1])
        o_chap = np.zeros(cap, dtype=np.int32)
        io.out_new_chap = o_chap.ctypes.data
        io.out, io.out_capacity = out.ctypes.data, cap
        io.out_combed, io.out_flags = o_combed.ctypes.data, o_flags.ctypes.data
        io.out_start, io.out_stop, io.out_duration = o_start.ctypes.data, o_stop.ctypes.data, o_dur.ctypes.data
        n = len(filters)
        protos = (C.c_void_p * n)(*[self.filter_object(f) for f in filters])
        sets = (C.c_char_p * n)(*[(s.encode() if s else None) for s in settings])
        rc = self.lib.hb_harness_run_chain(n, protos, sets, C.byref(io))
        if rc != 0:
            raise RuntimeError(f"filter chain {filters} failed (HB_FILTER_FAILED)")
        r = FilterResult()
        k = io.n_out
        r.frames, r.combed, r.flags = out[:k], o_combed[:k], o_flags[:k]
        r.start, r.stop, r.duration = o_start[:k], o_stop[:k], o_dur[:k]
        r.saw_eof, r.init_failed = bool(io.saw_eof), io.init_failed
        r.vrate, r.n_dropped = (io.vrate_num_out, io.vrate_den_out), io.n_dropped
        r.new_chap, r.cfr, r.info = o_chap[:k], io.cfr_out, io.info_text.decode()
        r.width, r.height, r.par = io.width_out, io.height_out, (io.par_num_out, io.par_den_out)
        return r
