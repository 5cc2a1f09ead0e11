"""The reference's filter objects, as the suite sees them without the reference.

Every `ref.run(...)` call of the suite was made once against the reference's own filters (oracle/_ref/libhbref.so, built
by oracle/Makefile from the HandBrake sources) and the digest of its result stored in tests/golden/ref_digests.json,
keyed by a digest of the call (filter objects, settings, input frames, flags, tags, geometry).

`GoldenRef.run` answers a call with the product's host-side filters over the plain-C restatement of the kernels
(oracle/_ref/libhostlogic.so, always built) and checks that the answer has the stored digest of the reference's result
before it hands it out: a test that compares with `ref` compares with the reference's output, bit for bit, on a machine
that never had the reference.  A call the store does not know is an error, not a skip.

Calls on full-size frames, where the restatement would take minutes, are made with `digest_only=True`: the store keeps
per-frame digests and the small per-frame fields of the reference's result, and `run` returns them as a `RecordedResult`
for the test to compare the CUDA result with.

With HBCU_RECORD_REF=1 and the reference built, calls go to the reference itself and their digests are added to the
store (see tests/golden/README.md).
"""
import hashlib
import json
import os
from pathlib import Path

import numpy as np

REPO = Path(__file__).resolve().parent.parent
STORE = Path(__file__).resolve().parent / "golden" / "ref_digests.json"
REF_SO = REPO / "oracle" / "_ref" / "libhbref.so"
HOSTLOGIC_SO = REPO / "oracle" / "_ref" / "libhostlogic.so"


class FilterFailed(RuntimeError):
    pass


def _h(*parts):
    m = hashlib.sha256()
    for p in parts:
        if isinstance(p, np.ndarray):
            p = np.ascontiguousarray(p)
            m.update(repr((p.dtype.str, p.shape)).encode())
            m.update(p.tobytes())
        else:
            m.update(repr(p).encode())
        m.update(b"\0")
    return m.hexdigest()[:20]


def call_key(filters, settings, frames, pix_fmt, width, height, flags=None, combed=None, max_out=None, out_scale=1, cpu_count=0):
    """cpu_count: the worker count set with set_cpu_count (0: the machine's own, left out of the key)"""
    if isinstance(filters, str):
        filters, settings = [filters], [settings]
    frames = np.ascontiguousarray(frames, dtype=np.uint8)
    fl = None if flags is None else np.ascontiguousarray(flags, dtype=np.uint16)
    cb = None if combed is None else np.ascontiguousarray(combed, dtype=np.uint8)
    parts = [list(filters), list(settings), int(pix_fmt), int(width), int(height), max_out, out_scale, frames, fl, cb]
    return _h(*(parts + [("cpu_count", int(cpu_count))] if cpu_count else parts))


def result_digest(r):
    """everything a FilterResult carries"""
    if isinstance(r, FilterFailed):
        return "failed"
    return _h(np.asarray(r.frames), np.asarray(r.combed), np.asarray(r.flags), np.asarray(r.start), np.asarray(r.stop),
              np.asarray(r.duration), bool(r.saw_eof), int(r.init_failed), tuple(int(v) for v in r.vrate), int(r.n_dropped))


def product_names(filters, settings):
    """the reference's objects -> the product's objects of the same filters (the multi-threaded wrappers of lapsharp,
    unsharp and chroma smooth compute what the plain objects compute)"""
    out = []
    for f in filters:
        base = f[:-3] if f.endswith("_mt") else f
        out.append(base + "_cuda")
    return out, list(settings)


def frame_digests(frames):
    return [_h(np.ascontiguousarray(f))[:12] for f in frames]


class RecordedResult:
    """the stored result of a digest_only call: per-frame digests instead of the frames"""

    def __init__(self, d):
        self.shape = tuple(d["shape"])
        self.frame_digests = d["frames"]
        self.start, self.stop = np.array(d["start"], np.int64), np.array(d["stop"], np.int64)
        self.combed, self.flags = np.array(d["combed"], np.uint8), np.array(d["flags"], np.uint16)
        self.vrate, self.saw_eof, self.init_failed = tuple(d["vrate"]), d["saw_eof"], d["init_failed"]

    @staticmethod
    def record(r):
        return dict(shape=list(r.frames.shape), frames=frame_digests(r.frames), start=[int(v) for v in r.start],
                    stop=[int(v) for v in r.stop], combed=[int(v) for v in r.combed], flags=[int(v) for v in r.flags],
                    vrate=[int(v) for v in r.vrate], saw_eof=bool(r.saw_eof), init_failed=int(r.init_failed))

    def frames_differing(self, frames):
        """indices of the frames of `frames` that differ from the reference's"""
        return [i for i, (a, b) in enumerate(zip(frame_digests(frames), self.frame_digests)) if a != b]


class GoldenRef:
    def __init__(self):
        from handbrake_b200.hblib import FilterLib
        self.recording = os.environ.get("HBCU_RECORD_REF") == "1"
        self.cpu_count = 0
        self.store = json.loads(STORE.read_text()) if STORE.exists() else {}
        if self.recording:
            self.lib = FilterLib(REF_SO)
        self.host = FilterLib(HOSTLOGIC_SO)

    def _save(self):
        STORE.write_text(json.dumps(dict(sorted(self.store.items())), indent=0) + "\n")

    def set_cpu_count(self, n):
        """the worker count (hb_get_cpu_count) of the following calls: part of their key, so that each count's stored
        result is checked on its own; the host filters answering a call run with the same count"""
        self.cpu_count = int(n)
        (self.lib if self.recording else self.host).set_cpu_count(n)

    def buffers_alive(self):
        return (self.lib if self.recording else self.host).buffers_alive()

    def run(self, filters, settings, frames, pix_fmt, width, height, flags=None, combed=None, max_out=None, out_scale=1,
            digest_only=False):
        if isinstance(filters, str):
            filters, settings = [filters], [settings]
        key = call_key(filters, settings, frames, pix_fmt, width, height, flags, combed, max_out, out_scale, self.cpu_count)
        kw = dict(flags=flags, combed=combed, max_out=max_out, out_scale=out_scale)
        if self.recording:
            try:
                r = self.lib.run(filters, settings, frames, pix_fmt, width, height, **kw)
            except RuntimeError as e:
                r = FilterFailed(str(e))
            if isinstance(r, FilterFailed):
                self.store[key] = "failed"
                self._save()
                raise r
            self.store[key] = RecordedResult.record(r) if digest_only else result_digest(r)
            self._save()
            return RecordedResult(self.store[key]) if digest_only else r
        want = self.store.get(key)
        if want is None:
            raise KeyError(f"no stored reference result for {filters} {settings} {width}x{height} ({key}): "
                           "record it with HBCU_RECORD_REF=1 where the reference is built")
        if digest_only:
            return RecordedResult(want)
        names, sets = product_names(filters, settings)
        try:
            r = self.host.run(names, sets, frames, pix_fmt, width, height, **kw)
        except RuntimeError as e:
            r = FilterFailed(str(e))
        got = result_digest(r)
        assert got == want, f"the CPU restatement of {filters} {settings} {width}x{height} no longer reproduces the reference's result"
        if isinstance(r, FilterFailed):
            raise RuntimeError(f"filter chain {filters} failed (HB_FILTER_FAILED)")
        return r
