"""GPU: frame-sharded runs of the CUDA filter objects == their unsharded run == the reference (SURVEY.md 8e; VERDICT r1
(e)(iv): round 1 checked comb-detect / decomb / lapsharp sharding with the CPU objects only).  Every block is a fresh
filter instance on the device, fed its frames plus the temporal halo of handbrake_b200.sharding; halo outputs are
dropped.  With two GPUs visible consecutive blocks alternate between them (HBCU_DEVICE)."""
import ctypes as C
import os

import numpy as np
import pytest

import handbrake_b200
from handbrake_b200 import sharding, synth
from test_oracle import decomb_inputs

pytestmark = pytest.mark.gpu


def ndev():
    return C.CDLL(str(handbrake_b200.LIBHBCU)).hbcu_device_count()


def sharded(blocks, world, clip_of, run, k=1):
    parts = {}
    for rank in range(world):
        os.environ["HBCU_DEVICE"] = str(rank % max(1, min(ndev(), world)))
        try:
            parts.update(sharding.run_rank(blocks, rank, clip_of, run, outputs_per_frame=k))
        finally:
            os.environ.pop("HBCU_DEVICE", None)
    return np.concatenate([parts[b.index] for b in blocks])


@pytest.mark.parametrize("world,block", [(2, 3), (4, 2)])
@pytest.mark.parametrize("depth", [8, 10])
def test_sharded_cuda_comb_detect_decomb_lapsharp(ref, cuda_filters, world, block, depth):
    w, h = 352, 288
    fmt = synth.PIX_FMT_YUV420P if depth == 8 else synth.PIX_FMT_YUV420P10
    clip, flags, combed = decomb_inputs(depth, w, h, 10, seed=4)
    n = clip.shape[0]
    blocks = sharding.plan_blocks(n, world, block, halo_before=1, halo_after=1)
    win = {}

    def clip_of(a, b):
        win["r"] = (a, b)
        return clip[a:b]

    s = "mode=3:motion-thresh=1:spatial-thresh=1"

    def comb(fr):
        a, b = win["r"]
        return np.asarray(cuda_filters.run("hb_filter_comb_detect_cuda", s, fr, fmt, w, h, flags=flags[a:b]).combed, np.uint8).reshape(-1, 1)
    whole = np.asarray(ref.run("hb_filter_comb_detect", s, clip, fmt, w, h, flags=flags).combed, np.uint8)
    assert np.array_equal(sharded(blocks, world, clip_of, comb).ravel(), whole)

    for mode, k, tags in ((7, 1, None), (39, 1, combed), (23, 2, None), (4, 1, None), (2, 1, None)):
        def decomb(fr):
            a, b = win["r"]
            return cuda_filters.run("hb_filter_decomb_cuda", f"mode={mode}", fr, fmt, w, h, flags=flags[a:b],
                                    combed=None if tags is None else tags[a:b]).frames
        whole = ref.run("hb_filter_decomb", f"mode={mode}", clip, fmt, w, h, flags=flags, combed=tags).frames
        assert np.array_equal(sharded(blocks, world, clip_of, decomb, k), whole), mode

    nohalo = sharding.plan_blocks(n, world, block)
    lap = lambda fr: cuda_filters.run("hb_filter_lapsharp_cuda", "y-strength=0.3:y-kernel=isolap", fr, fmt, w, h).frames
    assert np.array_equal(sharded(nohalo, world, lambda a, b: clip[a:b], lap),
                          ref.run("hb_filter_lapsharp_mt", "y-strength=0.3:y-kernel=isolap", clip, fmt, w, h).frames)

    nf = 3
    before, after = sharding.nlmeans_halo(nf)
    nlm_blocks = sharding.plan_blocks(n, world, block, halo_before=before, halo_after=after)
    sn = f"y-strength=6:y-frame-count={nf}"
    nlm = lambda fr: cuda_filters.run("hb_filter_nlmeans_cuda", sn, fr, fmt, w, h).frames
    assert np.array_equal(sharded(nlm_blocks, world, lambda a, b: clip[a:b], nlm), ref.run("hb_filter_nlmeans", sn + ":threads=2", clip, fmt, w, h).frames)
    assert cuda_filters.buffers_alive() == 0
