"""Deterministic synthetic yuv420p frames (SURVEY.md 8d) as packed planar numpy arrays.

A frame is one 1-D uint8 array: Y plane, then U, then V, rows tightly packed
(row pitch = width * bytes-per-sample) -- the layout hb_harness.c expects.
Noise comes from a counter-based integer hash of (x, y, t, plane, seed) so any
frame can be generated independently (needed when frames are sharded over ranks).
"""
import numpy as np

PIX_FMT_YUV420P = 0        # values follow the shim's enum AVPixelFormat
PIX_FMT_YUV420P10 = 62
PIX_FMT_YUV420P12 = 123
# semi-planar 4:2:0 (what NVDEC decodes into): Y, then one plane of Cb/Cr pairs; P010 keeps 10 bits in the high bits
PIX_FMT_NV12 = 23
PIX_FMT_P010 = 158
PIX_FMT_P016 = 169

PIC_FLAG_TOP_FIELD_FIRST = 0x0008
PIC_FLAG_PROGRESSIVE_FRAME = 0x0010


def depth_of(pix_fmt):
    return {PIX_FMT_YUV420P: 8, PIX_FMT_YUV420P10: 10, PIX_FMT_YUV420P12: 12}[pix_fmt]


def plane_dims(width, height):
    cw, ch = -((-width) >> 1), -((-height) >> 1)
    return [(width, height), (cw, ch), (cw, ch)]


def frame_bytes(pix_fmt, width, height):
    bps = 2 if depth_of(pix_fmt) > 8 else 1
    return sum(w * h for w, h in plane_dims(width, height)) * bps


def _hash32(x, y, t, p, seed):
    """murmur-style finaliser over the pixel coordinates; uint32 in, uint32 out."""
    with np.errstate(over="ignore"):
        h = (x.astype(np.uint32) * np.uint32(0x9E3779B1)) ^ (y.astype(np.uint32) * np.uint32(0x85EBCA77))
        h ^= np.uint32((t * 0xC2B2AE3D + p * 0x27D4EB2F + seed) & 0xFFFFFFFF)
        h ^= h >> np.uint32(15)
        h *= np.uint32(0x2C1B3C6D)
        h ^= h >> np.uint32(12)
        h *= np.uint32(0x297A2D39)
        h ^= h >> np.uint32(15)
    return h


def _noise(w, h, t, p, seed, amp):
    yy, xx = np.meshgrid(np.arange(h, dtype=np.uint32), np.arange(w, dtype=np.uint32), indexing="ij")
    r = _hash32(xx, yy, t, p, seed)
    return (r % np.uint32(2 * amp + 1)).astype(np.int32) - amp


def _luma_pattern(w, h, t, maxv, shift):
    yy, xx = np.meshgrid(np.arange(h, dtype=np.int32), np.arange(w, dtype=np.int32), indexing="ij")
    # moving 8x8 checker/gradient, kept in the mid range so noise does not clip everywhere
    base = (((xx // 8 + yy // 8 + t) * 7) & 0x7F) + 64
    return base << shift


def progressive_frame(pix_fmt, width, height, t, seed=12345, noise=8):
    depth = depth_of(pix_fmt)
    maxv = (1 << depth) - 1
    shift = depth - 8
    dt = np.uint16 if depth > 8 else np.uint8
    planes = []
    for p, (w, h) in enumerate(plane_dims(width, height)):
        n = _noise(w, h, t, p, seed, noise) << shift
        if p == 0:
            v = _luma_pattern(w, h, t, maxv, shift) + n
        else:
            v = (128 << shift) + n
        planes.append(np.clip(v, 0, maxv).astype(dt).reshape(-1))
    return np.concatenate(planes).view(np.uint8)


def interlaced_frame(pix_fmt, width, height, t, seed=12345, noise=2, static=False):
    """Even rows sampled at time 2t, odd rows at 2t+1, with a horizontally moving edge.
    `static=True` freezes the motion (both fields identical in time) -> not combed."""
    depth = depth_of(pix_fmt)
    maxv = (1 << depth) - 1
    shift = depth - 8
    dt = np.uint16 if depth > 8 else np.uint8
    planes = []
    for p, (w, h) in enumerate(plane_dims(width, height)):
        yy, xx = np.meshgrid(np.arange(h, dtype=np.int32), np.arange(w, dtype=np.int32), indexing="ij")
        field_t = np.where((yy & 1) == 0, 2 * t, 2 * t + 1) if not static else np.full_like(yy, 0)
        speed = 6 if p == 0 else 3
        period = max(w // 3, 16)
        pos = (xx + field_t * speed) % period
        if p == 0:
            bars = np.where(pos < period // 2, 200, 40)
            ramp = (yy * 3 // max(h // 32, 1)) & 0x0F
            v = (bars + ramp) << shift
        else:
            v = (np.where(pos < period // 2, 150, 100)) << shift
        v = v + (_noise(w, h, 0 if static else t, p, seed, noise) << shift)
        planes.append(np.clip(v, 0, maxv).astype(dt).reshape(-1))
    return np.concatenate(planes).view(np.uint8)


def progressive_clip(pix_fmt, width, height, n, seed=12345, noise=8, t0=0):
    return np.stack([progressive_frame(pix_fmt, width, height, t0 + t, seed, noise) for t in range(n)])


def interlaced_clip(pix_fmt, width, height, n, seed=12345, static_every=5, t0=0):
    """>= 20 % static frames so the selective (not combed) decomb path is exercised."""
    frames = []
    for t in range(t0, t0 + n):
        frames.append(interlaced_frame(pix_fmt, width, height, t, seed, static=(static_every and t % static_every == static_every - 1)))
    return np.stack(frames)


def split_planes(frame, pix_fmt, width, height):
    depth = depth_of(pix_fmt)
    dt = np.uint16 if depth > 8 else np.uint8
    a = frame.view(dt)
    out, off = [], 0
    for w, h in plane_dims(width, height):
        out.append(a[off:off + w * h].reshape(h, w))
        off += w * h
    return out


PIC_FLAG_REPEAT_FIRST_FIELD = 0x0100


def weave(top_frame, bottom_frame, pix_fmt, width, height):
    """picture whose even lines come from top_frame and odd lines from bottom_frame (all planes)"""
    depth = depth_of(pix_fmt)
    dt = np.uint16 if depth > 8 else np.uint8
    out = []
    for a, b in zip(split_planes(top_frame, pix_fmt, width, height), split_planes(bottom_frame, pix_fmt, width, height)):
        c = a.copy()
        c[1::2] = b[1::2]
        out.append(c.astype(dt).reshape(-1))
    return np.concatenate(out).view(np.uint8)


def telecined_clip(pix_fmt, width, height, n_film, seed=12345, noise=3, tff=True, soft=False, video_tail=0):
    """24 -> 30 pulldown of n_film synthetic film frames (a multiple of 4 keeps the cadence whole).
    hard: fields woven 2:3:2:3 into pictures (At Ab | Bt Bb | Bt Cb | Ct Db | Dt Db for TFF), flags carry only the field order;
    soft: the film frames themselves with REPEAT_FIRST_FIELD on every other one, as an MPEG-2 soft-telecined stream has them.
    video_tail: that many truly interlaced pictures appended (the cadence breaks).  Returns (clip, flags)."""
    film = [progressive_frame(pix_fmt, width, height, 3 * t, seed, noise) for t in range(n_film)]
    order = PIC_FLAG_TOP_FIELD_FIRST if tff else 0
    frames, flags = [], []
    if soft:
        first_is_top = tff
        for t, f in enumerate(film):
            rff = t % 2 == 0
            frames.append(f)
            flags.append((PIC_FLAG_TOP_FIELD_FIRST if first_is_top else 0) | (PIC_FLAG_REPEAT_FIRST_FIELD if rff else 0) | PIC_FLAG_PROGRESSIVE_FRAME)
            if rff:
                first_is_top = not first_is_top
    else:
        fields = []                                     # film frame index per field, in display order
        for t in range(n_film):
            fields += [t] * (3 if t % 2 else 2)
        for k in range(0, len(fields) - 1, 2):
            first, second = film[fields[k]], film[fields[k + 1]]
            top, bottom = (first, second) if tff else (second, first)
            frames.append(weave(top, bottom, pix_fmt, width, height))
            flags.append(order)
    for t in range(video_tail):
        frames.append(interlaced_frame(pix_fmt, width, height, 100 + t, seed))
        flags.append(order)
    return np.stack(frames), np.array(flags, np.uint16)
