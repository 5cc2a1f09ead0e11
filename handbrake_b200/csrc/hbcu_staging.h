// hbcu_staging.h -- the host side of a one-frame-in, one-frame-out device operation (hbcu_format_*, hbcu_rotate_*):
// either side is a device frame or host planes at any linesize.  A host side is staged in a per-slot device buffer at
// hb_image_stride pitches (64-byte rows); a slot's staging is reused only after the events of its previous frame say
// so.  A device source is read in place and the kernel is recorded as one of its readers; a device destination is
// written in place behind the frame's previous readers.  Three streams: upload, kernel, download.
#pragma once
#include "hbcu_common.h"
#include "hbcu_frames.h"
#include "../../include/hbcu.h"

#include <vector>

namespace hbcu {

struct StagePlane { int row_bytes, rows, pitch; size_t off; };

struct Staging
{
    const char *who = "";                    // error prefix ("format", "rotate")
    int device = 0, slots = 0, next = 0;
    StagePlane in[3], out[3];                // a plane of 0 rows is absent (the third plane of a semi-planar side)
    size_t in_bytes = 0, out_bytes = 0;
    std::vector<uint8_t *> in_stage, out_stage;    // per slot, allocated on first use by a host side
    std::vector<int64_t> ticket;
    cudaStream_t s_h2d = nullptr, s_compute = nullptr, s_d2h = nullptr;
    std::vector<cudaEvent_t> ev_up, ev_k, ev_down;
    cudaEvent_t ev_mark[2] = {nullptr, nullptr};
};

// one side's planes back to back at hb_image_stride pitches; returns the bytes of one staged frame
inline size_t stage_layout(StagePlane g[3], const int row_bytes[3], const int rows[3])
{
    size_t off = 0;
    for (int p = 0; p < 3; p++)
    {
        g[p].row_bytes = row_bytes[p];
        g[p].rows = rows[p];
        g[p].pitch = (row_bytes[p] + 63) / 64 * 64;
        g[p].off = off;
        off += (size_t)g[p].pitch * rows[p];
    }
    return off;
}

// streams and events of `slots` slots on `device` (the caller has set in / out and the byte counts); -1 with the
// error set, after which the caller still calls stage_destroy
inline int stage_init(Staging *s, const char *who, int device, int slots)
{
    s->who = who;
    s->device = device;
    s->slots = slots;
    s->next = 0;
    s->in_stage.assign(slots, nullptr);
    s->out_stage.assign(slots, nullptr);
    s->ticket.assign(slots, -1);
    s->ev_up.assign(slots, nullptr);
    s->ev_k.assign(slots, nullptr);
    s->ev_down.assign(slots, nullptr);
#define CK(expr)                                                                  \
    do {                                                                          \
        cudaError_t _e = (expr);                                                  \
        if (_e != cudaSuccess) {                                                  \
            set_error("%s failed: %s", #expr, cudaGetErrorString(_e));            \
            return -1;                                                            \
        }                                                                         \
    } while (0)
    CK(cudaStreamCreateWithFlags(&s->s_h2d, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&s->s_compute, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&s->s_d2h, cudaStreamNonBlocking));
    for (int i = 0; i < slots; i++)
    {
        CK(cudaEventCreateWithFlags(&s->ev_up[i], cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&s->ev_k[i], cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&s->ev_down[i], cudaEventDisableTiming));
    }
    CK(cudaEventCreate(&s->ev_mark[0]));
    CK(cudaEventCreate(&s->ev_mark[1]));
#undef CK
    return 0;
}

// waits for the work in flight and frees everything
inline void stage_destroy(Staging *s)
{
    cudaSetDevice(s->device);
    if (s->s_h2d) cudaStreamSynchronize(s->s_h2d);
    if (s->s_compute) cudaStreamSynchronize(s->s_compute);
    if (s->s_d2h) cudaStreamSynchronize(s->s_d2h);
    for (auto p : s->in_stage) if (p) cudaFree(p);
    for (auto p : s->out_stage) if (p) cudaFree(p);
    for (auto e : s->ev_up) if (e) cudaEventDestroy(e);
    for (auto e : s->ev_k) if (e) cudaEventDestroy(e);
    for (auto e : s->ev_down) if (e) cudaEventDestroy(e);
    if (s->ev_mark[0]) cudaEventDestroy(s->ev_mark[0]);
    if (s->ev_mark[1]) cudaEventDestroy(s->ev_mark[1]);
    if (s->s_h2d) cudaStreamDestroy(s->s_h2d);
    if (s->s_compute) cudaStreamDestroy(s->s_compute);
    if (s->s_d2h) cudaStreamDestroy(s->s_d2h);
}

inline bool stage_frame_fits(const Staging *s, const hbcu_frame_t *f, const StagePlane g[3])
{
    if (f->device != s->device) return false;
    for (int p = 0; p < 3; p++)
    {
        if (f->rows[p] != g[p].rows || f->row_bytes[p] != g[p].row_bytes) return false;
        if (g[p].rows > 0 && f->plane[p] == nullptr) return false;
    }
    return true;
}

inline bool stage_host_fits(const void *const planes[3], const int strides[3], const StagePlane g[3])
{
    for (int p = 0; p < 3; p++)
        if (g[p].rows > 0 && (planes[p] == nullptr || strides[p] < g[p].row_bytes)) return false;
    return true;
}

// one frame: stages a host source, orders the kernel stream behind the source's producer and the destination's
// readers, calls launch(src, spitch, dst, dpitch) to queue the kernel on s_compute, and queues a host destination's
// copy-out.  Asynchronous; `ticket` names the frame for stage_wait / stage_poll.
template <class Launch>
int stage_submit(Staging *h, const char *fn, int64_t ticket,
                 hbcu_frame_t *in_frame, const void *const in_planes[3], const int in_strides[3],
                 hbcu_frame_t *out_frame, void *const out_planes[3], const int out_strides[3], Launch launch)
{
    if ((in_frame == nullptr && (in_planes == nullptr || in_strides == nullptr)) ||
        (out_frame == nullptr && (out_planes == nullptr || out_strides == nullptr)))
    {
        set_error("%s_%s: bad argument", h->who, fn);
        return -1;
    }
    if ((in_frame ? !stage_frame_fits(h, in_frame, h->in) : !stage_host_fits(in_planes, in_strides, h->in)) ||
        (out_frame ? !stage_frame_fits(h, out_frame, h->out) : !stage_host_fits(out_planes, out_strides, h->out)))
    {
        set_error("%s_%s: a frame's planes do not match the handle's geometry and formats", h->who, fn);
        return -1;
    }
    HBCU_CHECK(cudaSetDevice(h->device));
    const int s = h->next;
    const uint8_t *src[3];
    uint8_t *dst[3];
    int spitch[3], dpitch[3];
    if (in_frame == nullptr)
    {
        if (h->in_stage[s] == nullptr) HBCU_CHECK(cudaMalloc(&h->in_stage[s], h->in_bytes));
        // the slot's previous kernel has read the staging
        HBCU_CHECK(cudaStreamWaitEvent(h->s_h2d, h->ev_k[s], 0));
        for (int p = 0; p < 3; p++)
        {
            src[p] = h->in_stage[s] + h->in[p].off;
            spitch[p] = h->in[p].pitch;
            if (h->in[p].rows > 0)
                HBCU_CHECK(cudaMemcpy2DAsync(h->in_stage[s] + h->in[p].off, (size_t)h->in[p].pitch, in_planes[p], (size_t)in_strides[p],
                                             (size_t)h->in[p].row_bytes, (size_t)h->in[p].rows, cudaMemcpyHostToDevice, h->s_h2d));
        }
        HBCU_CHECK(cudaEventRecord(h->ev_up[s], h->s_h2d));
        HBCU_CHECK(cudaStreamWaitEvent(h->s_compute, h->ev_up[s], 0));
    }
    else
    {
        for (int p = 0; p < 3; p++) { src[p] = in_frame->plane[p]; spitch[p] = in_frame->stride[p]; }
        if (frame_begin_read(in_frame, h->s_compute) != 0) return -1;
    }
    if (out_frame == nullptr)
    {
        if (h->out_stage[s] == nullptr) HBCU_CHECK(cudaMalloc(&h->out_stage[s], h->out_bytes));
        for (int p = 0; p < 3; p++) { dst[p] = h->out_stage[s] + h->out[p].off; dpitch[p] = h->out[p].pitch; }
        HBCU_CHECK(cudaStreamWaitEvent(h->s_compute, h->ev_down[s], 0));     // the slot's previous copy-out is done
    }
    else
    {
        for (int p = 0; p < 3; p++) { dst[p] = out_frame->plane[p]; dpitch[p] = out_frame->stride[p]; }
        if (frame_begin_write(out_frame, h->s_compute) != 0) return -1;
    }
    h->next = (h->next + 1) % h->slots;
    h->ticket[s] = -1;
    if (launch(src, spitch, dst, dpitch) != 0) return -1;
    HBCU_CHECK(cudaEventRecord(h->ev_k[s], h->s_compute));
    if (in_frame && frame_end_read(in_frame, h->s_compute) != 0) return -1;
    if (out_frame)
    {
        if (frame_end_write(out_frame, h->s_compute) != 0) return -1;
        HBCU_CHECK(cudaEventRecord(h->ev_down[s], h->s_compute));
    }
    else
    {
        HBCU_CHECK(cudaStreamWaitEvent(h->s_d2h, h->ev_k[s], 0));
        for (int p = 0; p < 3; p++)
            if (h->out[p].rows > 0)
                HBCU_CHECK(cudaMemcpy2DAsync(out_planes[p], (size_t)out_strides[p], dst[p], (size_t)dpitch[p],
                                             (size_t)h->out[p].row_bytes, (size_t)h->out[p].rows, cudaMemcpyDeviceToHost, h->s_d2h));
        HBCU_CHECK(cudaEventRecord(h->ev_down[s], h->s_d2h));
    }
    h->ticket[s] = ticket;
    return 0;
}

inline int stage_find(const Staging *h, int64_t ticket, const char *fn)
{
    for (int s = 0; s < h->slots; s++)
        if (h->ticket[s] == ticket) return s;
    set_error("%s_%s: ticket %lld is not in flight", h->who, fn, (long long)ticket);
    return -1;
}

inline int stage_wait(Staging *h, int64_t ticket)
{
    const int s = stage_find(h, ticket, "wait");
    if (s < 0) return -1;
    HBCU_CHECK(cudaEventSynchronize(h->ev_down[s]));
    return 0;
}

inline int stage_poll(Staging *h, int64_t ticket)
{
    const int s = stage_find(h, ticket, "poll");
    if (s < 0) return -1;
    cudaError_t e = cudaEventQuery(h->ev_down[s]);
    if (e == cudaSuccess) return 1;
    if (e == cudaErrorNotReady) return 0;
    set_error("%s_poll: %s", h->who, cudaGetErrorString(e));
    return -1;
}

inline int stage_sync(Staging *h)
{
    HBCU_CHECK(cudaSetDevice(h->device));
    HBCU_CHECK(cudaStreamSynchronize(h->s_h2d));
    HBCU_CHECK(cudaStreamSynchronize(h->s_compute));
    HBCU_CHECK(cudaStreamSynchronize(h->s_d2h));
    return 0;
}

inline int stage_mark(Staging *h, int which)
{
    HBCU_CHECK(cudaSetDevice(h->device));
    HBCU_CHECK(cudaEventRecord(h->ev_mark[which], h->s_compute));
    return 0;
}

inline int stage_elapsed_ms(Staging *h, float *ms)
{
    HBCU_CHECK(cudaEventSynchronize(h->ev_mark[1]));
    HBCU_CHECK(cudaEventElapsedTime(ms, h->ev_mark[0], h->ev_mark[1]));
    return 0;
}

}  // namespace hbcu
