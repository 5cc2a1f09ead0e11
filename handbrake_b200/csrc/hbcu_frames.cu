// hbcu_frames.cu -- device-resident frames: the HBCU_DEVICE backing of hb_buffer_t (SURVEY.md 8 f3).
//
// In libhb every filter owns a thread and frames travel between filters as hb_buffer_t through FIFOs
// (work.c:2527-2600).  With a CUDA filter on both sides of a FIFO the frame does not have to visit the host: the
// producer writes its output into a pooled device frame and hands the hb_buffer_t on at once; the consumer makes
// its own stream wait for the frame's `ready` event.  Nothing blocks on the host, the order of work on the GPU is
// carried by two events per frame:
//   ready     producer -> readers   (recorded behind the last write)
//   consumed  readers  -> next life (a reader, when done, waits for the previous record and records its own in one
//                                    locked step, so the most recent record stands for all readers on all host
//                                    threads; the pool hands a frame out again at once and the next producer's
//                                    stream waits for `ready` (write after write) and `consumed` before writing)
// This mirrors how libhb already carries non-host frames (AVFRAME / COREMEDIA storage, handbrake/internal.h:152-153,
// fifo.c:1016-1034) and its VideoToolbox adapter filters (platform/macosx/adapter_vt.c).
#include "hbcu_frames.h"
#include "../../include/hbcu.h"

#include <mutex>
#include <new>
#include <vector>

namespace {

std::mutex g_frame_lock;
std::mutex g_reader_lock;       // makes a reader's wait-then-record on `consumed` one step
hbcu_frame_s *g_frame_free = nullptr;
long g_frames_alive = 0;          // frames handed out and not yet released (leak check for the tests)

// a semi-planar frame (NV12, P010, P016) has no third plane: it is given as 0 rows of 0 bytes
bool absent_plane(int p, const int row_bytes[3], const int rows[3]) { return p == 2 && rows[2] == 0 && row_bytes[2] == 0; }

bool same_geometry(const hbcu_frame_s *f, int device, const int row_bytes[3], const int rows[3], const int strides[3])
{
    if (f->device != device) return false;
    for (int p = 0; p < 3; p++)
        if (f->row_bytes[p] != row_bytes[p] || f->rows[p] != rows[p] || f->stride[p] != strides[p]) return false;
    return true;
}

}  // namespace

namespace hbcu {

int frame_begin_write(hbcu_frame_s *f, cudaStream_t st)
{
    // behind every reader of the previous life AND behind its producer: a frame that was written but never read (its
    // buffer dropped on an error path) comes back from the pool with the old producer's kernels possibly still queued
    HBCU_CHECK(cudaStreamWaitEvent(st, f->ready, 0));
    HBCU_CHECK(cudaStreamWaitEvent(st, f->consumed, 0));
    return 0;
}

int frame_end_write(hbcu_frame_s *f, cudaStream_t st)
{
    HBCU_CHECK(cudaEventRecord(f->ready, st));
    return 0;
}

int frame_begin_read(hbcu_frame_s *f, cudaStream_t st)
{
    HBCU_CHECK(cudaStreamWaitEvent(st, f->ready, 0));
    return 0;
}

int frame_end_read(hbcu_frame_s *f, cudaStream_t st)
{
    // readers chain: wait for the previous reader's record, then record -- atomically, so that two holders of a
    // shallow-dup'ed frame reading from different host threads cannot both chain behind the same older record
    // (the next writer waits for the LAST record only, which must imply all the others)
    std::lock_guard<std::mutex> g(g_reader_lock);
    HBCU_CHECK(cudaStreamWaitEvent(st, f->consumed, 0));
    HBCU_CHECK(cudaEventRecord(f->consumed, st));
    return 0;
}

}  // namespace hbcu

struct hbcu_xfer_s
{
    int device;
    cudaStream_t st;
    std::vector<cudaEvent_t> ev;       // ring of completion events, slot = ticket % size
    std::vector<int64_t> ticket;
};

extern "C" {

int hbcu_frame_alloc(hbcu_frame_t **out, int device, const int row_bytes[3], const int rows[3], const int strides[3])
{
    if (out == nullptr || row_bytes == nullptr || rows == nullptr || strides == nullptr)
    {
        hbcu::set_error("hbcu_frame_alloc: null argument");
        return -1;
    }
    *out = nullptr;
    int stride_of[3];                                   // an absent plane's stride is 0 whatever was passed (pool key)
    for (int p = 0; p < 3; p++)
    {
        stride_of[p] = absent_plane(p, row_bytes, rows) ? 0 : strides[p];
        if (absent_plane(p, row_bytes, rows)) continue;
        if (row_bytes[p] <= 0 || rows[p] <= 0 || strides[p] < row_bytes[p] || (strides[p] % 16) != 0)
        {
            hbcu::set_error("hbcu_frame_alloc: plane %d: %d bytes x %d rows, stride %d (strides must be multiples of 16)", p,
                            row_bytes[p], rows[p], strides[p]);
            return -1;
        }
    }
    strides = stride_of;
    {
        std::lock_guard<std::mutex> g(g_frame_lock);
        hbcu_frame_s **link = &g_frame_free;
        while (*link != nullptr)
        {
            if (same_geometry(*link, device, row_bytes, rows, strides))
            {
                hbcu_frame_s *f = *link;
                *link = f->next;
                f->next = nullptr;
                f->refs = 1;
                g_frames_alive++;
                *out = f;
                return 0;
            }
            link = &(*link)->next;
        }
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev)
    {
        cudaGetLastError();
        hbcu::set_error("hbcu_frame_alloc: CUDA device %d not available (%d devices)", device, ndev);
        return -1;
    }
    HBCU_CHECK(cudaSetDevice(device));
    hbcu_frame_s *f = new (std::nothrow) hbcu_frame_s();
    if (f == nullptr) { hbcu::set_error("hbcu_frame_alloc: out of memory"); return -1; }
    f->device = device;
    size_t off = 0;
    for (int p = 0; p < 3; p++)
    {
        f->row_bytes[p] = row_bytes[p];
        f->rows[p] = rows[p];
        f->stride[p] = strides[p];
        off += (size_t)strides[p] * rows[p];
    }
    f->bytes = off;
    f->base = nullptr;
    f->ready = f->consumed = nullptr;
    f->next = nullptr;
    f->refs = 1;
    f->external = false;
    f->ext_release = nullptr;
    f->ext_opaque = nullptr;
    // 256 bytes of zeroed slack behind the last plane: lapsharp and EEDI2 read a little past a plane's end
    if (cudaMalloc(&f->base, off + 256) != cudaSuccess || cudaMemset(f->base, 0, off + 256) != cudaSuccess ||
        cudaEventCreateWithFlags(&f->ready, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&f->consumed, cudaEventDisableTiming) != cudaSuccess)
    {
        hbcu::set_error("hbcu_frame_alloc: %s", cudaGetErrorString(cudaGetLastError()));
        if (f->base) cudaFree(f->base);
        if (f->ready) cudaEventDestroy(f->ready);
        if (f->consumed) cudaEventDestroy(f->consumed);
        delete f;
        return -1;
    }
    // the clearing memset runs on the legacy default stream, which the filters' non-blocking streams do not wait for:
    // the first producer of the frame orders itself behind `consumed`, so record it behind the memset
    if (cudaEventRecord(f->consumed, 0) != cudaSuccess)
    {
        hbcu::set_error("hbcu_frame_alloc: %s", cudaGetErrorString(cudaGetLastError()));
        cudaFree(f->base);
        cudaEventDestroy(f->ready);
        cudaEventDestroy(f->consumed);
        delete f;
        return -1;
    }
    off = 0;
    for (int p = 0; p < 3; p++)
    {
        f->plane[p] = absent_plane(p, row_bytes, rows) ? nullptr : f->base + off;
        off += (size_t)strides[p] * rows[p];
    }
    {
        std::lock_guard<std::mutex> g(g_frame_lock);
        g_frames_alive++;
    }
    *out = f;
    return 0;
}

void hbcu_frame_retain(hbcu_frame_t *f)
{
    if (f == nullptr) return;
    std::lock_guard<std::mutex> g(g_frame_lock);
    f->refs++;
}

void hbcu_frame_release(hbcu_frame_t *f)
{
    if (f == nullptr) return;
    {
        // no wait: whoever writes the frame next orders itself behind `consumed`
        std::lock_guard<std::mutex> g(g_frame_lock);
        if (--f->refs > 0) return;
        g_frames_alive--;
        if (!f->external)
        {
            f->next = g_frame_free;
            g_frame_free = f;
            return;
        }
    }
    // a wrapped frame goes back to its owner, who may overwrite it at once: only after every queued reader is done
    cudaSetDevice(f->device);
    cudaEventSynchronize(f->consumed);
    cudaGetLastError();
    if (f->ext_release != nullptr) f->ext_release(f->ext_opaque);
    cudaEventDestroy(f->ready);
    cudaEventDestroy(f->consumed);
    delete f;
}

// The NVDEC / NVENC seam (nvenc_common.c:329-336, hwaccel.c:15-60: hw_pix_fmt = AV_PIX_FMT_CUDA): a frame that already
// lives in device memory somebody else owns -- what an AVFrame of AV_PIX_FMT_CUDA carries (data[i] = device pointer,
// linesize[i]) -- becomes an hbcu_frame_t without a copy.
int hbcu_frame_wrap(hbcu_frame_t **out, int device, void *const dplanes[3], const int row_bytes[3], const int rows[3],
                    const int strides[3], size_t readable_tail_bytes, void *producer_stream,
                    hbcu_frame_release_fn release, void *opaque)
{
    if (out == nullptr || dplanes == nullptr || row_bytes == nullptr || rows == nullptr || strides == nullptr)
    {
        hbcu::set_error("hbcu_frame_wrap: null argument");
        return -1;
    }
    *out = nullptr;
    const bool two_planes = absent_plane(2, row_bytes, rows) && dplanes[2] == nullptr;
    for (int p = 0; p < (two_planes ? 2 : 3); p++)
    {
        if (dplanes[p] == nullptr || ((uintptr_t)dplanes[p] % 16) != 0 || row_bytes[p] <= 0 || rows[p] <= 0 ||
            strides[p] < row_bytes[p] || (strides[p] % 16) != 0)
        {
            hbcu::set_error("hbcu_frame_wrap: plane %d: %d bytes x %d rows, stride %d (pointers and strides must be multiples of 16)", p,
                            row_bytes[p], rows[p], strides[p]);
            return -1;
        }
    }
    if (readable_tail_bytes < 256)
    {
        // the pooled frames carry 256 bytes of slack behind the last plane because the stencil kernels read whole
        // vectors past a plane's end; a wrapped surface has to promise the same (decoder surfaces do: their height
        // is aligned up)
        hbcu::set_error("hbcu_frame_wrap: the allocation must stay readable for 256 bytes past every plane's last row");
        return -1;
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev)
    {
        cudaGetLastError();
        hbcu::set_error("hbcu_frame_wrap: CUDA device %d not available (%d devices)", device, ndev);
        return -1;
    }
    HBCU_CHECK(cudaSetDevice(device));
    hbcu_frame_s *f = new (std::nothrow) hbcu_frame_s();
    if (f == nullptr) { hbcu::set_error("hbcu_frame_wrap: out of memory"); return -1; }
    f->device = device;
    f->base = nullptr;
    f->bytes = 0;
    for (int p = 0; p < 3; p++)
    {
        f->plane[p] = (uint8_t *)dplanes[p];
        f->row_bytes[p] = row_bytes[p];
        f->rows[p] = rows[p];
        f->stride[p] = (two_planes && p == 2) ? 0 : strides[p];
    }
    f->ready = f->consumed = nullptr;
    f->next = nullptr;
    f->refs = 1;
    f->external = true;
    f->ext_release = release;
    f->ext_opaque = opaque;
    if (cudaEventCreateWithFlags(&f->ready, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&f->consumed, cudaEventDisableTiming) != cudaSuccess ||
        // the producer (the decoder's stream; NULL = the legacy default stream, i.e. work already synchronised) wrote the
        // planes: readers order themselves behind this record exactly as behind a filter's
        cudaEventRecord(f->ready, (cudaStream_t)producer_stream) != cudaSuccess)
    {
        hbcu::set_error("hbcu_frame_wrap: %s", cudaGetErrorString(cudaGetLastError()));
        if (f->ready) cudaEventDestroy(f->ready);
        if (f->consumed) cudaEventDestroy(f->consumed);
        delete f;
        return -1;
    }
    {
        std::lock_guard<std::mutex> g(g_frame_lock);
        g_frames_alive++;
    }
    *out = f;
    return 0;
}

// an external consumer (the encoder's stream) reads a device frame: acquire orders `cuda_stream` behind the frame's
// producer, done marks the reads queued so far on that stream as the frame's latest reader
int hbcu_frame_acquire(hbcu_frame_t *f, void *cuda_stream)
{
    if (f == nullptr) { hbcu::set_error("hbcu_frame_acquire: null frame"); return -1; }
    return hbcu::frame_begin_read(f, (cudaStream_t)cuda_stream);
}

int hbcu_frame_done(hbcu_frame_t *f, void *cuda_stream)
{
    if (f == nullptr) { hbcu::set_error("hbcu_frame_done: null frame"); return -1; }
    return hbcu::frame_end_read(f, (cudaStream_t)cuda_stream);
}

void *hbcu_frame_plane(const hbcu_frame_t *f, int plane) { return f && plane >= 0 && plane < 3 ? f->plane[plane] : nullptr; }
int hbcu_frame_stride(const hbcu_frame_t *f, int plane) { return f && plane >= 0 && plane < 3 ? f->stride[plane] : 0; }
int hbcu_frame_device(const hbcu_frame_t *f) { return f ? f->device : -1; }
long hbcu_frames_alive(void) { std::lock_guard<std::mutex> g(g_frame_lock); return g_frames_alive; }

void hbcu_frame_trim(void)
{
    std::lock_guard<std::mutex> g(g_frame_lock);
    while (g_frame_free != nullptr)
    {
        hbcu_frame_s *f = g_frame_free;
        g_frame_free = f->next;
        cudaSetDevice(f->device);
        cudaEventSynchronize(f->consumed);
        cudaFree(f->base);
        cudaEventDestroy(f->ready);
        cudaEventDestroy(f->consumed);
        delete f;
    }
}

// ---------------------------------------------------------------------------
// hbcu_xfer: the two ends of a device-resident chain -- host frame -> device frame in front of the first CUDA
// filter when the decoder delivers host memory, device frame -> host frame in front of the encoder (the role of
// libhb's adapter filters, platform/macosx/adapter_vt.c).  Asynchronous, tickets complete in order.
// ---------------------------------------------------------------------------
int hbcu_xfer_create(hbcu_xfer_t **out, int device, int depth)
{
    if (out == nullptr) { hbcu::set_error("hbcu_xfer_create: null argument"); return -1; }
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev)
    {
        cudaGetLastError();
        hbcu::set_error("hbcu_xfer_create: CUDA device %d not available (%d devices); there is no CPU fallback", device, ndev);
        return -1;
    }
    HBCU_CHECK(cudaSetDevice(device));
    hbcu_xfer_s *x = new (std::nothrow) hbcu_xfer_s();
    if (x == nullptr) { hbcu::set_error("hbcu_xfer_create: out of memory"); return -1; }
    x->device = device;
    x->st = nullptr;
    if (depth < 2) depth = 8;
    x->ev.assign(depth, nullptr);
    x->ticket.assign(depth, -1);
    if (cudaStreamCreateWithFlags(&x->st, cudaStreamNonBlocking) != cudaSuccess)
    {
        hbcu::set_error("hbcu_xfer_create: %s", cudaGetErrorString(cudaGetLastError()));
        delete x;
        return -1;
    }
    for (auto &e : x->ev)
    {
        if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess)
        {
            hbcu::set_error("hbcu_xfer_create: %s", cudaGetErrorString(cudaGetLastError()));
            hbcu_xfer_destroy(x);
            return -1;
        }
    }
    *out = x;
    return 0;
}

void hbcu_xfer_destroy(hbcu_xfer_t *x)
{
    if (x == nullptr) return;
    cudaSetDevice(x->device);
    if (x->st) { cudaStreamSynchronize(x->st); cudaStreamDestroy(x->st); }
    for (auto e : x->ev) if (e) cudaEventDestroy(e);
    delete x;
}

static bool host_matches_frame(const hbcu_frame_t *f, const void *const planes[3], const int strides[3])
{
    size_t off = 0;
    for (int p = 0; p < 3; p++)
    {
        if (f->plane[p] == nullptr) continue;                // the absent third plane of a semi-planar frame
        if (strides[p] != f->stride[p] || (const uint8_t *)planes[p] != (const uint8_t *)planes[0] + off) return false;
        off += (size_t)f->stride[p] * f->rows[p];
    }
    return true;
}

static int xfer_copy(hbcu_xfer_t *x, int64_t ticket, hbcu_frame_t *f, void *const planes[3], const int strides[3], bool download)
{
    if (x == nullptr || f == nullptr || planes == nullptr || strides == nullptr || ticket < 0)
    {
        hbcu::set_error("hbcu_xfer: bad argument");
        return -1;
    }
    if (f->device != x->device) { hbcu::set_error("hbcu_xfer: frame lives on device %d, not %d", f->device, x->device); return -1; }
    HBCU_CHECK(cudaSetDevice(x->device));
    const int slot = (int)(ticket % (int64_t)x->ev.size());
    if (download) { if (hbcu::frame_begin_read(f, x->st) != 0) return -1; }
    else          { if (hbcu::frame_begin_write(f, x->st) != 0) return -1; }
    const cudaMemcpyKind kind = download ? cudaMemcpyDeviceToHost : cudaMemcpyHostToDevice;
    if (host_matches_frame(f, planes, strides))
    {
        if (download) HBCU_CHECK(cudaMemcpyAsync(planes[0], f->base, f->bytes, kind, x->st));
        else          HBCU_CHECK(cudaMemcpyAsync(f->base, planes[0], f->bytes, kind, x->st));
    }
    else
    {
        for (int p = 0; p < 3; p++)
        {
            if (f->plane[p] == nullptr) continue;
            if (download)
                HBCU_CHECK(cudaMemcpy2DAsync(planes[p], (size_t)strides[p], f->plane[p], (size_t)f->stride[p], (size_t)f->row_bytes[p],
                                             (size_t)f->rows[p], kind, x->st));
            else
                HBCU_CHECK(cudaMemcpy2DAsync(f->plane[p], (size_t)f->stride[p], planes[p], (size_t)strides[p], (size_t)f->row_bytes[p],
                                             (size_t)f->rows[p], kind, x->st));
        }
    }
    if (download) { if (hbcu::frame_end_read(f, x->st) != 0) return -1; }
    else          { if (hbcu::frame_end_write(f, x->st) != 0) return -1; }
    HBCU_CHECK(cudaEventRecord(x->ev[slot], x->st));
    x->ticket[slot] = ticket;
    return 0;
}

int hbcu_xfer_download(hbcu_xfer_t *x, int64_t ticket, hbcu_frame_t *f, void *const planes[3], const int strides[3])
{
    return xfer_copy(x, ticket, f, planes, strides, true);
}

int hbcu_xfer_upload(hbcu_xfer_t *x, int64_t ticket, hbcu_frame_t *f, const void *const planes[3], const int strides[3])
{
    return xfer_copy(x, ticket, f, const_cast<void *const *>(planes), strides, false);
}

int hbcu_xfer_wait(hbcu_xfer_t *x, int64_t ticket)
{
    if (x == nullptr || ticket < 0) { hbcu::set_error("hbcu_xfer_wait: bad argument"); return -1; }
    const int slot = (int)(ticket % (int64_t)x->ev.size());
    if (x->ticket[slot] != ticket) { hbcu::set_error("hbcu_xfer_wait: ticket %lld is not in flight", (long long)ticket); return -1; }
    HBCU_CHECK(cudaEventSynchronize(x->ev[slot]));
    return 0;
}

int hbcu_xfer_poll(hbcu_xfer_t *x, int64_t ticket)
{
    if (x == nullptr || ticket < 0) { hbcu::set_error("hbcu_xfer_poll: bad argument"); return -1; }
    const int slot = (int)(ticket % (int64_t)x->ev.size());
    if (x->ticket[slot] != ticket) { hbcu::set_error("hbcu_xfer_poll: ticket %lld is not in flight", (long long)ticket); return -1; }
    cudaError_t e = cudaEventQuery(x->ev[slot]);
    if (e == cudaSuccess) return 1;
    if (e == cudaErrorNotReady) return 0;
    hbcu::set_error("hbcu_xfer_poll: %s", cudaGetErrorString(e));
    return -1;
}

}  // extern "C"
