// motion_metric.cu -- vfr's frame-to-frame motion metric for sm_90a behind the C-ABI of include/hbcu.h.
//
// Replaces (reference: HandBrake's libhb/motion_metric.c, the x86 variant): build_gamma_lut's table is built by the host
// and uploaded; approximate_frame_data_{8,16}, sse_block16_{8,16}, motion_metric_{8,16} and motion_metric_fast_{8,16}
// are one kernel.  Bit-exact with the reference's uint64 sum:
//   - only whole 16x16 blocks count (bw = width / 16, bh = height / 16); remainder rows and columns are ignored;
//   - per block, int diff = lut[a] - lut[b] and the squares add into a uint32 that wraps (a full-scale 8-bit block
//     reaches 256 * 4130^2 > 2^32), then the block sums add into a uint64.  Block sums are exact integers, so the order
//     the kernel adds them in does not matter;
//   - fast path: each image is first reduced to width/4 x height/4, every output sample the nested rounding average
//     APPROX(APPROX(..), ..) of a 4x4 cell in the reference's argument order, in integers at the sample width.  The
//     reduced images are packed (row pitch width/4), and above 8 bits the reference walks them with half that pitch
//     (motion_metric_fast_16 passes a pitch in samples that motion_metric_16 divides by the sample size again): block
//     sample (x, y) is packed sample y * (width/4/2) + x.  The kernel reads and compares exactly those samples.
// The host divides: (float)sum / (w * h), as the reference.
//
// Each new frame B is read once.  On the fast path the kernel reduces B, stores the reduced image of its whole blocks in
// B's slot and compares it with the slot of frame A; below 1080p it compares B's luma with A's luma in A's slot (a
// reference on A's device frame, or the device copy of A's host luma).  One CTA works through 16x16 blocks, one sample
// per thread; the gamma table sits in shared memory up to 12 bits and is read through the read-only path above.
#include "hbcu_common.h"
#include "hbcu_frames.h"
#include "../../include/hbcu.h"

#include <algorithm>
#include <new>
#include <vector>

namespace {

using hbcu::set_error;

std::atomic<uint64_t> g_waits{0};
std::atomic<uint64_t> g_launches{0};

constexpr int kThreads = 256;          // one 16x16 block, one sample per thread
constexpr int kSmemLutMaxDepth = 12;   // 4096 entries, 16 KB

struct MetricArgs
{
    const uint8_t *b;                  // frame B: full-resolution luma
    int b_pitch;
    const uint8_t *a;                  // frame A: its slot (reduced image on the fast path, else its luma); null: none
    int a_pitch;
    uint8_t *out;                      // fast path: B's slot, receives B's packed reduced image; else null
    int red_w;                         // fast path: width of the reduced image (its packed pitch, in samples)
    int sse_pitch;                     // fast path: the pitch, in samples, the block sums walk the packed images with
    const unsigned *lut;
    unsigned maxv;
    int bw, bh;                        // whole 16x16 blocks of the compared images
    unsigned long long *result;
};

__device__ __forceinline__ unsigned approx(unsigned a, unsigned b, unsigned c, unsigned d)
{
    return (((a + b + 1) >> 1) + ((c + d + 1) >> 1) + 1) >> 1;
}

template <typename T>
__device__ __forceinline__ unsigned px(const uint8_t *base, int pitch, int x, int y)
{
    return reinterpret_cast<const T *>(base + (size_t)y * pitch)[x];
}

// FAST: B is reduced 4x4 first.  SMEM_LUT: the gamma table is staged in shared memory.
template <typename T, bool FAST, bool SMEM_LUT>
__global__ void __launch_bounds__(kThreads) motion_metric_kernel(const MetricArgs a)
{
    extern __shared__ unsigned s_lut[];
    __shared__ unsigned s_part[2][kThreads / 32];
    const unsigned *lut = a.lut;
    if (SMEM_LUT)
    {
        for (unsigned i = threadIdx.x; i <= a.maxv; i += kThreads) s_lut[i] = a.lut[i];
        __syncthreads();
        lut = s_lut;
    }
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4, warp = threadIdx.x >> 5;
    const int nblocks = a.bw * a.bh;
    unsigned long long total = 0;
    int it = 0;
    for (int blk = blockIdx.x; blk < nblocks; blk += gridDim.x, it ^= 1)
    {
        const int x = (blk % a.bw) * 16 + tx, y = (blk / a.bw) * 16 + ty;
        unsigned vb, va;
        if (FAST)
        {
            // the packed sample the block sum reads, and the reduced-image position it holds
            const int l = y * a.sse_pitch + x, xr = l % a.red_w, yr = l / a.red_w;
            // approximate_frame_data: cell rows 4yr..4yr+3, columns 4xr..4xr+3; APPROX(a, b, c, d) pairs (a, b), (c, d)
            const int c0 = 4 * xr, r0 = 4 * yr;
            unsigned s[4][4];
#pragma unroll
            for (int r = 0; r < 4; r++)
#pragma unroll
                for (int c = 0; c < 4; c++) s[r][c] = px<T>(a.b, a.b_pitch, c0 + c, r0 + r);
            const unsigned tl = approx(s[0][0], s[1][0], s[0][1], s[1][1]);
            const unsigned tr = approx(s[0][2], s[1][2], s[0][3], s[1][3]);
            const unsigned bl = approx(s[2][0], s[3][0], s[2][1], s[3][1]);
            const unsigned br = approx(s[2][2], s[3][2], s[2][3], s[3][3]);
            vb = approx(tl, tr, bl, br);
            reinterpret_cast<T *>(a.out)[l] = (T)vb;      // threads sharing l (half pitch) store the same value
            if (a.a == nullptr) continue;
            va = reinterpret_cast<const T *>(a.a)[l];
        }
        else
        {
            if (a.a == nullptr) continue;
            vb = px<T>(a.b, a.b_pitch, x, y);
            va = px<T>(a.a, a.a_pitch, x, y);
        }
        // sse_block16: int diff, diff * diff added into an unsigned (values beyond the depth's range are clamped to the
        // table instead of reading past it)
        const unsigned ia = min(va, a.maxv), ib = min(vb, a.maxv);
        const int diff = SMEM_LUT ? (int)lut[ia] - (int)lut[ib] : (int)__ldg(&lut[ia]) - (int)__ldg(&lut[ib]);
        const unsigned sq = __reduce_add_sync(0xffffffffu, (unsigned)(diff * diff));   // wraps mod 2^32, as the block sum
        if ((threadIdx.x & 31) == 0) s_part[it][warp] = sq;
        __syncthreads();
        if (threadIdx.x == 0)
        {
            unsigned block = 0;
#pragma unroll
            for (int w = 0; w < kThreads / 32; w++) block += s_part[it][w];
            total += block;
        }
    }
    if (a.a != nullptr && threadIdx.x == 0 && total != 0) atomicAdd(a.result, total);
}

struct Slot
{
    uint8_t *buf = nullptr;            // packed reduced image (fast) or a device copy of host luma
    size_t cap = 0;
    int buf_pitch = 0;
    hbcu_frame_t *frame = nullptr;     // below 1080p: the device frame the slot reads in place (one reference)
    const uint8_t *ptr = nullptr;      // what the kernel reads as A
    int pitch = 0;
    bool filled = false;
};

}  // namespace

struct hbcu_motion_metric_s
{
    hbcu_motion_metric_config_t cfg;
    int bps = 1, bw = 0, bh = 0, ctas = 1;
    unsigned maxv = 255;
    bool smem_lut = false;
    cudaStream_t st = nullptr;
    unsigned *lut = nullptr;
    unsigned long long *d_res = nullptr, *h_res = nullptr;
    std::vector<cudaEvent_t> res_ev;
    std::vector<Slot> slots;
    uint8_t *stage = nullptr;          // fast path, host luma: the full-resolution copy the kernel reduces
    int stage_pitch = 0;
    cudaEvent_t ev_copy = nullptr, ev_mark[2] = {nullptr, nullptr};
};

namespace {

void drop_frame(Slot &s)
{
    if (s.frame) hbcu_frame_release(s.frame);
    s.frame = nullptr;
}

int ensure_buf(Slot &s, int pitch, int rows)
{
    const size_t bytes = (size_t)pitch * rows;
    if (bytes > s.cap)
    {
        if (s.buf) HBCU_CHECK(cudaFree(s.buf));
        s.buf = nullptr;
        s.cap = 0;
        HBCU_CHECK(cudaMalloc(&s.buf, bytes));
        s.cap = bytes;
    }
    s.buf_pitch = pitch;
    return 0;
}

int launch(hbcu_motion_metric_s *h, const uint8_t *b, int b_pitch, const Slot *a, Slot *out, int result)
{
    MetricArgs m;
    m.b = b; m.b_pitch = b_pitch;
    m.a = a ? a->ptr : nullptr; m.a_pitch = a ? a->pitch : 0;
    m.out = out ? out->buf : nullptr;
    m.red_w = h->cfg.width / 4;
    m.sse_pitch = h->bps == 1 ? m.red_w : m.red_w / 2;
    m.lut = h->lut; m.maxv = h->maxv;
    m.bw = h->bw; m.bh = h->bh;
    m.result = a ? h->d_res + result : nullptr;
    const size_t smem = h->smem_lut ? sizeof(unsigned) * (h->maxv + 1) : 0;
    const bool fast = h->cfg.fast != 0;
#define MM_LAUNCH(T, F, S) motion_metric_kernel<T, F, S><<<h->ctas, kThreads, smem, h->st>>>(m)
    if (h->bps == 1)
    {
        if (fast) { if (h->smem_lut) MM_LAUNCH(uint8_t, true, true); else MM_LAUNCH(uint8_t, true, false); }
        else      { if (h->smem_lut) MM_LAUNCH(uint8_t, false, true); else MM_LAUNCH(uint8_t, false, false); }
    }
    else
    {
        if (fast) { if (h->smem_lut) MM_LAUNCH(uint16_t, true, true); else MM_LAUNCH(uint16_t, true, false); }
        else      { if (h->smem_lut) MM_LAUNCH(uint16_t, false, true); else MM_LAUNCH(uint16_t, false, false); }
    }
#undef MM_LAUNCH
    HBCU_CHECK(cudaGetLastError());
    hbcu::count_launch();
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return 0;
}

}  // namespace

extern "C" {

uint64_t hbcu_motion_metric_waits(void) { return g_waits.load(std::memory_order_relaxed); }
uint64_t hbcu_motion_metric_launches(void) { return g_launches.load(std::memory_order_relaxed); }

int hbcu_motion_metric_create(hbcu_motion_metric_t **out, const hbcu_motion_metric_config_t *cfg)
{
    if (out == nullptr || cfg == nullptr || cfg->gamma_lut == nullptr) { set_error("motion_metric_create: null argument"); return -1; }
    *out = nullptr;
    if (cfg->width < 1 || cfg->height < 1 || cfg->depth < 8 || cfg->depth > 16 || cfg->slots < 2 || cfg->results < 1)
    {
        set_error("motion_metric_create: unsupported geometry %dx%d depth %d, %d slots, %d results", cfg->width, cfg->height,
                  cfg->depth, cfg->slots, cfg->results);
        return -1;
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || cfg->device < 0 || cfg->device >= ndev)
    {
        cudaGetLastError();
        set_error("motion_metric_create: CUDA device %d not available (%d devices); there is no CPU fallback", cfg->device, ndev);
        return -1;
    }
    HBCU_CHECK(cudaSetDevice(cfg->device));
    cudaDeviceProp prop;
    HBCU_CHECK(cudaGetDeviceProperties(&prop, cfg->device));
    if (prop.major != 9 || prop.minor != 0)
    {
        set_error("motion_metric_create: device %d is sm_%d%d; this library is built for sm_90a only", cfg->device, prop.major, prop.minor);
        return -1;
    }
    hbcu_motion_metric_s *h = new (std::nothrow) hbcu_motion_metric_s();
    if (h == nullptr) { set_error("motion_metric_create: out of memory"); return -1; }
    h->cfg = *cfg;
    h->cfg.gamma_lut = nullptr;
    h->bps = cfg->depth > 8 ? 2 : 1;
    h->maxv = (1u << cfg->depth) - 1;
    const int w = cfg->fast ? cfg->width / 4 : cfg->width, hh = cfg->fast ? cfg->height / 4 : cfg->height;
    h->bw = w / 16;
    h->bh = hh / 16;
    h->smem_lut = cfg->depth <= kSmemLutMaxDepth;
    h->ctas = std::max(1, std::min(h->bw * h->bh, prop.multiProcessorCount * 4));
    h->slots.resize(cfg->slots);
    h->res_ev.assign(cfg->results, nullptr);
#define CK(expr)                                                                  \
    do {                                                                          \
        cudaError_t _e = (expr);                                                  \
        if (_e != cudaSuccess) {                                                  \
            set_error("%s failed: %s", #expr, cudaGetErrorString(_e));            \
            hbcu_motion_metric_destroy(h);                                        \
            return -1;                                                            \
        }                                                                         \
    } while (0)
    CK(cudaStreamCreateWithFlags(&h->st, cudaStreamNonBlocking));
    CK(cudaEventCreateWithFlags(&h->ev_copy, cudaEventDisableTiming));
    CK(cudaEventCreate(&h->ev_mark[0]));
    CK(cudaEventCreate(&h->ev_mark[1]));
    for (auto &e : h->res_ev) CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    CK(cudaMalloc(&h->lut, sizeof(unsigned) * (h->maxv + 1)));
    CK(cudaMemcpy(h->lut, cfg->gamma_lut, sizeof(unsigned) * (h->maxv + 1), cudaMemcpyHostToDevice));
    CK(cudaMalloc(&h->d_res, sizeof(unsigned long long) * cfg->results));
    CK(cudaMallocHost(&h->h_res, sizeof(unsigned long long) * cfg->results));
    if (h->smem_lut && sizeof(unsigned) * (h->maxv + 1) > 48 * 1024)
    {
        set_error("motion_metric_create: gamma table too large for shared memory");
        hbcu_motion_metric_destroy(h);
        return -1;
    }
#undef CK
    *out = h;
    return 0;
}

void hbcu_motion_metric_destroy(hbcu_motion_metric_t *h)
{
    if (h == nullptr) return;
    cudaSetDevice(h->cfg.device);
    if (h->st) cudaStreamSynchronize(h->st);
    for (Slot &s : h->slots)
    {
        drop_frame(s);
        if (s.buf) cudaFree(s.buf);
    }
    for (cudaEvent_t e : h->res_ev)
        if (e) cudaEventDestroy(e);
    if (h->stage) cudaFree(h->stage);
    if (h->lut) cudaFree(h->lut);
    if (h->d_res) cudaFree(h->d_res);
    if (h->h_res) cudaFreeHost(h->h_res);
    if (h->ev_copy) cudaEventDestroy(h->ev_copy);
    if (h->ev_mark[0]) cudaEventDestroy(h->ev_mark[0]);
    if (h->ev_mark[1]) cudaEventDestroy(h->ev_mark[1]);
    if (h->st) cudaStreamDestroy(h->st);
    delete h;
}

int hbcu_motion_metric_enqueue(hbcu_motion_metric_t *h, int slot, int a_slot, int result,
                               hbcu_frame_t *frame, const void *luma, int stride)
{
    if (h == nullptr || slot < 0 || slot >= (int)h->slots.size() || a_slot >= (int)h->slots.size() || a_slot == slot ||
        (a_slot >= 0 && (result < 0 || result >= (int)h->res_ev.size())) || (frame == nullptr && luma == nullptr))
    {
        set_error("motion_metric_enqueue: bad argument");
        return -1;
    }
    const int W = h->cfg.width, H = h->cfg.height, row_bytes = W * h->bps;
    if (frame != nullptr && (frame->device != h->cfg.device || frame->row_bytes[0] != row_bytes || frame->rows[0] != H))
    {
        set_error("motion_metric_enqueue: frame geometry differs from the handle's %dx%d", W, H);
        return -1;
    }
    if (frame == nullptr && stride < row_bytes)
    {
        set_error("motion_metric_enqueue: luma stride %d below the row size %d", stride, row_bytes);
        return -1;
    }
    if (a_slot >= 0 && !h->slots[a_slot].filled)
    {
        set_error("motion_metric_enqueue: slot %d holds no frame", a_slot);
        return -1;
    }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    const bool fast = h->cfg.fast != 0;
    Slot &sb = h->slots[slot];
    drop_frame(sb);
    sb.ptr = nullptr;
    sb.filled = false;

    // B's luma on the device
    const uint8_t *b = nullptr;
    int b_pitch = 0;
    if (frame != nullptr)
    {
        if (hbcu::frame_begin_read(frame, h->st) != 0) return -1;
        b = frame->plane[0];
        b_pitch = frame->stride[0];
    }
    else
    {
        const int pitch = (row_bytes + 255) / 256 * 256;
        uint8_t *dst;
        if (fast)
        {
            if (h->stage == nullptr) HBCU_CHECK(cudaMalloc(&h->stage, (size_t)pitch * H));
            h->stage_pitch = pitch;
            dst = h->stage;
        }
        else
        {
            if (ensure_buf(sb, pitch, H) != 0) return -1;
            dst = sb.buf;
        }
        HBCU_CHECK(cudaMemcpy2DAsync(dst, pitch, luma, stride, row_bytes, H, cudaMemcpyHostToDevice, h->st));
        HBCU_CHECK(cudaEventRecord(h->ev_copy, h->st));
        HBCU_CHECK(cudaEventSynchronize(h->ev_copy));     // the caller may free the luma once this returns
        b = dst;
        b_pitch = pitch;
    }

    const Slot *a = a_slot >= 0 ? &h->slots[a_slot] : nullptr;
    if (a != nullptr) HBCU_CHECK(cudaMemsetAsync(h->d_res + result, 0, sizeof(unsigned long long), h->st));
    const bool blocks = h->bw > 0 && h->bh > 0;
    if (fast)
    {
        if (blocks)
        {
            if (ensure_buf(sb, h->cfg.width / 4 * h->bps, h->cfg.height / 4) != 0) return -1;
            if (launch(h, b, b_pitch, a, &sb, result) != 0) return -1;
        }
        sb.ptr = sb.buf;                                  // null without whole blocks: then nothing is ever read
        sb.pitch = sb.buf_pitch;
    }
    else
    {
        if (a != nullptr && blocks && launch(h, b, b_pitch, a, nullptr, result) != 0) return -1;
        if (a != nullptr && a->frame != nullptr && hbcu::frame_end_read(a->frame, h->st) != 0) return -1;
        if (frame != nullptr)
        {
            hbcu_frame_retain(frame);                     // the slot reads the frame in place when the next one comes
            sb.frame = frame;
        }
        sb.ptr = b;
        sb.pitch = b_pitch;
    }
    sb.filled = true;
    if (frame != nullptr && hbcu::frame_end_read(frame, h->st) != 0) return -1;
    if (a != nullptr)
    {
        HBCU_CHECK(cudaMemcpyAsync(h->h_res + result, h->d_res + result, sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->st));
        HBCU_CHECK(cudaEventRecord(h->res_ev[result], h->st));
    }
    return 0;
}

int hbcu_motion_metric_result(hbcu_motion_metric_t *h, int result, uint64_t *sum)
{
    if (h == nullptr || sum == nullptr || result < 0 || result >= (int)h->res_ev.size())
    {
        set_error("motion_metric_result: bad argument");
        return -1;
    }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    const cudaError_t q = cudaEventQuery(h->res_ev[result]);
    if (q == cudaErrorNotReady)
    {
        g_waits.fetch_add(1, std::memory_order_relaxed);
        HBCU_CHECK(cudaEventSynchronize(h->res_ev[result]));
    }
    else HBCU_CHECK(q);
    *sum = h->h_res[result];
    return 0;
}

int hbcu_motion_metric_sync(hbcu_motion_metric_t *h)
{
    if (h == nullptr) { set_error("motion_metric_sync: null handle"); return -1; }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    HBCU_CHECK(cudaStreamSynchronize(h->st));
    return 0;
}

int hbcu_motion_metric_mark(hbcu_motion_metric_t *h, int which)
{
    if (h == nullptr || which < 0 || which > 1) { set_error("motion_metric_mark: bad argument"); return -1; }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    HBCU_CHECK(cudaEventRecord(h->ev_mark[which], h->st));
    return 0;
}

int hbcu_motion_metric_elapsed_ms(hbcu_motion_metric_t *h, float *ms)
{
    if (h == nullptr || ms == nullptr) { set_error("motion_metric_elapsed_ms: bad argument"); return -1; }
    HBCU_CHECK(cudaEventSynchronize(h->ev_mark[1]));
    HBCU_CHECK(cudaEventElapsedTime(ms, h->ev_mark[0], h->ev_mark[1]));
    return 0;
}

}  // extern "C"
