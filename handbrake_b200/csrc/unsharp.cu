// unsharp.cu -- unsharp mask and chroma smoothing for sm_90a behind the C-ABI of include/hbcu.h.
//
// Replaces (reference: HandBrake's libhb): DEF_UNSHARP_FUNC (unsharp.c:88-168) and DEF_CHROMA_SMOOTH_FUNC
// (chroma_smooth.c:86-168) -- with lapsharp the three clients of hb_filter_mt_frame (common.c:5497-5517); the frame
// batching of mt_frame_filter.c:169-237 becomes frames in flight on streams, as in lapsharp.cu.
//
// The reference blurs with a cascade of running sums: per axis `steps` pairs of [1 1] accumulators (SR[] along x,
// one SC[] row per stage along y).  That cascade IS the convolution with the binomial row of order 2*steps in each
// direction (weights C(2s,i)*C(2s,j), total 2^(4*steps) = 1 << scalebits) over a size x size window with the edge
// pixel replicated, evaluated in uint32 arithmetic that wraps (255 * 2^28 overflows for size 15).  The cascade is
// serial along x and y; the convolution is not: a CTA stages a tile plus halo in shared memory, one pass of
// horizontal binomial sums (uint32, wrapping like the reference), one vertical pass, then
//   unsharp        res = src + (((src - blur) * amount) >> 16)   clamped to [0, (int16_t)max]
//   chroma_smooth  res = src - (((src - blur) * amount) >> 16)   clamped to [(int16_t)(max/16), (int16_t)(max - max/16)]
// (the bounds are int16_t in the reference and wrap at depth 16; reproduced).  Bit-exact, integer only.
// HBM bound: 2F per frame.
#include "hbcu_common.h"
#include "hbcu_frames.h"
#include "../../include/hbcu.h"

#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>

namespace {

using hbcu::set_error;

constexpr int kTW = 128, kTH = 32, kThreads = 256;
constexpr int kMaxSteps = 7;

struct UnsharpParams
{
    const void *src;
    void *dst;
    int spitch, dpitch;       // elements
    int w, h;
    int amount, smooth;
    int minv, maxv;
    uint32_t coef[2 * kMaxSteps + 1];
};

template <typename PIX, int S>
__global__ void __launch_bounds__(kThreads) unsharp_kernel(const UnsharpParams p)
{
    constexpr int N = 2 * S + 1;
    constexpr int EPW = 4 / (int)sizeof(PIX);                     // samples per 32-bit word
    // source tile: columns X0 - S - lead .. X0 + kTW + S, where lead = (X0 - S) mod EPW aligns the tile's first column to
    // a word of the (word-aligned) source row; the pitch keeps every tile row word aligned too
    constexpr int SW = (kTW + 2 * S + (EPW - 1) + EPW - 1) / EPW * EPW + EPW;
    constexpr int SR = kTH + 2 * S;               // source tile rows
    __shared__ __align__(16) PIX      s_src[SR * SW];
    __shared__ __align__(16) uint32_t s_h[SR * kTW];
    const PIX *src = (const PIX *)p.src;
    PIX *dst = (PIX *)p.dst;
    const int X0 = blockIdx.x * kTW, Y0 = blockIdx.y * kTH;
    const int tid = threadIdx.x;
    const int xs = X0 - S;                                        // first staged column (may be negative at the left edge)
    const int lead = ((xs % EPW) + EPW) % EPW;                    // staged column c sits at s_src[r * SW + lead + c]
    const bool interior = xs - lead >= 0 && X0 + kTW + S <= p.w && Y0 - S >= 0 && Y0 + kTH + S <= p.h &&
                          ((uintptr_t)src % 4 == 0) && (((size_t)p.spitch * sizeof(PIX)) % 4 == 0);
    if (interior)
    {
        // no clamping anywhere in this tile: aligned 32-bit words straight from the row (read-only path) into the tile
        constexpr int WPR = (kTW + 2 * S + 2 * (EPW - 1) + EPW - 1) / EPW;       // words per tile row (covers any lead)
        const int x_word0 = xs - lead;
        for (int i = tid; i < SR * WPR; i += kThreads)
        {
            const int r = i / WPR, wq = i - r * WPR;
            const int x = x_word0 + wq * EPW;
            if (x < p.spitch)
            {
                const uint32_t v = __ldg(reinterpret_cast<const uint32_t *>(src + (size_t)(Y0 + r - S) * p.spitch + x));
                *reinterpret_cast<uint32_t *>(&s_src[r * SW + wq * EPW]) = v;
            }
        }
    }
    else
    {
        // stage the tile with the edge pixel replicated (x <= 0 -> src[0], x >= w -> src[w-1]; rows likewise)
        for (int i = tid; i < SR * (kTW + 2 * S); i += kThreads)
        {
            const int r = i / (kTW + 2 * S), c = i - r * (kTW + 2 * S);
            const int y = min(max(Y0 + r - S, 0), p.h - 1), x = min(max(X0 + c - S, 0), p.w - 1);
            s_src[r * SW + lead + c] = src[(size_t)y * p.spitch + x];
        }
    }
    __syncthreads();
    // horizontal binomial sums, 4 outputs per item share their 4 + 2S inputs
    for (int i = tid; i < SR * (kTW / 4); i += kThreads)
    {
        const int r = i / (kTW / 4), x4 = (i - r * (kTW / 4)) * 4;
        uint32_t v[4 + 2 * S];
#pragma unroll
        for (int k = 0; k < 4 + 2 * S; k++) v[k] = s_src[r * SW + lead + x4 + k];
        uint32_t a[4] = { 0, 0, 0, 0 };
#pragma unroll
        for (int k = 0; k < N; k++)
        {
            const uint32_t c = p.coef[k];
#pragma unroll
            for (int j = 0; j < 4; j++) a[j] += c * v[j + k];
        }
        *reinterpret_cast<uint4 *>(&s_h[r * kTW + x4]) = make_uint4(a[0], a[1], a[2], a[3]);
    }
    __syncthreads();
    // vertical sums + the sharpening / smoothing expression: one item = 4 rows x 4 columns (the 4 + 2S rows of horizontal
    // sums arrive as 128-bit words, the results leave as one vector store per row); 8 x 32 items = one per thread
    constexpr int scalebits = 4 * S;
    constexpr uint32_t halfscale = 1u << (scalebits - 1);
    for (int i = tid; i < (kTH / 4) * (kTW / 4); i += kThreads)
    {
        const int y4 = (i / (kTW / 4)) * 4, x4 = (i - (i / (kTW / 4)) * (kTW / 4)) * 4;
        if (X0 + x4 >= p.w || Y0 + y4 >= p.h) continue;
        uint32_t a[4][4];
#pragma unroll
        for (int j = 0; j < 4; j++)
#pragma unroll
            for (int q = 0; q < 4; q++) a[j][q] = 0;
#pragma unroll
        for (int k = 0; k < 4 + 2 * S; k++)
        {
            const uint4 hv = *reinterpret_cast<const uint4 *>(&s_h[(y4 + k) * kTW + x4]);
            const uint32_t h4[4] = { hv.x, hv.y, hv.z, hv.w };
#pragma unroll
            for (int j = 0; j < 4; j++)
            {
                // row k of the window feeds output row j with coefficient index k - j
                if (k - j < 0 || k - j >= N) continue;
                const uint32_t c = p.coef[k - j];
#pragma unroll
                for (int q = 0; q < 4; q++) a[j][q] += c * h4[q];
            }
        }
#pragma unroll
        for (int j = 0; j < 4; j++)
        {
            const int y = Y0 + y4 + j;
            if (y >= p.h) break;
            int out[4];
#pragma unroll
            for (int q = 0; q < 4; q++)
            {
                const int32_t sv = (int32_t)s_src[(y4 + j + S) * SW + lead + x4 + q + S];
                const int32_t blur = (int32_t)((a[j][q] + halfscale) >> scalebits);
                const int32_t delta = (int32_t)((uint32_t)(sv - blur) * (uint32_t)p.amount) >> 16;   // 32-bit product, arithmetic shift
                const int32_t res = p.smooth ? sv - delta : sv + delta;
                out[q] = res > p.maxv ? p.maxv : res < p.minv ? p.minv : res;
            }
            PIX *drow = dst + (size_t)y * p.dpitch + X0 + x4;
            if (X0 + x4 + 3 < p.w && ((uintptr_t)drow % (4 * sizeof(PIX))) == 0)
            {
                if (sizeof(PIX) == 1) *reinterpret_cast<uchar4 *>(drow) = make_uchar4(out[0], out[1], out[2], out[3]);
                else                  *reinterpret_cast<ushort4 *>(drow) = make_ushort4(out[0], out[1], out[2], out[3]);
            }
            else
            {
#pragma unroll
                for (int q = 0; q < 4; q++)
                    if (X0 + x4 + q < p.w) drow[q] = (PIX)out[q];
            }
        }
    }
}

template <typename PIX>
__global__ void __launch_bounds__(256) plane_copy_kernel(const PIX *__restrict__ src, int spitch, PIX *__restrict__ dst, int dpitch, int w, int h)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x < w && y < h) dst[(size_t)y * dpitch + x] = src[(size_t)y * spitch + x];
}

struct Geom { int w, h, pitch; size_t bytes; };

}  // namespace

struct hbcu_unsharp_s
{
    hbcu_unsharp_config_t cfg;
    int bps, slots, next;
    Geom g[3];
    size_t frame_bytes, plane_off[3];
    std::vector<uint8_t *> in_base, out_base;
    std::vector<int64_t> ticket;
    cudaStream_t s_h2d, s_compute, s_d2h;
    cudaStream_t s_chroma[2];            // the chroma planes run beside luma (forked from / joined to s_compute): their CTAs fill luma's last wave
    cudaEvent_t ev_fork, ev_join[2];
    std::vector<cudaEvent_t> ev_up, ev_k, ev_down;
    cudaEvent_t ev_mark[2];
    uint32_t coef[3][2 * kMaxSteps + 1];
};

namespace {

template <typename PIX>
int launch_steps(const UnsharpParams &p, int steps, dim3 grid, cudaStream_t st)
{
    switch (steps)
    {
        case 1: unsharp_kernel<PIX, 1><<<grid, kThreads, 0, st>>>(p); break;
        case 2: unsharp_kernel<PIX, 2><<<grid, kThreads, 0, st>>>(p); break;
        case 3: unsharp_kernel<PIX, 3><<<grid, kThreads, 0, st>>>(p); break;
        case 4: unsharp_kernel<PIX, 4><<<grid, kThreads, 0, st>>>(p); break;
        case 5: unsharp_kernel<PIX, 5><<<grid, kThreads, 0, st>>>(p); break;
        case 6: unsharp_kernel<PIX, 6><<<grid, kThreads, 0, st>>>(p); break;
        case 7: unsharp_kernel<PIX, 7><<<grid, kThreads, 0, st>>>(p); break;
        default: return -1;
    }
    return 0;
}

int launch_plane(hbcu_unsharp_s *h, int pl, const void *src, void *dst, cudaStream_t st)
{
    const Geom &g = h->g[pl];
    const int amount = h->cfg.amount[pl];
    if (amount == 0)
    {
        // hb_image_copy_plane (unsharp.c:113-117)
        dim3 blk(64, 4), grid((g.w + 63) / 64, (g.h + 3) / 4);
        if (h->bps == 1) plane_copy_kernel<uint8_t><<<grid, blk, 0, st>>>((const uint8_t *)src, g.pitch, (uint8_t *)dst, g.pitch, g.w, g.h);
        else             plane_copy_kernel<uint16_t><<<grid, blk, 0, st>>>((const uint16_t *)src, g.pitch, (uint16_t *)dst, g.pitch, g.w, g.h);
    }
    else
    {
        UnsharpParams p;
        p.src = src; p.dst = dst; p.spitch = g.pitch; p.dpitch = g.pitch; p.w = g.w; p.h = g.h;
        p.amount = amount; p.smooth = h->cfg.smooth;
        const int maxi = 1 << h->cfg.depth;
        // `const int16_t max_value / min_value` in the reference (unsharp.c:108, chroma_smooth.c:112-113)
        p.maxv = (int)(int16_t)(h->cfg.smooth ? maxi - maxi / 16 : maxi - 1);
        p.minv = (int)(int16_t)(h->cfg.smooth ? maxi / 16 : 0);
        memcpy(p.coef, h->coef[pl], sizeof(p.coef));
        dim3 grid((g.w + kTW - 1) / kTW, (g.h + kTH - 1) / kTH);
        const int rc = h->bps == 1 ? launch_steps<uint8_t>(p, h->cfg.steps[pl], grid, st)
                                   : launch_steps<uint16_t>(p, h->cfg.steps[pl], grid, st);
        if (rc != 0) { set_error("unsharp: steps %d out of range", h->cfg.steps[pl]); return -1; }
    }
    hbcu::count_launch();
    HBCU_CHECK(cudaGetLastError());
    return 0;
}

bool same_layout(const hbcu_unsharp_s *h, const void *const planes[3], const int strides[3])
{
    for (int pl = 0; pl < 3; pl++)
    {
        if ((size_t)strides[pl] != (size_t)h->g[pl].pitch * h->bps) return false;
        if ((const uint8_t *)planes[pl] != (const uint8_t *)planes[0] + h->plane_off[pl]) return false;
    }
    return true;
}

bool frame_fits(const hbcu_unsharp_s *h, const hbcu_frame_t *f)
{
    if (f->device != h->cfg.device) return false;
    for (int pl = 0; pl < 3; pl++)
        if (f->row_bytes[pl] != h->g[pl].w * h->bps || f->rows[pl] != h->g[pl].h || f->stride[pl] != h->g[pl].pitch * h->bps) return false;
    return true;
}

int find_slot(const hbcu_unsharp_s *h, int64_t ticket)
{
    for (int s = 0; s < h->slots; s++)
        if (h->ticket[s] == ticket) return s;
    return -1;
}

}  // namespace

extern "C" {

int hbcu_unsharp_create(hbcu_unsharp_t **out, const hbcu_unsharp_config_t *cfg)
{
    if (out == nullptr || cfg == nullptr) { set_error("unsharp_create: null argument"); return -1; }
    *out = nullptr;
    if (cfg->width < 1 || cfg->height < 1 || cfg->depth < 8 || cfg->depth > 16)
    {
        set_error("unsharp_create: unsupported geometry %dx%d depth %d", cfg->width, cfg->height, cfg->depth);
        return -1;
    }
    for (int pl = 0; pl < 3; pl++)
    {
        if (cfg->amount[pl] != 0 && (cfg->steps[pl] < 1 || cfg->steps[pl] > kMaxSteps))
        {
            set_error("unsharp_create: plane %d: size %d out of range", pl, 2 * cfg->steps[pl] + 1);
            return -1;
        }
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || cfg->device < 0 || cfg->device >= ndev)
    {
        cudaGetLastError();
        set_error("unsharp_create: CUDA device %d not available (%d devices); there is no CPU fallback", cfg->device, ndev);
        return -1;
    }
    HBCU_CHECK(cudaSetDevice(cfg->device));
    cudaDeviceProp prop;
    HBCU_CHECK(cudaGetDeviceProperties(&prop, cfg->device));
    if (prop.major != 9 || prop.minor != 0)
    {
        set_error("unsharp_create: device %d is sm_%d%d; this library is built for sm_90a only", cfg->device, prop.major, prop.minor);
        return -1;
    }
    hbcu_unsharp_s *h = new (std::nothrow) hbcu_unsharp_s();
    if (h == nullptr) { set_error("unsharp_create: out of memory"); return -1; }
    h->cfg = *cfg;
    h->bps = cfg->depth > 8 ? 2 : 1;
    h->slots = cfg->slots >= 2 ? cfg->slots : 4;
    h->next = 0;
    h->s_h2d = h->s_compute = h->s_d2h = nullptr;
    h->s_chroma[0] = h->s_chroma[1] = nullptr;
    h->ev_fork = h->ev_join[0] = h->ev_join[1] = nullptr;
    h->ev_mark[0] = h->ev_mark[1] = nullptr;
    for (int pl = 0; pl < 3; pl++)
    {
        Geom &g = h->g[pl];
        g.w = pl == 0 ? cfg->width : -((-cfg->width) >> cfg->chroma_shift_w);
        g.h = pl == 0 ? cfg->height : -((-cfg->height) >> cfg->chroma_shift_h);
        g.pitch = ((g.w * h->bps + 63) / 64 * 64) / h->bps;          // hb_image_stride: the layout of a STANDARD hb_buffer_t
        g.bytes = (size_t)g.pitch * g.h * h->bps;
        h->plane_off[pl] = pl == 0 ? 0 : h->plane_off[pl - 1] + h->g[pl - 1].bytes;
        h->frame_bytes = h->plane_off[pl] + g.bytes;
        // binomial row of order 2*steps
        memset(h->coef[pl], 0, sizeof(h->coef[pl]));
        const int n = 2 * cfg->steps[pl];
        uint64_t c = 1;
        for (int k = 0; k <= n && n <= 2 * kMaxSteps; k++)
        {
            h->coef[pl][k] = (uint32_t)c;
            c = c * (uint64_t)(n - k) / (uint64_t)(k + 1);
        }
    }
#define CK(expr)                                                                  \
    do {                                                                          \
        cudaError_t _e = (expr);                                                  \
        if (_e != cudaSuccess) {                                                  \
            set_error("%s failed: %s", #expr, cudaGetErrorString(_e));            \
            hbcu_unsharp_destroy(h);                                              \
            return -1;                                                            \
        }                                                                         \
    } while (0)
    CK(cudaStreamCreateWithFlags(&h->s_h2d, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&h->s_compute, cudaStreamNonBlocking));
    CK(cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming));
    for (int i = 0; i < 2; i++)
    {
        CK(cudaStreamCreateWithFlags(&h->s_chroma[i], cudaStreamNonBlocking));
        CK(cudaEventCreateWithFlags(&h->ev_join[i], cudaEventDisableTiming));
    }
    CK(cudaStreamCreateWithFlags(&h->s_d2h, cudaStreamNonBlocking));
    h->in_base.assign(h->slots, nullptr);
    h->out_base.assign(h->slots, nullptr);
    h->ticket.assign(h->slots, -1);
    h->ev_up.assign(h->slots, nullptr);
    h->ev_k.assign(h->slots, nullptr);
    h->ev_down.assign(h->slots, nullptr);
    for (int s = 0; s < h->slots; s++)
    {
        CK(cudaEventCreateWithFlags(&h->ev_up[s], cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&h->ev_k[s], cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&h->ev_down[s], cudaEventDisableTiming));
        CK(cudaMalloc(&h->in_base[s], h->frame_bytes));
        CK(cudaMalloc(&h->out_base[s], h->frame_bytes));
        CK(cudaMemset(h->out_base[s], 0, h->frame_bytes));       // the stride padding is never written
    }
    CK(cudaEventCreate(&h->ev_mark[0]));
    CK(cudaEventCreate(&h->ev_mark[1]));
    // the clearing memsets above ran on the legacy default stream; the handle's non-blocking streams do not wait for it
    CK(cudaDeviceSynchronize());
#undef CK
    *out = h;
    return 0;
}

void hbcu_unsharp_destroy(hbcu_unsharp_t *h)
{
    if (h == nullptr) return;
    cudaSetDevice(h->cfg.device);
    cudaDeviceSynchronize();
    for (auto p : h->in_base) if (p) cudaFree(p);
    for (auto p : h->out_base) if (p) cudaFree(p);
    for (auto e : h->ev_up) if (e) cudaEventDestroy(e);
    for (auto e : h->ev_k) if (e) cudaEventDestroy(e);
    for (auto e : h->ev_down) if (e) cudaEventDestroy(e);
    if (h->ev_mark[0]) cudaEventDestroy(h->ev_mark[0]);
    if (h->ev_mark[1]) cudaEventDestroy(h->ev_mark[1]);
    if (h->s_h2d) cudaStreamDestroy(h->s_h2d);
    if (h->s_compute) cudaStreamDestroy(h->s_compute);
    for (int i = 0; i < 2; i++)
    {
        if (h->s_chroma[i]) cudaStreamDestroy(h->s_chroma[i]);
        if (h->ev_join[i]) cudaEventDestroy(h->ev_join[i]);
    }
    if (h->ev_fork) cudaEventDestroy(h->ev_fork);
    if (h->s_d2h) cudaStreamDestroy(h->s_d2h);
    delete h;
}

int hbcu_unsharp_filter_frames(hbcu_unsharp_t *h, int64_t ticket,
                               hbcu_frame_t *in_frame, const void *const in_planes[3], const int in_strides[3],
                               hbcu_frame_t *out_frame, void *const out_planes[3], const int out_strides[3])
{
    if (h == nullptr || (in_frame == nullptr && (in_planes == nullptr || in_strides == nullptr)) ||
        (out_frame == nullptr && (out_planes == nullptr || out_strides == nullptr)) ||
        (in_frame && !frame_fits(h, in_frame)) || (out_frame && !frame_fits(h, out_frame)))
    {
        set_error("unsharp_filter_frames: bad argument or frame geometry");
        return -1;
    }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    const int s = h->next;
    h->next = (h->next + 1) % h->slots;
    if (in_frame == nullptr)
    {
        // the slot's previous frame must have left it (kernel read the input)
        HBCU_CHECK(cudaStreamWaitEvent(h->s_h2d, h->ev_k[s], 0));
        if (same_layout(h, in_planes, in_strides))
            HBCU_CHECK(cudaMemcpyAsync(h->in_base[s], in_planes[0], h->frame_bytes, cudaMemcpyHostToDevice, h->s_h2d));
        else
            for (int pl = 0; pl < 3; pl++)
                HBCU_CHECK(cudaMemcpy2DAsync(h->in_base[s] + h->plane_off[pl], (size_t)h->g[pl].pitch * h->bps, in_planes[pl], (size_t)in_strides[pl],
                                             (size_t)h->g[pl].w * h->bps, (size_t)h->g[pl].h, cudaMemcpyHostToDevice, h->s_h2d));
        HBCU_CHECK(cudaEventRecord(h->ev_up[s], h->s_h2d));
        HBCU_CHECK(cudaStreamWaitEvent(h->s_compute, h->ev_up[s], 0));
    }
    else if (hbcu::frame_begin_read(in_frame, h->s_compute) != 0) return -1;
    HBCU_CHECK(cudaStreamWaitEvent(h->s_compute, h->ev_down[s], 0));
    if (out_frame && hbcu::frame_begin_write(out_frame, h->s_compute) != 0) return -1;
    HBCU_CHECK(cudaEventRecord(h->ev_fork, h->s_compute));
    for (int pl = 0; pl < 3; pl++)
    {
        const void *src = in_frame ? (const void *)in_frame->plane[pl] : (const void *)(h->in_base[s] + h->plane_off[pl]);
        void *dst = out_frame ? (void *)out_frame->plane[pl] : (void *)(h->out_base[s] + h->plane_off[pl]);
        cudaStream_t st = pl == 0 ? h->s_compute : h->s_chroma[pl - 1];
        if (pl > 0) HBCU_CHECK(cudaStreamWaitEvent(st, h->ev_fork, 0));
        if (launch_plane(h, pl, src, dst, st) != 0) return -1;
        if (pl > 0) HBCU_CHECK(cudaEventRecord(h->ev_join[pl - 1], st));
    }
    for (int i = 0; i < 2; i++) HBCU_CHECK(cudaStreamWaitEvent(h->s_compute, h->ev_join[i], 0));
    HBCU_CHECK(cudaEventRecord(h->ev_k[s], h->s_compute));
    if (in_frame && hbcu::frame_end_read(in_frame, h->s_compute) != 0) return -1;
    if (out_frame)
    {
        if (hbcu::frame_end_write(out_frame, h->s_compute) != 0) return -1;
        HBCU_CHECK(cudaEventRecord(h->ev_down[s], h->s_compute));
    }
    else
    {
        HBCU_CHECK(cudaStreamWaitEvent(h->s_d2h, h->ev_k[s], 0));
        if (same_layout(h, out_planes, out_strides))
            HBCU_CHECK(cudaMemcpyAsync(out_planes[0], h->out_base[s], h->frame_bytes, cudaMemcpyDeviceToHost, h->s_d2h));
        else
            for (int pl = 0; pl < 3; pl++)
                HBCU_CHECK(cudaMemcpy2DAsync(out_planes[pl], (size_t)out_strides[pl], h->out_base[s] + h->plane_off[pl], (size_t)h->g[pl].pitch * h->bps,
                                             (size_t)h->g[pl].w * h->bps, (size_t)h->g[pl].h, cudaMemcpyDeviceToHost, h->s_d2h));
        HBCU_CHECK(cudaEventRecord(h->ev_down[s], h->s_d2h));
    }
    h->ticket[s] = ticket;
    return 0;
}

int hbcu_unsharp_wait(hbcu_unsharp_t *h, int64_t ticket)
{
    if (h == nullptr) { set_error("unsharp_wait: null handle"); return -1; }
    const int s = find_slot(h, ticket);
    if (s < 0) { set_error("unsharp_wait: ticket %lld is not in flight", (long long)ticket); return -1; }
    HBCU_CHECK(cudaEventSynchronize(h->ev_down[s]));
    return 0;
}

int hbcu_unsharp_poll(hbcu_unsharp_t *h, int64_t ticket)
{
    if (h == nullptr) { set_error("unsharp_poll: null handle"); return -1; }
    const int s = find_slot(h, ticket);
    if (s < 0) { set_error("unsharp_poll: ticket %lld is not in flight", (long long)ticket); return -1; }
    cudaError_t e = cudaEventQuery(h->ev_down[s]);
    if (e == cudaSuccess) return 1;
    if (e == cudaErrorNotReady) return 0;
    set_error("unsharp_poll: %s", cudaGetErrorString(e));
    return -1;
}

int hbcu_unsharp_sync(hbcu_unsharp_t *h)
{
    if (h == nullptr) { set_error("unsharp_sync: null handle"); return -1; }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    HBCU_CHECK(cudaStreamSynchronize(h->s_h2d));
    HBCU_CHECK(cudaStreamSynchronize(h->s_compute));
    HBCU_CHECK(cudaStreamSynchronize(h->s_d2h));
    return 0;
}

int hbcu_unsharp_mark(hbcu_unsharp_t *h, int which)
{
    if (h == nullptr || which < 0 || which > 1) { set_error("unsharp_mark: bad argument"); return -1; }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    HBCU_CHECK(cudaEventRecord(h->ev_mark[which], h->s_compute));
    return 0;
}

int hbcu_unsharp_elapsed_ms(hbcu_unsharp_t *h, float *ms)
{
    if (h == nullptr || ms == nullptr) { set_error("unsharp_elapsed_ms: bad argument"); return -1; }
    HBCU_CHECK(cudaEventSynchronize(h->ev_mark[1]));
    HBCU_CHECK(cudaEventElapsedTime(ms, h->ev_mark[0], h->ev_mark[1]));
    return 0;
}

}  // extern "C"
