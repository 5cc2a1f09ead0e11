// deinterlace.cu -- Yadif and Bwdif deinterlacing for sm_90a behind the C-ABI of include/hbcu.h (hbcu_deint_*).
//
// What libhb's Deinterlace filter (deinterlace.c) asks FFmpeg's avfilter graph for: yadif or bwdif, one picture per
// frame or one per field.  The arithmetic is restated in DESIGN.md 4.9, rule by rule; the names below (c, e, d, td0..2,
// diff, m, n, df) are the ones used there.
//
// One launch per frame covers every plane through a flat work list (as rotate.cu does): a work unit is one sample
// column x of one row pair (2r, 2r+1) of one plane.  For each of the two rows and each picture k the thread either
// copies cur or filters, so every thread of a picture filters exactly one sample per row pair and the warps stay
// uniform; in field mode the two pictures' parities differ, so the row one picture copies is the row the other
// filters, and the thread reads cur's rows once for both (the neighbour rows come from L1).  Loads go through the
// read-only path; all arithmetic is in 32-bit ints, with >> an arithmetic shift.  HBM bound: 3.5 frames of traffic per
// picture in frame mode, 5 per frame in field mode (DESIGN.md 4.9).
#include "hbcu_common.h"
#include "hbcu_frames.h"
#include "../../include/hbcu.h"

#include <climits>
#include <new>

namespace {

using hbcu::set_error;

constexpr int kThreads = 256;

struct DeintPlane
{
    const uint8_t *src[3];       // prev, cur, next
    int spitch[3];               // bytes
    uint8_t *dst[2];             // pictures 0 and 1
    int dpitch[2];
    int w, h;                    // samples
};

struct DeintArgs
{
    DeintPlane p[3];
    unsigned first[4];           // first work unit of each plane; [3] = total
    int npics, parity[2], intra[2];
    int tff, spatial, maxv, df;
};

struct Src { const uint8_t *b; int pitch; };

// the five views of one picture: prev, cur, next and the field pair p = parity ^ tff picks, (prev2, next2)
struct Rows { Src prev, cur, next, prev2, next2; };

template <typename T>
__device__ __forceinline__ int at(const Src &s, int y, int x)
{
    return (int)__ldg((const T *)(s.b + (size_t)y * s.pitch) + x);
}

__device__ __forceinline__ int imax3(int a, int b, int c) { return max(a, max(b, c)); }
__device__ __forceinline__ int imin3(int a, int b, int c) { return min(a, min(b, c)); }

// Yadif at (x, y): DESIGN.md 4.9, "Yadif"
template <typename T>
__device__ int yadif_sample(const Rows &R, int x, int y, int w, int h, bool spatial)
{
    const int m = y ? -1 : 1, n = y + 1 < h ? 1 : -1;
    const int c = at<T>(R.cur, y + m, x), e = at<T>(R.cur, y + n, x);
    const int a2 = at<T>(R.prev2, y, x), b2 = at<T>(R.next2, y, x);
    const int d = (a2 + b2) >> 1;
    const int td0 = abs(a2 - b2);
    const int td1 = (abs(at<T>(R.prev, y + m, x) - c) + abs(at<T>(R.prev, y + n, x) - e)) >> 1;
    const int td2 = (abs(at<T>(R.next, y + m, x) - c) + abs(at<T>(R.next, y + n, x) - e)) >> 1;
    int diff = imax3(td0 >> 1, td1, td2);
    int pred = (c + e) >> 1;
    if (x >= 3 && x < w - 3)
    {
        const Src U = {R.cur.b + (size_t)(y + m) * R.cur.pitch, 0}, D = {R.cur.b + (size_t)(y + n) * R.cur.pitch, 0};
        int score = abs(at<T>(U, 0, x - 1) - at<T>(D, 0, x - 1)) + abs(c - e) + abs(at<T>(U, 0, x + 1) - at<T>(D, 0, x + 1)) - 1;
#pragma unroll
        for (int side = -1; side <= 1; side += 2)
        {
#pragma unroll
            for (int j = side; j == side || j == 2 * side; j += side)
            {
                const int s = abs(at<T>(U, 0, x - 1 + j) - at<T>(D, 0, x - 1 - j)) + abs(at<T>(U, 0, x + j) - at<T>(D, 0, x - j)) +
                              abs(at<T>(U, 0, x + 1 + j) - at<T>(D, 0, x + 1 - j));
                if (s >= score) break;           // CHECK(+-2) only after CHECK(+-1) improved the score
                score = s;
                pred = (at<T>(U, 0, x + j) + at<T>(D, 0, x - j)) >> 1;
            }
        }
    }
    if (spatial && y != 1 && y != h - 2)
    {
        const int b = (at<T>(R.prev2, y + 2 * m, x) + at<T>(R.next2, y + 2 * m, x)) >> 1;
        const int f = (at<T>(R.prev2, y + 2 * n, x) + at<T>(R.next2, y + 2 * n, x)) >> 1;
        // -max(d-e, d-c, min(b-c, f-e)) written as the minimum of the negated terms: ptxas (CUDA 12.9) fuses
        // max(diff, max(mn, -mx)) into one 3-input VIMNMX3 and drops the negation (tools/ptxas_vimnmx3_negate.cu)
        const int nmx = imin3(e - d, c - d, max(c - b, e - f));
        const int mn = imin3(d - e, d - c, max(b - c, f - e));
        diff = imax3(diff, mn, nmx);
    }
    return pred > d + diff ? d + diff : pred < d - diff ? d - diff : pred;
}

// Bwdif at (x, y): DESIGN.md 4.9, "Bwdif"
template <typename T>
__device__ int bwdif_sample(const Rows &R, int x, int y, int w, int h, bool intra, int df, int maxv)
{
    if (intra)
    {
        // rows the row-step quirk puts outside a plane of 4..6 rows (9-16-bit) are clamped to the plane
        const int m = y > df - 1 ? -1 : 1, n = y + df < h ? 1 : -1;
        const int m3 = y > 3 * df - 1 ? -3 : 1, n3 = y + 3 * df < h ? 3 : -1;
        const int c = at<T>(R.cur, y + m, x), e = at<T>(R.cur, y + n, x);
        const int r3 = at<T>(R.cur, min(max(y + m3, 0), h - 1), x) + at<T>(R.cur, min(max(y + n3, 0), h - 1), x);
        return min(max((5077 * (c + e) - 981 * r3) >> 13, 0), maxv);
    }
    const bool edge = y < 4 || y + 5 > h;
    const int m = edge ? (y > df - 1 ? -1 : 1) : -1, n = edge ? (y + df < h ? 1 : -1) : 1;
    const int c = at<T>(R.cur, y + m, x), e = at<T>(R.cur, y + n, x);
    const int a2 = at<T>(R.prev2, y, x), b2 = at<T>(R.next2, y, x);
    const int d = (a2 + b2) >> 1;
    const int td0 = abs(a2 - b2);
    const int td1 = (abs(at<T>(R.prev, y + m, x) - c) + abs(at<T>(R.prev, y + n, x) - e)) >> 1;
    const int td2 = (abs(at<T>(R.next, y + m, x) - c) + abs(at<T>(R.next, y + n, x) - e)) >> 1;
    int diff = imax3(td0 >> 1, td1, td2);
    if (diff == 0) return d;
    const bool spat = !edge || !(y < 2 || y + 3 > h);
    int pu2 = 0, pd2 = 0;
    if (spat)
    {
        pu2 = at<T>(R.prev2, y - 2, x) + at<T>(R.next2, y - 2, x);
        pd2 = at<T>(R.prev2, y + 2, x) + at<T>(R.next2, y + 2, x);
        const int b = (pu2 >> 1) - c, f = (pd2 >> 1) - e;
        const int nmx = imin3(e - d, c - d, max(-b, -f));     // -max(d-e, d-c, min(b, f)), as in yadif_sample
        const int mn = imin3(d - e, d - c, max(b, f));
        diff = imax3(diff, mn, nmx);
    }
    int interpol;
    if (edge)
    {
        interpol = (c + e) >> 1;
    }
    else
    {
        const int r3 = at<T>(R.cur, y - 3, x) + at<T>(R.cur, y + 3, x);
        if (abs(c - e) > td0)
        {
            const int p4 = at<T>(R.prev2, y - 4, x) + at<T>(R.next2, y - 4, x) + at<T>(R.prev2, y + 4, x) + at<T>(R.next2, y + 4, x);
            interpol = (((5570 * (a2 + b2) - 3801 * (pu2 + pd2) + 1016 * p4) >> 2) + 4309 * (c + e) - 213 * r3) >> 13;
        }
        else
        {
            interpol = (5077 * (c + e) - 981 * r3) >> 13;
        }
    }
    interpol = interpol > d + diff ? d + diff : interpol < d - diff ? d - diff : interpol;
    return min(max(interpol, 0), maxv);
}

__device__ __forceinline__ int plane_of(const DeintArgs &a, unsigned u)
{
    return u >= a.first[1] ? (u >= a.first[2] ? 2 : 1) : 0;
}

template <typename T, bool BWDIF>
__global__ void __launch_bounds__(kThreads) deint_kernel(const DeintArgs a)
{
    const unsigned g = blockIdx.x * kThreads + threadIdx.x;
    if (g >= a.first[3]) return;
    const int pl = plane_of(a, g);
    const DeintPlane P = pl == 0 ? a.p[0] : pl == 1 ? a.p[1] : a.p[2];
    const unsigned u = g - (pl == 0 ? a.first[0] : pl == 1 ? a.first[1] : a.first[2]);
    const int x = (int)(u % (unsigned)P.w), y0 = 2 * (int)(u / (unsigned)P.w);
    const Src prev = {P.src[0], P.spitch[0]}, cur = {P.src[1], P.spitch[1]}, next = {P.src[2], P.spitch[2]};
#pragma unroll
    for (int dy = 0; dy < 2; dy++)
    {
        const int y = y0 + dy;
        if (y >= P.h) break;
        const T kept = (T)at<T>(cur, y, x);
#pragma unroll
        for (int k = 0; k < 2; k++)
        {
            if (k >= a.npics) break;
            const int parity = a.parity[k];
            T v = kept;
            if ((y ^ parity) & 1)
            {
                const bool p = (parity ^ a.tff) != 0;
                const Rows R = {prev, cur, next, p ? prev : cur, p ? cur : next};
                v = BWDIF ? (T)bwdif_sample<T>(R, x, y, P.w, P.h, a.intra[k] != 0, a.df, a.maxv)
                          : (T)yadif_sample<T>(R, x, y, P.w, P.h, a.spatial != 0);
            }
            ((T *)(P.dst[k] + (size_t)y * P.dpitch[k]))[x] = v;
        }
    }
}

}  // namespace

struct hbcu_deint_s
{
    hbcu_deint_config_t cfg;
    DeintArgs geom;              // everything but the plane pointers, pitches and per-call flags
    unsigned blocks;
    cudaStream_t st = nullptr;
    cudaEvent_t ev_mark[2] = {nullptr, nullptr};
};

extern "C" {

int hbcu_deint_create(hbcu_deint_t **out, const hbcu_deint_config_t *cfg)
{
    if (out == nullptr || cfg == nullptr) { set_error("deint_create: null argument"); return -1; }
    *out = nullptr;
    if (cfg->algorithm != HBCU_DEINT_YADIF && cfg->algorithm != HBCU_DEINT_BWDIF)
    {
        set_error("deint_create: unknown algorithm %d", cfg->algorithm);
        return -1;
    }
    if (!((cfg->sample_bytes == 1 && cfg->depth == 8) || (cfg->sample_bytes == 2 && cfg->depth >= 9 && cfg->depth <= 16)))
    {
        set_error("deint_create: %d-byte samples of %d bits (1 byte at 8 bits, 2 bytes at 9-16 bits)", cfg->sample_bytes, cfg->depth);
        return -1;
    }
    const int min_w = cfg->algorithm == HBCU_DEINT_BWDIF ? 3 : 1, min_h = cfg->algorithm == HBCU_DEINT_BWDIF ? 4 : 2;
    for (int p = 0; p < 3; p++)
        if (cfg->width[p] < min_w || cfg->height[p] < min_h || cfg->width[p] > (1 << 16) || cfg->height[p] > (1 << 16))
        {
            set_error("deint_create: plane %d is %dx%d samples", p, cfg->width[p], cfg->height[p]);
            return -1;
        }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || cfg->device < 0 || cfg->device >= ndev)
    {
        cudaGetLastError();
        set_error("deint_create: CUDA device %d not available (%d devices); there is no CPU fallback", cfg->device, ndev);
        return -1;
    }
    HBCU_CHECK(cudaSetDevice(cfg->device));
    cudaDeviceProp prop;
    HBCU_CHECK(cudaGetDeviceProperties(&prop, cfg->device));
    if (prop.major != 9 || prop.minor != 0)
    {
        set_error("deint_create: device %d is sm_%d%d; this library is built for sm_90a only", cfg->device, prop.major, prop.minor);
        return -1;
    }
    hbcu_deint_s *h = new (std::nothrow) hbcu_deint_s();
    if (h == nullptr) { set_error("deint_create: out of memory"); return -1; }
    h->cfg = *cfg;
    DeintArgs &g = h->geom;
    g = DeintArgs();
    size_t total = 0;
    for (int p = 0; p < 3; p++)
    {
        g.first[p] = (unsigned)total;
        g.p[p].w = cfg->width[p];
        g.p[p].h = cfg->height[p];
        total += (size_t)cfg->width[p] * ((cfg->height[p] + 1) / 2);
    }
    g.first[3] = (unsigned)total;
    g.maxv = (1 << cfg->depth) - 1;
    g.df = cfg->sample_bytes;
    h->blocks = (unsigned)((total + kThreads - 1) / kThreads);
    if (total > (size_t)INT_MAX)
    {
        set_error("deint_create: frame too large");
        delete h;
        return -1;
    }
    if (cudaStreamCreateWithFlags(&h->st, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreate(&h->ev_mark[0]) != cudaSuccess || cudaEventCreate(&h->ev_mark[1]) != cudaSuccess)
    {
        set_error("deint_create: %s", cudaGetErrorString(cudaGetLastError()));
        hbcu_deint_destroy(h);
        return -1;
    }
    *out = h;
    return 0;
}

void hbcu_deint_destroy(hbcu_deint_t *h)
{
    if (h == nullptr) return;
    cudaSetDevice(h->cfg.device);
    if (h->st) cudaStreamSynchronize(h->st);
    if (h->ev_mark[0]) cudaEventDestroy(h->ev_mark[0]);
    if (h->ev_mark[1]) cudaEventDestroy(h->ev_mark[1]);
    if (h->st) cudaStreamDestroy(h->st);
    delete h;
}

static bool frame_fits(const hbcu_deint_s *h, const hbcu_frame_t *f)
{
    if (f == nullptr || f->device != h->cfg.device) return false;
    for (int p = 0; p < 3; p++)
        if (f->plane[p] == nullptr || f->rows[p] != h->cfg.height[p] || f->row_bytes[p] != h->cfg.width[p] * h->cfg.sample_bytes)
            return false;
    return true;
}

int hbcu_deint_frame(hbcu_deint_t *h, hbcu_frame_t *prev, hbcu_frame_t *cur, hbcu_frame_t *next, int tff, int spatial,
                     int npictures, hbcu_frame_t *const out[2], const int parity[2], const int intra[2])
{
    if (h == nullptr || out == nullptr || parity == nullptr || intra == nullptr || npictures < 1 || npictures > 2)
    {
        set_error("deint_frame: bad argument");
        return -1;
    }
    hbcu_frame_t *src[3] = {prev, cur, next};
    for (int f = 0; f < 3; f++)
        if (!frame_fits(h, src[f])) { set_error("deint_frame: source %d does not match the handle's geometry", f); return -1; }
    for (int k = 0; k < npictures; k++)
        if (!frame_fits(h, out[k]) || out[k] == prev || out[k] == cur || out[k] == next || (k == 1 && out[1] == out[0]))
        {
            set_error("deint_frame: output %d does not match the handle's geometry, or is a source", k);
            return -1;
        }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    for (int f = 0; f < 3; f++)
        if (hbcu::frame_begin_read(src[f], h->st) != 0) return -1;
    for (int k = 0; k < npictures; k++)
        if (hbcu::frame_begin_write(out[k], h->st) != 0) return -1;
    DeintArgs a = h->geom;
    for (int p = 0; p < 3; p++)
    {
        for (int f = 0; f < 3; f++) { a.p[p].src[f] = src[f]->plane[p]; a.p[p].spitch[f] = src[f]->stride[p]; }
        for (int k = 0; k < 2; k++)
        {
            a.p[p].dst[k] = k < npictures ? out[k]->plane[p] : nullptr;
            a.p[p].dpitch[k] = k < npictures ? out[k]->stride[p] : 0;
        }
    }
    a.npics = npictures;
    for (int k = 0; k < 2; k++) { a.parity[k] = k < npictures ? parity[k] & 1 : 0; a.intra[k] = k < npictures && intra[k]; }
    a.tff = tff ? 1 : 0;
    a.spatial = spatial ? 1 : 0;
    const bool bw = h->cfg.algorithm == HBCU_DEINT_BWDIF;
    if (h->cfg.sample_bytes == 1)
    {
        if (bw) deint_kernel<uint8_t, true><<<h->blocks, kThreads, 0, h->st>>>(a);
        else    deint_kernel<uint8_t, false><<<h->blocks, kThreads, 0, h->st>>>(a);
    }
    else
    {
        if (bw) deint_kernel<uint16_t, true><<<h->blocks, kThreads, 0, h->st>>>(a);
        else    deint_kernel<uint16_t, false><<<h->blocks, kThreads, 0, h->st>>>(a);
    }
    hbcu::count_launch();
    HBCU_CHECK(cudaGetLastError());
    for (int f = 0; f < 3; f++)
        if (hbcu::frame_end_read(src[f], h->st) != 0) return -1;
    for (int k = 0; k < npictures; k++)
        if (hbcu::frame_end_write(out[k], h->st) != 0) return -1;
    return 0;
}

int hbcu_deint_sync(hbcu_deint_t *h)
{
    if (h == nullptr) { set_error("deint_sync: null handle"); return -1; }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    HBCU_CHECK(cudaStreamSynchronize(h->st));
    return 0;
}

int hbcu_deint_mark(hbcu_deint_t *h, int which)
{
    if (h == nullptr || which < 0 || which > 1) { set_error("deint_mark: bad argument"); return -1; }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    HBCU_CHECK(cudaEventRecord(h->ev_mark[which], h->st));
    return 0;
}

int hbcu_deint_elapsed_ms(hbcu_deint_t *h, float *ms)
{
    if (h == nullptr || ms == nullptr) { set_error("deint_elapsed_ms: bad argument"); return -1; }
    HBCU_CHECK(cudaEventSynchronize(h->ev_mark[1]));
    HBCU_CHECK(cudaEventElapsedTime(ms, h->ev_mark[0], h->ev_mark[1]));
    return 0;
}

}  // extern "C"
