// format.cu -- semi-planar <-> planar 4:2:0 repacks for sm_90a behind the C-ABI of include/hbcu.h (hbcu_format_*).
//
// What the reference's format filter (format.c) asks FFmpeg's avfilter graph for when a job mixes NVDEC's semi-planar
// frames with planar-only filters, or planar filters with a 10-bit NVENC encoder.  Each conversion is a lossless repack
// fully defined by FFmpeg's pixel-format descriptors (component plane, step, offset, shift):
//   nv12        -> yuv420p      luma copied; the Cb/Cr pairs of plane 1 split into planes 1 and 2
//   yuv420p     -> nv12         the reverse
//   p010le      -> yuv420p10le  v >> 6 on every sample (P010 keeps its 10 bits in the high bits); chroma split
//   yuv420p10le -> p010le       v << 6 (kept to 16 bits); chroma interleaved
// Integer only, bit-exact.  Chroma geometry rounds up (hb_image_width / hb_image_height).
//
// Thread mapping: one launch per frame covers every plane.  blockIdx.y is a row: luma rows first, then chroma rows.
// Along a row every thread owns one 16-byte chunk of the row's 16-byte side: 16 bytes of luma, or the 16 bytes of
// interleaved Cb/Cr (8 pairs at 8 bits, 4 at 16) and the two 8-byte runs of planar Cb and Cr they map to.  At 4:2:0 a
// luma row and a chroma row have the same number of chunks, so no thread of a row idles.  A chunk whose rows are
// aligned for the vector width is one 16-byte load and one 16-byte store (luma), or one 16-byte and two 8-byte
// accesses (chroma), with __byte_perm splitting or merging the pairs; a row tail, an odd width or a pitch that breaks
// the alignment takes a scalar loop over the same samples.  Rows are independent: input pitches are whatever the
// producer used (a decoder's pitch, hb_image_stride, any host linesize); nothing outside a row's samples is written.
// HBM bound: read one frame, write one frame.
#include "hbcu_common.h"
#include "hbcu_frames.h"
#include "hbcu_staging.h"
#include "../../include/hbcu.h"

#include <cstdlib>
#include <cstring>
#include <new>

namespace {

using hbcu::set_error;

constexpr int kThreads = 128;

struct FormatArgs
{
    const uint8_t *src[3];       // source planes: 2 for a semi-planar source (src[2] unused)
    uint8_t *dst[3];
    int spitch[3], dpitch[3];    // bytes
    int w, h, cw, ch;            // luma and chroma geometry in samples
    int luma_chunks, chroma_chunks;
};

__device__ __forceinline__ bool aligned(const void *p, unsigned a) { return ((uintptr_t)p & (a - 1)) == 0; }

// two 16-bit samples in one word
template <int SHIFT, bool UP>
__device__ __forceinline__ uint32_t shift2(uint32_t v)
{
    if (SHIFT == 0) return v;
    return UP ? (v << SHIFT) & (((0xFFFFu << SHIFT) & 0xFFFFu) * 0x10001u)
              : (v >> SHIFT) & ((0xFFFFu >> SHIFT) * 0x10001u);
}

template <typename T, int SHIFT, bool UP>
__device__ __forceinline__ T shift1(T v)
{
    return UP ? (T)(v << SHIFT) : (T)(v >> SHIFT);
}

// TO_SEMI: planar -> semi-planar (shift up); otherwise semi-planar -> planar (shift down).  T: uint8_t or uint16_t.
template <typename T, int SHIFT, bool TO_SEMI>
__global__ void __launch_bounds__(kThreads) format_kernel(const FormatArgs a)
{
    const int chunk = blockIdx.x * kThreads + threadIdx.x;
    const int row = blockIdx.y;
    if (row < a.h)
    {
        if (chunk >= a.luma_chunks) return;
        constexpr int NS = 16 / sizeof(T);
        const T *s = (const T *)(a.src[0] + (size_t)row * a.spitch[0]);
        T *d = (T *)(a.dst[0] + (size_t)row * a.dpitch[0]);
        const int x0 = chunk * NS;
        if (x0 + NS <= a.w && aligned(s, 16) && aligned(d, 16))
        {
            uint4 v = __ldg((const uint4 *)(s + x0));
            if (sizeof(T) == 2)
            {
                v.x = shift2<SHIFT, TO_SEMI>(v.x); v.y = shift2<SHIFT, TO_SEMI>(v.y);
                v.z = shift2<SHIFT, TO_SEMI>(v.z); v.w = shift2<SHIFT, TO_SEMI>(v.w);
            }
            *(uint4 *)(d + x0) = v;
        }
        else
        {
            const int x1 = min(x0 + NS, a.w);
            for (int x = x0; x < x1; x++) d[x] = shift1<T, SHIFT, TO_SEMI>(s[x]);
        }
        return;
    }
    if (chunk >= a.chroma_chunks) return;
    const int cy = row - a.h;
    constexpr int G = 8 / sizeof(T);                       // Cb/Cr pairs per chunk: 16 interleaved bytes, 8 per planar plane
    const uint8_t *semi = TO_SEMI ? nullptr : a.src[1] + (size_t)cy * a.spitch[1];
    uint8_t *semi_d = TO_SEMI ? a.dst[1] + (size_t)cy * a.dpitch[1] : nullptr;
    const uint8_t *pu = TO_SEMI ? a.src[1] + (size_t)cy * a.spitch[1] : nullptr;
    const uint8_t *pv = TO_SEMI ? a.src[2] + (size_t)cy * a.spitch[2] : nullptr;
    uint8_t *du = TO_SEMI ? nullptr : a.dst[1] + (size_t)cy * a.dpitch[1];
    uint8_t *dv = TO_SEMI ? nullptr : a.dst[2] + (size_t)cy * a.dpitch[2];
    const int p0 = chunk * G;
    if (TO_SEMI)
    {
        if (p0 + G <= a.cw && aligned(pu, 8) && aligned(pv, 8) && aligned(semi_d, 16))
        {
            const uint2 u = __ldg((const uint2 *)(pu + p0 * sizeof(T)));
            const uint2 v = __ldg((const uint2 *)(pv + p0 * sizeof(T)));
            uint4 o;
            if (sizeof(T) == 1)
            {
                // u = u0..u7, v = v0..v7  ->  u0 v0 u1 v1 | u2 v2 u3 v3 | ...
                o.x = __byte_perm(u.x, v.x, 0x5140); o.y = __byte_perm(u.x, v.x, 0x7362);
                o.z = __byte_perm(u.y, v.y, 0x5140); o.w = __byte_perm(u.y, v.y, 0x7362);
            }
            else
            {
                // u = u0 u1 | u2 u3 (16-bit)  ->  u0 v0 | u1 v1 | u2 v2 | u3 v3
                o.x = shift2<SHIFT, true>(__byte_perm(u.x, v.x, 0x5410)); o.y = shift2<SHIFT, true>(__byte_perm(u.x, v.x, 0x7632));
                o.z = shift2<SHIFT, true>(__byte_perm(u.y, v.y, 0x5410)); o.w = shift2<SHIFT, true>(__byte_perm(u.y, v.y, 0x7632));
            }
            *(uint4 *)(semi_d + 2 * p0 * sizeof(T)) = o;
        }
        else
        {
            const int p1 = min(p0 + G, a.cw);
            for (int p = p0; p < p1; p++)
            {
                ((T *)semi_d)[2 * p]     = shift1<T, SHIFT, true>(((const T *)pu)[p]);
                ((T *)semi_d)[2 * p + 1] = shift1<T, SHIFT, true>(((const T *)pv)[p]);
            }
        }
    }
    else
    {
        if (p0 + G <= a.cw && aligned(semi, 16) && aligned(du, 8) && aligned(dv, 8))
        {
            const uint4 i = __ldg((const uint4 *)(semi + 2 * p0 * sizeof(T)));
            uint2 u, v;
            if (sizeof(T) == 1)
            {
                // u0 v0 u1 v1 | u2 v2 u3 v3 | ...  ->  u0..u7, v0..v7
                u.x = __byte_perm(i.x, i.y, 0x6420); v.x = __byte_perm(i.x, i.y, 0x7531);
                u.y = __byte_perm(i.z, i.w, 0x6420); v.y = __byte_perm(i.z, i.w, 0x7531);
            }
            else
            {
                u.x = shift2<SHIFT, false>(__byte_perm(i.x, i.y, 0x5410)); v.x = shift2<SHIFT, false>(__byte_perm(i.x, i.y, 0x7632));
                u.y = shift2<SHIFT, false>(__byte_perm(i.z, i.w, 0x5410)); v.y = shift2<SHIFT, false>(__byte_perm(i.z, i.w, 0x7632));
            }
            *(uint2 *)(du + p0 * sizeof(T)) = u;
            *(uint2 *)(dv + p0 * sizeof(T)) = v;
        }
        else
        {
            const int p1 = min(p0 + G, a.cw);
            for (int p = p0; p < p1; p++)
            {
                ((T *)du)[p] = shift1<T, SHIFT, false>(((const T *)semi)[2 * p]);
                ((T *)dv)[p] = shift1<T, SHIFT, false>(((const T *)semi)[2 * p + 1]);
            }
        }
    }
}

}  // namespace

struct hbcu_format_s
{
    hbcu_format_config_t cfg;
    int bps;
    int cw, ch;
    hbcu::Staging st;                        // in / out: the two sides' planes; the third plane of the semi-planar side
                                             // has 0 rows
};

namespace {

int launch(hbcu_format_s *h, const uint8_t *const src[3], const int spitch[3], uint8_t *const dst[3], const int dpitch[3])
{
    FormatArgs a;
    for (int p = 0; p < 3; p++)
    {
        a.src[p] = src[p]; a.dst[p] = dst[p];
        a.spitch[p] = spitch[p]; a.dpitch[p] = dpitch[p];
    }
    a.w = h->cfg.width; a.h = h->cfg.height; a.cw = h->cw; a.ch = h->ch;
    a.luma_chunks = (a.w * h->bps + 15) / 16;
    a.chroma_chunks = (2 * a.cw * h->bps + 15) / 16;
    const int chunks = a.luma_chunks > a.chroma_chunks ? a.luma_chunks : a.chroma_chunks;
    const dim3 grid((chunks + kThreads - 1) / kThreads, a.h + a.ch);
    const bool semi = h->cfg.to_semi_planar != 0;
    cudaStream_t st = h->st.s_compute;
    if (h->bps == 1)
    {
        if (semi) format_kernel<uint8_t, 0, true><<<grid, kThreads, 0, st>>>(a);
        else      format_kernel<uint8_t, 0, false><<<grid, kThreads, 0, st>>>(a);
    }
    else
    {
        if (semi) format_kernel<uint16_t, 6, true><<<grid, kThreads, 0, st>>>(a);
        else      format_kernel<uint16_t, 6, false><<<grid, kThreads, 0, st>>>(a);
    }
    hbcu::count_launch();
    HBCU_CHECK(cudaGetLastError());
    return 0;
}

// the planes of one side: semi-planar (Y, Cb/Cr pairs) or planar (Y, Cb, Cr)
size_t side_layout(hbcu::StagePlane g[3], bool semi, int w, int h, int cw, int ch, int bps)
{
    const int rb[3] = {w * bps, semi ? 2 * cw * bps : cw * bps, semi ? 0 : cw * bps};
    const int rows[3] = {h, ch, semi ? 0 : ch};
    return hbcu::stage_layout(g, rb, rows);
}

}  // namespace

extern "C" {

int hbcu_format_create(hbcu_format_t **out, const hbcu_format_config_t *cfg)
{
    if (out == nullptr || cfg == nullptr) { set_error("format_create: null argument"); return -1; }
    *out = nullptr;
    const int ch = (cfg->height + 1) >> 1;
    if (cfg->width < 1 || cfg->height < 1 || cfg->width > (1 << 16) || cfg->height + ch > 65535 ||
        (cfg->depth != 8 && cfg->depth != 10))
    {
        set_error("format_create: unsupported geometry %dx%d or depth %d (8: nv12 / yuv420p, 10: p010le / yuv420p10le)",
                  cfg->width, cfg->height, cfg->depth);
        return -1;
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || cfg->device < 0 || cfg->device >= ndev)
    {
        cudaGetLastError();
        set_error("format_create: CUDA device %d not available (%d devices); there is no CPU fallback", cfg->device, ndev);
        return -1;
    }
    HBCU_CHECK(cudaSetDevice(cfg->device));
    cudaDeviceProp prop;
    HBCU_CHECK(cudaGetDeviceProperties(&prop, cfg->device));
    if (prop.major != 9 || prop.minor != 0)
    {
        set_error("format_create: device %d is sm_%d%d; this library is built for sm_90a only", cfg->device, prop.major, prop.minor);
        return -1;
    }
    hbcu_format_s *h = new (std::nothrow) hbcu_format_s();
    if (h == nullptr) { set_error("format_create: out of memory"); return -1; }
    h->cfg = *cfg;
    h->bps = cfg->depth > 8 ? 2 : 1;
    h->cw = (cfg->width + 1) >> 1;
    h->ch = ch;
    const bool to_semi = cfg->to_semi_planar != 0;
    h->st.in_bytes = side_layout(h->st.in, !to_semi, cfg->width, cfg->height, h->cw, h->ch, h->bps);
    h->st.out_bytes = side_layout(h->st.out, to_semi, cfg->width, cfg->height, h->cw, h->ch, h->bps);
    if (hbcu::stage_init(&h->st, "format", cfg->device, cfg->slots >= 2 ? cfg->slots : 4) != 0)
    {
        hbcu_format_destroy(h);
        return -1;
    }
    *out = h;
    return 0;
}

void hbcu_format_destroy(hbcu_format_t *h)
{
    if (h == nullptr) return;
    hbcu::stage_destroy(&h->st);
    delete h;
}

int hbcu_format_convert(hbcu_format_t *h, int64_t ticket,
                        hbcu_frame_t *in_frame, const void *const in_planes[3], const int in_strides[3],
                        hbcu_frame_t *out_frame, void *const out_planes[3], const int out_strides[3])
{
    if (h == nullptr) { set_error("format_convert: bad argument"); return -1; }
    return hbcu::stage_submit(&h->st, "convert", ticket, in_frame, in_planes, in_strides, out_frame, out_planes, out_strides,
                              [h](const uint8_t *const src[3], const int spitch[3], uint8_t *const dst[3], const int dpitch[3])
                              { return launch(h, src, spitch, dst, dpitch); });
}

int hbcu_format_wait(hbcu_format_t *h, int64_t ticket)
{
    if (h == nullptr) { set_error("format_wait: null handle"); return -1; }
    return hbcu::stage_wait(&h->st, ticket);
}

int hbcu_format_poll(hbcu_format_t *h, int64_t ticket)
{
    if (h == nullptr) { set_error("format_poll: null handle"); return -1; }
    return hbcu::stage_poll(&h->st, ticket);
}

int hbcu_format_sync(hbcu_format_t *h)
{
    if (h == nullptr) { set_error("format_sync: null handle"); return -1; }
    return hbcu::stage_sync(&h->st);
}

int hbcu_format_mark(hbcu_format_t *h, int which)
{
    if (h == nullptr || which < 0 || which > 1) { set_error("format_mark: bad argument"); return -1; }
    return hbcu::stage_mark(&h->st, which);
}

int hbcu_format_elapsed_ms(hbcu_format_t *h, float *ms)
{
    if (h == nullptr || ms == nullptr) { set_error("format_elapsed_ms: bad argument"); return -1; }
    return hbcu::stage_elapsed_ms(&h->st, ms);
}

}  // extern "C"
