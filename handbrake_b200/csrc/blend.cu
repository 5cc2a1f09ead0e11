// blend.cu -- subtitle overlay compositing for sm_90a behind the C-ABI of include/hbcu.h.
//
// Replaces (reference: HandBrake's libhb): blend8on8 / blend8on1x (blend.c:425-604, the plain path: overlay and frame
// share their chroma subsampling) and blend_subsample_8on8 / blend_subsample_8on1x (blend.c:48-140, 236-328: a YUVA
// 4:4:4 overlay on a 4:2:0 or 4:2:2 frame).  Bit-exact with the reference for every sample inside the picture:
//   - every value is uint32; the plain path divides by max = (256 << shift) - 1 without rounding, the subsample path
//     adds max >> 1 first, then averages the blended chroma of a group with the chroma-location weights
//     coeff[0][x] * coeff[1][y] and rounds (accu + accu_c / 2) / accu_c;
//   - the loop bounds are the reference's, quirks included (the subsample clip is min(overlay, frame) in size, the
//     plain clip of an overlay that starts left of the picture is wider than the overlay's visible part);
//   - overlays are applied in list order, so a sample covered by several sees them in that order.
// The one deliberate difference: the reference writes samples outside the picture in some of those cases (an overlay
// crossing the right or bottom edge in the subsample path, an odd negative position or an overlay wider than the frame
// in the plain path); here nothing outside the picture is ever written.
//
// Semi-planar 4:2:0 frames (NV12, P010, P016: plane 1 holds Cb/Cr pairs) follow blend.c's own *bi* functions
// (blend8onbi8 / blend8onbi1x, blend.c:606-786; blend_subsample_8onbi8 / blend_subsample_8onbi1x, blend.c:142-234,
// 330-422), which are not the planar ones with another address:
//   - above 8 bits an overlay sample v enters as av_bswap16(v) = v << 8, whatever the depth; alpha is still
//     << (depth - 8) and max still (256 << (depth - 8)) - 1 (blend.c:193, 214-217, 747, 778-783);
//   - blend_subsample_8onbi8's group loops do not stop at the overlay's right / bottom edge (blend.c:388-390): every
//     sample of the group is weighted into accu_c, the ones outside the overlay with the frame's unblended chroma.
//
// Thread mapping: one thread per chroma group (2x2, 2x1 or 1x1 luma samples and the chroma sample they share) of the
// union of the rectangles the overlays can touch; each thread loads its samples once, runs through all overlay
// descriptors in order and stores once.  A frame is one launch whatever the number of overlays.  No two groups share a
// sample, so threads never communicate.
//
// Overlays are copied into page-locked staging when they are handed over (the caller frees them right after) and
// uploaded on the handle's stream; two slots alternate, each guarded by an event, so a new list never overwrites the
// one a queued blend still reads.  An unchanged list (changed == 0, same count and geometry) is not uploaded again.
#include "hbcu_common.h"
#include "hbcu_frames.h"
#include "../../include/hbcu.h"

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>

namespace {

using hbcu::set_error;

std::atomic<uint64_t> g_uploads{0};

constexpr int kThreads = 128;
constexpr int kSlots = 2;

struct OvDesc
{
    int x, y, w, h;
    uint32_t off[4];          // byte offsets of Y, Cb, Cr, A in the slot's blob
    int stride[4];
};

struct BlendArgs
{
    uint8_t *plane[3];
    int pitch[3];             // bytes
    int W, H, CW, CH;
    int ws, hs;
    int shift;
    int oshift;               // overlay samples enter as v << oshift: shift, or 8 on a semi-planar frame above 8 bits
    int full_groups;          // blend_subsample_8onbi8: weigh every sample of a group (blend.c:388-390)
    unsigned maxv;
    unsigned c0[4], c1[4];
    int gx0, gy0, gw;
    const uint8_t *blob;
    const OvDesc *ov;
    int n;
};

template <typename T>
__device__ __forceinline__ unsigned ld(const uint8_t *plane, int pitch, int x, int y)
{
    return reinterpret_cast<const T *>(plane + (size_t)y * pitch)[x];
}

template <typename T>
__device__ __forceinline__ void st(uint8_t *plane, int pitch, int x, int y, unsigned v)
{
    reinterpret_cast<T *>(plane + (size_t)y * pitch)[x] = (T)v;
}

// SUB: blend_subsample_8on{8,1x}; else blend8on{8,1x}.  NV: the *bi* variants, Cb/Cr interleaved in plane 1.
// T: the frame's sample type.
template <typename T, bool SUB, bool NV>
__global__ void __launch_bounds__(kThreads) blend_kernel(const BlendArgs a)
{
    const int gx = a.gx0 + blockIdx.x * kThreads + threadIdx.x;
    const int gy = a.gy0 + blockIdx.y;
    if (gx >= a.gx0 + a.gw) return;
    const int sw = 1 << a.ws, sh = 1 << a.hs;
    const int X = gx << a.ws, Y = gy << a.hs;
    const unsigned maxv = a.maxv, half = maxv >> 1;
    const int shift = a.shift, oshift = a.oshift;

    unsigned yv[2][2] = {{0, 0}, {0, 0}};
    for (int j = 0; j < sh; j++)
        for (int i = 0; i < sw; i++)
            if (X + i < a.W && Y + j < a.H) yv[j][i] = ld<T>(a.plane[0], a.pitch[0], X + i, Y + j);
    unsigned u = NV ? ld<T>(a.plane[1], a.pitch[1], 2 * gx, gy) : ld<T>(a.plane[1], a.pitch[1], gx, gy);
    unsigned v = NV ? ld<T>(a.plane[1], a.pitch[1], 2 * gx + 1, gy) : ld<T>(a.plane[2], a.pitch[2], gx, gy);

    for (int k = 0; k < a.n; k++)
    {
        const OvDesc o = a.ov[k];
        const uint8_t *oY = a.blob + o.off[0], *oU = a.blob + o.off[1], *oV = a.blob + o.off[2], *oA = a.blob + o.off[3];
        if (SUB)
        {
            // blend.c:57-74: the clip reduces to min(overlay, frame) in size
            const int width = min(o.w, a.W), height = min(o.h, a.H);
            for (int j = 0; j < sh; j++)
                for (int i = 0; i < sw; i++)
                {
                    const int ox = X + i - o.x, oy = Y + j - o.y;
                    if (X + i < a.W && Y + j < a.H && ox >= 0 && ox < width && oy >= 0 && oy < height)
                    {
                        const unsigned alpha = (unsigned)oA[oy * o.stride[3] + ox] << shift;
                        yv[j][i] = (yv[j][i] * (maxv - alpha) + ((unsigned)oY[oy * o.stride[0] + ox] << oshift) * alpha + half) / maxv;
                    }
                }
            // the chroma of a group is visited when its top-left luma sample is inside the loop (blend.c:81-102)
            const int x0c = max(0, o.x & ~(sw - 1)), y0c = max(0, o.y & ~(sh - 1));
            const int ox = X - o.x, oy = Y - o.y;
            if (X >= x0c && ox < width && Y >= y0c && oy < height)
            {
                unsigned accu_a = 0, accu_b = 0, accu_c = 0;
                for (int yz = 0; yz < sh && (a.full_groups || oy + yz < height); yz++)
                    for (int xz = 0; xz < sw && (a.full_groups || ox + xz < width); xz++)
                    {
                        const unsigned coeff = a.c0[xz] * a.c1[yz];
                        unsigned ru = u, rv = v;
                        if (ox + xz >= 0 && oy + yz >= 0 && ox + xz < width && oy + yz < height)
                        {
                            const int oxz = ox + xz, oyz = oy + yz;
                            const unsigned alpha = (unsigned)oA[oyz * o.stride[3] + oxz] << shift;
                            ru = (ru * (maxv - alpha) + ((unsigned)oU[oyz * o.stride[1] + oxz] << oshift) * alpha + half) / maxv;
                            rv = (rv * (maxv - alpha) + ((unsigned)oV[oyz * o.stride[2] + oxz] << oshift) * alpha + half) / maxv;
                        }
                        accu_a += coeff * ru;
                        accu_b += coeff * rv;
                        accu_c += coeff;
                    }
                u = (accu_a + (accu_c >> 1)) / accu_c;
                v = (accu_b + (accu_c >> 1)) / accu_c;
            }
        }
        else
        {
            // blend.c:434-456: overlay samples [x0, ww) x [y0, hh) land at left + xx, top + yy
            const int x0 = max(0, -o.x), y0 = max(0, -o.y);
            const int ww = (o.w - x0 > a.W - o.x) ? a.W - o.x + x0 : o.w;
            const int hh = (o.h - y0 > a.H - o.y) ? a.H - o.y + y0 : o.h;
            for (int j = 0; j < sh; j++)
                for (int i = 0; i < sw; i++)
                {
                    const int xx = X + i - o.x, yy = Y + j - o.y;
                    if (X + i < a.W && Y + j < a.H && xx >= x0 && xx < ww && yy >= y0 && yy < hh)
                    {
                        const unsigned alpha = (unsigned)oA[yy * o.stride[3] + xx] << shift;
                        yv[j][i] = (yv[j][i] * (maxv - alpha) + ((unsigned)oY[yy * o.stride[0] + xx] << oshift) * alpha) / maxv;
                    }
                }
            // blend.c:486-508: chroma row yy lands at yy + (top >> hshift) (arithmetic shift), alpha from the top-left
            // luma sample of the group; an odd hh drops the last overlay row's chroma
            const int xx = gx - (o.x >> a.ws), yy = gy - (o.y >> a.hs);
            if (xx >= (x0 >> a.ws) && xx < (ww >> a.ws) && yy >= (y0 >> a.hs) && yy < (hh >> a.hs))
            {
                const unsigned alpha = (unsigned)oA[(yy << a.hs) * o.stride[3] + (xx << a.ws)] << shift;
                u = (u * (maxv - alpha) + ((unsigned)oU[yy * o.stride[1] + xx] << oshift) * alpha) / maxv;
                v = (v * (maxv - alpha) + ((unsigned)oV[yy * o.stride[2] + xx] << oshift) * alpha) / maxv;
            }
        }
    }

    for (int j = 0; j < sh; j++)
        for (int i = 0; i < sw; i++)
            if (X + i < a.W && Y + j < a.H) st<T>(a.plane[0], a.pitch[0], X + i, Y + j, yv[j][i]);
    if (NV)
    {
        st<T>(a.plane[1], a.pitch[1], 2 * gx, gy, u);
        st<T>(a.plane[1], a.pitch[1], 2 * gx + 1, gy, v);
    }
    else
    {
        st<T>(a.plane[1], a.pitch[1], gx, gy, u);
        st<T>(a.plane[2], a.pitch[2], gx, gy, v);
    }
}

struct Slot
{
    uint8_t *host = nullptr, *dev = nullptr;   // page-locked staging and its device copy: descriptors, then planes
    size_t cap = 0;
    std::vector<OvDesc> desc;                  // host copy of the descriptors (geometry for the launch box)
    cudaEvent_t done = nullptr;                // behind the upload and every blend that reads the slot
};

}  // namespace

struct hbcu_blend_s
{
    hbcu_blend_config_t cfg;
    int bps, cw, ch, subsample;
    int nplanes;                               // 3, or 2 for a semi-planar frame (plane 2 absent: 0 rows of 0 bytes)
    int sample_bytes[3];                       // bytes per sample position of each plane (a Cb/Cr pair counts once)
    int row_bytes[3], pitch[3];
    size_t plane_off[3], frame_bytes;
    uint8_t *staging = nullptr;                // host frames: the band the overlays touch is blended here
    cudaStream_t st = nullptr;
    cudaEvent_t ev_done = nullptr, ev_mark[2] = {nullptr, nullptr};
    Slot slot[kSlots];
    int cur = -1;                              // slot holding the current list
};

namespace {

bool frame_fits(const hbcu_blend_s *h, const hbcu_frame_t *f)
{
    if (f->device != h->cfg.device) return false;
    const int rows[3] = {h->cfg.height, h->ch, h->nplanes == 3 ? h->ch : 0};
    for (int p = 0; p < 3; p++)
        if (f->row_bytes[p] != h->row_bytes[p] || f->rows[p] != rows[p]) return false;
    return true;
}

// union, in chroma groups, of the rectangles the current overlays can touch inside the picture (a superset: the kernel
// applies the reference's exact bounds per sample); false when it is empty
bool launch_box(const hbcu_blend_s *h, int &gx0, int &gx1, int &gy0, int &gy1)
{
    const int W = h->cfg.width, H = h->cfg.height, ws = h->cfg.chroma_shift_w, hs = h->cfg.chroma_shift_h;
    gx0 = gy0 = INT32_MAX;
    gx1 = gy1 = 0;
    for (const OvDesc &o : h->slot[h->cur].desc)
    {
        const int xl = std::max(0, (o.x & ~1) - 2), xh = (int)std::min<int64_t>(W, (int64_t)o.x + o.w + 2);
        const int yl = std::max(0, (o.y & ~1) - 2), yh = (int)std::min<int64_t>(H, (int64_t)o.y + o.h + 2);
        if (xl >= xh || yl >= yh) continue;
        gx0 = std::min(gx0, xl >> ws);
        gy0 = std::min(gy0, yl >> hs);
        gx1 = std::max(gx1, std::min(h->cw, (xh + (1 << ws) - 1) >> ws));
        gy1 = std::max(gy1, std::min(h->ch, (yh + (1 << hs) - 1) >> hs));
    }
    return gx0 < gx1 && gy0 < gy1;
}

int launch(hbcu_blend_s *h, uint8_t *const planes[3], const int pitches[3], int gx0, int gx1, int gy0, int gy1)
{
    const Slot &s = h->slot[h->cur];
    BlendArgs a;
    for (int p = 0; p < 3; p++) { a.plane[p] = planes[p]; a.pitch[p] = pitches[p]; }
    a.W = h->cfg.width; a.H = h->cfg.height; a.CW = h->cw; a.CH = h->ch;
    a.ws = h->cfg.chroma_shift_w; a.hs = h->cfg.chroma_shift_h;
    a.shift = h->cfg.depth - 8;
    a.oshift = (h->cfg.interleaved_chroma && h->bps == 2) ? 8 : a.shift;
    a.full_groups = h->cfg.interleaved_chroma && h->bps == 1 && h->subsample;
    a.maxv = (256u << a.shift) - 1;
    for (int i = 0; i < 4; i++) { a.c0[i] = h->cfg.chroma_coeffs[0][i]; a.c1[i] = h->cfg.chroma_coeffs[1][i]; }
    a.gx0 = gx0; a.gy0 = gy0; a.gw = gx1 - gx0;
    a.ov = reinterpret_cast<const OvDesc *>(s.dev);
    a.blob = s.dev;
    a.n = (int)s.desc.size();
    const dim3 grid((a.gw + kThreads - 1) / kThreads, gy1 - gy0);
    if (h->cfg.interleaved_chroma)
    {
        if (h->bps == 1) { if (h->subsample) blend_kernel<uint8_t, true, true><<<grid, kThreads, 0, h->st>>>(a); else blend_kernel<uint8_t, false, true><<<grid, kThreads, 0, h->st>>>(a); }
        else             { if (h->subsample) blend_kernel<uint16_t, true, true><<<grid, kThreads, 0, h->st>>>(a); else blend_kernel<uint16_t, false, true><<<grid, kThreads, 0, h->st>>>(a); }
    }
    else
    {
        if (h->bps == 1) { if (h->subsample) blend_kernel<uint8_t, true, false><<<grid, kThreads, 0, h->st>>>(a); else blend_kernel<uint8_t, false, false><<<grid, kThreads, 0, h->st>>>(a); }
        else             { if (h->subsample) blend_kernel<uint16_t, true, false><<<grid, kThreads, 0, h->st>>>(a); else blend_kernel<uint16_t, false, false><<<grid, kThreads, 0, h->st>>>(a); }
    }
    HBCU_CHECK(cudaGetLastError());
    hbcu::count_launch();
    return 0;
}

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

}  // namespace

extern "C" {

uint64_t hbcu_blend_uploads(void) { return g_uploads.load(std::memory_order_relaxed); }

int hbcu_blend_create(hbcu_blend_t **out, const hbcu_blend_config_t *cfg)
{
    if (out == nullptr || cfg == nullptr) { set_error("blend_create: null argument"); return -1; }
    *out = nullptr;
    const int ws = cfg->chroma_shift_w, hs = cfg->chroma_shift_h, ows = cfg->overlay_shift_w, ohs = cfg->overlay_shift_h;
    const bool frame_ok = (ws == 1 && hs == 1) || (ws == 1 && hs == 0) || (ws == 0 && hs == 0);
    const bool overlay_ok = (ows == ws && ohs == hs) || (ows == 0 && ohs == 0);
    // the semi-planar formats of NVDEC are 4:2:0 only
    const bool interleave_ok = cfg->interleaved_chroma == 0 || (cfg->interleaved_chroma == 1 && ws == 1 && hs == 1);
    if (cfg->width < 1 || cfg->height < 1 || cfg->depth < 8 || cfg->depth > 16 || !frame_ok || !overlay_ok || !interleave_ok)
    {
        set_error("blend_create: unsupported geometry %dx%d depth %d, frame chroma shifts %d,%d, overlay %d,%d, interleaved chroma %d",
                  cfg->width, cfg->height, cfg->depth, ws, hs, ows, ohs, cfg->interleaved_chroma);
        return -1;
    }
    const int cw = -((-cfg->width) >> ws), ch = -((-cfg->height) >> hs);
    const bool subsample = ows != ws || ohs != hs;
    // the plain path takes its shifts from the plane sizes (blend.c:475-484); they differ from the format's only for a
    // one-sample-wide or -high frame, which is refused rather than given a third set of rules
    if (!subsample && (((cw < cfg->width) ? 1 : 0) != ws || ((ch < cfg->height) ? 1 : 0) != hs))
    {
        set_error("blend_create: a %dx%d frame is too small for the plain blend path", cfg->width, cfg->height);
        return -1;
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || cfg->device < 0 || cfg->device >= ndev)
    {
        cudaGetLastError();
        set_error("blend_create: CUDA device %d not available (%d devices); there is no CPU fallback", cfg->device, ndev);
        return -1;
    }
    HBCU_CHECK(cudaSetDevice(cfg->device));
    cudaDeviceProp prop;
    HBCU_CHECK(cudaGetDeviceProperties(&prop, cfg->device));
    if (prop.major != 9 || prop.minor != 0)
    {
        set_error("blend_create: device %d is sm_%d%d; this library is built for sm_90a only", cfg->device, prop.major, prop.minor);
        return -1;
    }
    hbcu_blend_s *h = new (std::nothrow) hbcu_blend_s();
    if (h == nullptr) { set_error("blend_create: out of memory"); return -1; }
    h->cfg = *cfg;
    h->bps = cfg->depth > 8 ? 2 : 1;
    h->cw = cw;
    h->ch = ch;
    h->subsample = subsample;
    h->nplanes = cfg->interleaved_chroma ? 2 : 3;
    size_t off = 0;
    for (int p = 0; p < 3; p++)
    {
        h->sample_bytes[p] = p >= h->nplanes ? 0 : (p == 1 && cfg->interleaved_chroma ? 2 : 1) * h->bps;
        h->row_bytes[p] = (p ? cw : cfg->width) * h->sample_bytes[p];
        h->pitch[p] = (h->row_bytes[p] + 63) / 64 * 64;
        h->plane_off[p] = off;
        off += (size_t)h->pitch[p] * (p ? ch : cfg->height);
    }
    h->frame_bytes = off;
#define CK(expr)                                                                  \
    do {                                                                          \
        cudaError_t _e = (expr);                                                  \
        if (_e != cudaSuccess) {                                                  \
            set_error("%s failed: %s", #expr, cudaGetErrorString(_e));            \
            hbcu_blend_destroy(h);                                                \
            return -1;                                                            \
        }                                                                         \
    } while (0)
    CK(cudaStreamCreateWithFlags(&h->st, cudaStreamNonBlocking));
    CK(cudaEventCreateWithFlags(&h->ev_done, cudaEventDisableTiming));
    CK(cudaEventCreate(&h->ev_mark[0]));
    CK(cudaEventCreate(&h->ev_mark[1]));
    for (int s = 0; s < kSlots; s++) CK(cudaEventCreateWithFlags(&h->slot[s].done, cudaEventDisableTiming));
    CK(cudaMalloc(&h->staging, h->frame_bytes));
#undef CK
    *out = h;
    return 0;
}

void hbcu_blend_destroy(hbcu_blend_t *h)
{
    if (h == nullptr) return;
    cudaSetDevice(h->cfg.device);
    if (h->st) cudaStreamSynchronize(h->st);
    for (Slot &s : h->slot)
    {
        if (s.host) cudaFreeHost(s.host);
        if (s.dev) cudaFree(s.dev);
        if (s.done) cudaEventDestroy(s.done);
    }
    if (h->staging) cudaFree(h->staging);
    if (h->ev_done) cudaEventDestroy(h->ev_done);
    if (h->ev_mark[0]) cudaEventDestroy(h->ev_mark[0]);
    if (h->ev_mark[1]) cudaEventDestroy(h->ev_mark[1]);
    if (h->st) cudaStreamDestroy(h->st);
    delete h;
}

int hbcu_blend_set_overlays(hbcu_blend_t *h, const hbcu_blend_overlay_t *list, int count, int changed)
{
    if (h == nullptr || count < 0 || (count > 0 && list == nullptr)) { set_error("blend_set_overlays: bad argument"); return -1; }
    const int ows = h->cfg.overlay_shift_w, ohs = h->cfg.overlay_shift_h;
    for (int i = 0; i < count; i++)
        if (list[i].width < 1 || list[i].height < 1 || !list[i].planes[0] || !list[i].planes[1] || !list[i].planes[2] || !list[i].planes[3])
        {
            set_error("blend_set_overlays: overlay %d is empty or lacks a plane", i);
            return -1;
        }
    if (!changed && h->cur >= 0 && (int)h->slot[h->cur].desc.size() == count)
    {
        bool same = true;
        for (int i = 0; i < count && same; i++)
        {
            const OvDesc &d = h->slot[h->cur].desc[i];
            same = d.x == list[i].x && d.y == list[i].y && d.w == list[i].width && d.h == list[i].height;
        }
        if (same) return 0;                  // the overlays on the device are still the right ones
    }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    const int s = (h->cur + 1) % kSlots;
    Slot &sl = h->slot[s];
    HBCU_CHECK(cudaEventSynchronize(sl.done));   // no queued blend reads this slot any more, its staging has been copied
    std::vector<OvDesc> desc(count);
    size_t bytes = align_up(sizeof(OvDesc) * (size_t)std::max(count, 1), 256);
    for (int i = 0; i < count; i++)
    {
        OvDesc &d = desc[i];
        d.x = list[i].x; d.y = list[i].y; d.w = list[i].width; d.h = list[i].height;
        for (int p = 0; p < 4; p++)
        {
            const int pw = (p == 1 || p == 2) ? -((-d.w) >> ows) : d.w;
            const int ph = (p == 1 || p == 2) ? -((-d.h) >> ohs) : d.h;
            d.off[p] = (uint32_t)bytes;
            d.stride[p] = pw;
            bytes = align_up(bytes + (size_t)pw * ph, 16);
        }
    }
    if (bytes > UINT32_MAX) { set_error("blend_set_overlays: overlays too large"); return -1; }
    if (bytes > sl.cap)
    {
        if (sl.host) cudaFreeHost(sl.host);
        if (sl.dev) cudaFree(sl.dev);
        sl.host = sl.dev = nullptr;
        sl.cap = 0;
        const size_t cap = align_up(bytes + bytes / 2, 1 << 16);
        HBCU_CHECK(cudaMallocHost(&sl.host, cap));
        HBCU_CHECK(cudaMalloc(&sl.dev, cap));
        sl.cap = cap;
    }
    memcpy(sl.host, desc.data(), sizeof(OvDesc) * count);
    for (int i = 0; i < count; i++)
        for (int p = 0; p < 4; p++)
        {
            const OvDesc &d = desc[i];
            const int ph = (p == 1 || p == 2) ? -((-d.h) >> ohs) : d.h;
            for (int y = 0; y < ph; y++)
                memcpy(sl.host + d.off[p] + (size_t)y * d.stride[p], list[i].planes[p] + (size_t)y * list[i].strides[p], d.stride[p]);
        }
    HBCU_CHECK(cudaMemcpyAsync(sl.dev, sl.host, bytes, cudaMemcpyHostToDevice, h->st));
    HBCU_CHECK(cudaEventRecord(sl.done, h->st));
    sl.desc.swap(desc);
    h->cur = s;
    g_uploads.fetch_add(1, std::memory_order_relaxed);
    return 0;
}

int hbcu_blend_frames(hbcu_blend_t *h, hbcu_frame_t *in_frame, const void *const in_planes[3], const int in_strides[3],
                      hbcu_frame_t *out_frame, void *const out_planes[3], const int out_strides[3])
{
    if (h == nullptr || h->cur < 0 || (in_frame == nullptr) != (out_frame == nullptr) ||
        (in_frame == nullptr && (in_planes == nullptr || in_strides == nullptr || out_planes == nullptr || out_strides == nullptr)) ||
        (in_frame && (!frame_fits(h, in_frame) || !frame_fits(h, out_frame))))
    {
        set_error("blend_frames: bad argument or frame geometry (no overlays set, or a host and a device side)");
        return -1;
    }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    int gx0, gx1, gy0, gy1;
    const bool any = launch_box(h, gx0, gx1, gy0, gy1);
    const int ws = h->cfg.chroma_shift_w, hs = h->cfg.chroma_shift_h;
    if (in_frame)
    {
        if (hbcu::frame_begin_read(in_frame, h->st) != 0) return -1;
        if (hbcu::frame_begin_write(out_frame, h->st) != 0) return -1;
        for (int p = 0; p < h->nplanes; p++)
            HBCU_CHECK(cudaMemcpy2DAsync(out_frame->plane[p], out_frame->stride[p], in_frame->plane[p], in_frame->stride[p],
                                         h->row_bytes[p], in_frame->rows[p], cudaMemcpyDeviceToDevice, h->st));
        if (hbcu::frame_end_read(in_frame, h->st) != 0) return -1;
        if (any && launch(h, out_frame->plane, out_frame->stride, gx0, gx1, gy0, gy1) != 0) return -1;
        if (hbcu::frame_end_write(out_frame, h->st) != 0) return -1;
    }
    else if (any)
    {
        // the band of rows and columns the overlays touch, per plane: luma in samples, chroma in groups
        const int x0[3] = {gx0 << ws, gx0, gx0}, x1[3] = {std::min(h->cfg.width, gx1 << ws), gx1, gx1};
        const int y0[3] = {gy0 << hs, gy0, gy0}, y1[3] = {std::min(h->cfg.height, gy1 << hs), gy1, gy1};
        uint8_t *dplanes[3] = {nullptr, nullptr, nullptr};
        for (int p = 0; p < h->nplanes; p++)
        {
            const int sb = h->sample_bytes[p];
            dplanes[p] = h->staging + h->plane_off[p];
            const size_t dst_off = (size_t)y0[p] * h->pitch[p] + (size_t)x0[p] * sb;
            const size_t src_off = (size_t)y0[p] * in_strides[p] + (size_t)x0[p] * sb;
            HBCU_CHECK(cudaMemcpy2DAsync(dplanes[p] + dst_off, h->pitch[p], (const uint8_t *)in_planes[p] + src_off, in_strides[p],
                                         (size_t)(x1[p] - x0[p]) * sb, y1[p] - y0[p], cudaMemcpyHostToDevice, h->st));
        }
        if (launch(h, dplanes, h->pitch, gx0, gx1, gy0, gy1) != 0) return -1;
        for (int p = 0; p < h->nplanes; p++)
        {
            const int sb = h->sample_bytes[p];
            const size_t dev_off = (size_t)y0[p] * h->pitch[p] + (size_t)x0[p] * sb;
            const size_t host_off = (size_t)y0[p] * out_strides[p] + (size_t)x0[p] * sb;
            HBCU_CHECK(cudaMemcpy2DAsync((uint8_t *)out_planes[p] + host_off, out_strides[p], dplanes[p] + dev_off, h->pitch[p],
                                         (size_t)(x1[p] - x0[p]) * sb, y1[p] - y0[p], cudaMemcpyDeviceToHost, h->st));
        }
    }
    HBCU_CHECK(cudaEventRecord(h->slot[h->cur].done, h->st));
    HBCU_CHECK(cudaEventRecord(h->ev_done, h->st));
    return 0;
}

int hbcu_blend_wait(hbcu_blend_t *h)
{
    if (h == nullptr) { set_error("blend_wait: null handle"); return -1; }
    HBCU_CHECK(cudaEventSynchronize(h->ev_done));
    return 0;
}

int hbcu_blend_sync(hbcu_blend_t *h)
{
    if (h == nullptr) { set_error("blend_sync: null handle"); return -1; }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    HBCU_CHECK(cudaStreamSynchronize(h->st));
    return 0;
}

int hbcu_blend_mark(hbcu_blend_t *h, int which)
{
    if (h == nullptr || which < 0 || which > 1) { set_error("blend_mark: bad argument"); return -1; }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    HBCU_CHECK(cudaEventRecord(h->ev_mark[which], h->st));
    return 0;
}

int hbcu_blend_elapsed_ms(hbcu_blend_t *h, float *ms)
{
    if (h == nullptr || ms == nullptr) { set_error("blend_elapsed_ms: bad argument"); return -1; }
    HBCU_CHECK(cudaEventSynchronize(h->ev_mark[1]));
    HBCU_CHECK(cudaEventElapsedTime(ms, h->ev_mark[0], h->ev_mark[1]));
    return 0;
}

}  // extern "C"
