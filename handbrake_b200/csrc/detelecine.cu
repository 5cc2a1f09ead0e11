// detelecine.cu -- the data-parallel half of pullup (inverse telecine) for sm_90a behind include/hbcu.h (SURVEY.md 8 f4).
//
// Replaces, of the reference's libhb/detelecine.c:
//   pullup_diff_y / pullup_licomb_y / pullup_var_y (:159-207) driven by pullup_compute_metric (:230-265)
//   the max-reductions of pullup_compute_breaks (:369-374) and pullup_compute_affinity (:405-418)
//   pullup_copy_field (:298-317) and the plane copies in and out of the pullup buffers (:1159-1164, :1250-1252)
// The field-queue state machine that decides what a frame is made of works on a handful of integers per field; it is
// host code (handbrake_b200/libhb/detelecine_cuda.c) driving the calls below.  Pictures and metric arrays stay in HBM:
// per input picture the device reads the metric plane ~3 times (8 x 4 sample blocks, one thread per block, 8- or 16-byte
// loads) and writes 3 ints per block; what returns to the host is two ints per reduction.
//
// Geometry quirks kept (they cancel out in the reference, so they are restated rather than "fixed"):
//   * c->bpp is BITS per sample (8 / 16) but steps bytes along a row: 8 bytes = 8 samples at 8 bit, 16 bytes = 8
//     samples at 16 bit -- i.e. blocks are always 8 samples wide and junk_left/right count blocks (:237, :617);
//   * the field stride handed to the metric functions is stride << 1 bytes at 8 bit and stride bytes, used as uint16
//     elements, above: two picture lines either way (:239, :1049).
#include "hbcu_common.h"
#include "hbcu_frames.h"
#include "../../include/hbcu.h"

#include <cstdlib>
#include <cstring>
#include <new>

namespace {

using hbcu::set_error;

template <typename PIX> struct Row8;
template <> struct Row8<uint8_t>
{
    static __device__ __forceinline__ void load(const uint8_t *p, int v[8])
    {
        const uint2 q = *reinterpret_cast<const uint2 *>(p);
#pragma unroll
        for (int i = 0; i < 4; i++) { v[i] = (q.x >> (8 * i)) & 255; v[4 + i] = (q.y >> (8 * i)) & 255; }
    }
};
template <> struct Row8<uint16_t>
{
    static __device__ __forceinline__ void load(const uint16_t *p, int v[8])
    {
        const uint4 q = *reinterpret_cast<const uint4 *>(p);
        const unsigned w[4] = { q.x, q.y, q.z, q.w };
#pragma unroll
        for (int i = 0; i < 4; i++) { v[2 * i] = w[i] & 0xffff; v[2 * i + 1] = w[i] >> 16; }
    }
};

__device__ __forceinline__ int iabs(int a) { return a < 0 ? -a : a; }

// One thread = one 8-sample x 4-field-line block of the metric plane.  All pointers address sample (0,0) of block (0,0)
// of the field in question (field offset and junk offset included); `pitch` is the PICTURE pitch in samples.
// diff_mode: 0 leave diffs alone, 1 zero them, 2 compute against dprev.  ctop == nullptr leaves comb alone.
template <typename PIX>
__global__ void __launch_bounds__(256) k_metrics(const PIX *__restrict__ cur, const PIX *__restrict__ dprev, int diff_mode,
                                                 const PIX *__restrict__ ctop, const PIX *__restrict__ cbot,
                                                 int *__restrict__ diffs, int *__restrict__ comb, int *__restrict__ var,
                                                 int pitch, int mw, int mh)
{
    const int bx = blockIdx.x * blockDim.x + threadIdx.x, by = blockIdx.y * blockDim.y + threadIdx.y;
    if (bx >= mw || by >= mh) return;
    const size_t off = (size_t)by * 8 * pitch + (size_t)bx * 8;
    const int s = 2 * pitch;                                   // field line stride
    const int o = by * mw + bx;
    int a[5][8];
    // var_y (:194-207): three line differences of the field itself, times 4
#pragma unroll
    for (int r = 0; r < 4; r++) Row8<PIX>::load(cur + off + (size_t)r * s, a[r]);
    {
        int v = 0;
#pragma unroll
        for (int r = 0; r < 3; r++)
#pragma unroll
            for (int j = 0; j < 8; j++) v += iabs(a[r][j] - a[r + 1][j]);
        var[o] = 4 * v;
    }
    // diff_y (:159-174): 4 lines x 8 samples of absolute differences against the same-parity field two fields back
    if (diff_mode == 1) diffs[o] = 0;
    else if (diff_mode == 2)
    {
        int d = 0, b[8];
#pragma unroll
        for (int r = 0; r < 4; r++)
        {
            Row8<PIX>::load(dprev + off + (size_t)r * s, b);
#pragma unroll
            for (int j = 0; j < 8; j++) d += iabs(a[r][j] - b[j]);
        }
        diffs[o] = d;
    }
    // licomb_y (:176-192): a = top field, b = bottom field; each line against the average of its two neighbours in the
    // woven picture: |2a - b(line above) - b| + |2b - a - a(line below)|
    if (ctop != nullptr)
    {
        int b[5][8];
#pragma unroll
        for (int r = 0; r < 5; r++)
        {
            Row8<PIX>::load(ctop + off + (size_t)r * s, a[r]);                         // a lines 0..4
            Row8<PIX>::load(cbot + off + (ptrdiff_t)(r - 1) * s, b[r]);                // b lines -1..3
        }
        int c = 0;
#pragma unroll
        for (int r = 0; r < 4; r++)
#pragma unroll
            for (int j = 0; j < 8; j++)
                c += iabs((a[r][j] << 1) - b[r][j] - b[r + 1][j]) + iabs((b[r + 1][j] << 1) - a[r][j] - a[r + 1][j]);
        comb[o] = c;
    }
}

__device__ __forceinline__ void reduce_pair(int max_l, int max_r, int *__restrict__ result)
{
#pragma unroll
    for (int d = 16; d > 0; d >>= 1)
    {
        max_l = max(max_l, __shfl_xor_sync(0xffffffffu, max_l, d));
        max_r = max(max_r, __shfl_xor_sync(0xffffffffu, max_r, d));
    }
    if ((threadIdx.x & 31) == 0)
    {
        if (max_l > 0) atomicMax(result + 0, max_l);
        if (max_r > 0) atomicMax(result + 1, max_r);
    }
}

// pullup_compute_breaks (:369-374); result[] starts at {0, 0}
__global__ void __launch_bounds__(256) k_breaks(const int *__restrict__ d2, const int *__restrict__ d3, int n, int *__restrict__ result)
{
    int max_l = 0, max_r = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    {
        const int l = d2[i] - d3[i];
        max_l = max(max_l, l);
        max_r = max(max_r, -l);
    }
    reduce_pair(max_l, max_r, result);
}

// pullup_compute_affinity (:405-418)
__global__ void __launch_bounds__(256) k_affinity(const int *__restrict__ var_prev, const int *__restrict__ var_cur, const int *__restrict__ var_next,
                                                  const int *__restrict__ comb_cur, const int *__restrict__ comb_next, int n, int *__restrict__ result)
{
    int max_l = 0, max_r = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    {
        const int lv = var_prev[i], rv = var_next[i], v = var_cur[i];
        const int lc = max(comb_cur[i] - (v + lv) + iabs(v - lv), 0);
        const int rc = max(comb_next[i] - (v + rv) + iabs(v - rv), 0);
        const int l = lc - rc;
        max_l = max(max_l, l);
        max_r = max(max_r, -l);
    }
    reduce_pair(max_l, max_r, result);
}

struct Plane { int w, h, pitch_bytes; size_t off; };

}  // namespace

struct hbcu_detelecine_s
{
    hbcu_detelecine_config_t cfg;
    int bps;
    Plane pl[3];
    size_t picture_bytes;
    int metric_w, metric_h, metric_len;
    size_t metric_off_bytes;            // junk offset inside the metric plane (:617)
    uint8_t *d_pictures;
    uint8_t *d_staging;                 // download_begin: the woven picture is parked here, so the picture itself is free at once
    int *d_metrics;                     // [fields][3][metric_len]: diffs, comb, var
    int *d_results, *h_results;
    cudaStream_t s;
    cudaStream_t s_d2h;                 // hbcu_detelecine_download_begin: the copy out overlaps the next picture's upload and metrics
    cudaEvent_t ev_woven, ev_d2h;
    cudaEvent_t ev_mark[2];
};

namespace {

inline uint8_t *picture_plane(const hbcu_detelecine_s *h, int picture, int p)
{
    return h->d_pictures + (size_t)picture * h->picture_bytes + h->pl[p].off;
}
inline int *metric_array(const hbcu_detelecine_s *h, int field, int which)
{
    return h->d_metrics + ((size_t)field * 3 + which) * h->metric_len;
}
inline bool bad_picture(const hbcu_detelecine_s *h, int i) { return i < 0 || i >= h->cfg.pictures; }
inline bool bad_field(const hbcu_detelecine_s *h, int i) { return i < 0 || i >= h->cfg.fields; }

}  // namespace

extern "C" {

int hbcu_detelecine_create(hbcu_detelecine_t **out, const hbcu_detelecine_config_t *cfg)
{
    if (out == nullptr || cfg == nullptr) { set_error("detelecine_create: null argument"); return -1; }
    *out = nullptr;
    if (cfg->width < 1 || cfg->height < 1 || cfg->depth < 8 || cfg->depth > 16 || cfg->pictures < 2 || cfg->fields < 4 || cfg->results < 1 ||
        cfg->metric_plane < 0 || cfg->metric_plane > 2)
    {
        set_error("detelecine_create: unsupported configuration %dx%d depth %d (%d pictures, %d fields)", cfg->width, cfg->height, cfg->depth,
                  cfg->pictures, cfg->fields);
        return -1;
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || cfg->device < 0 || cfg->device >= ndev)
    {
        cudaGetLastError();
        set_error("detelecine_create: CUDA device %d not available (%d devices); there is no CPU fallback", cfg->device, ndev);
        return -1;
    }
    HBCU_CHECK(cudaSetDevice(cfg->device));
    cudaDeviceProp prop;
    HBCU_CHECK(cudaGetDeviceProperties(&prop, cfg->device));
    if (prop.major != 9 || prop.minor != 0)
    {
        set_error("detelecine_create: device %d is sm_%d%d; this library is built for sm_90a only", cfg->device, prop.major, prop.minor);
        return -1;
    }
    hbcu_detelecine_s *h = new (std::nothrow) hbcu_detelecine_s();
    if (h == nullptr) { set_error("detelecine_create: out of memory"); return -1; }
    h->cfg = *cfg;
    h->bps = cfg->depth > 8 ? 2 : 1;
    h->d_pictures = nullptr;
    h->d_staging = nullptr;
    h->s_d2h = nullptr;
    h->ev_woven = h->ev_d2h = nullptr;
    h->d_metrics = h->d_results = h->h_results = nullptr;
    h->s = nullptr;
    h->ev_mark[0] = h->ev_mark[1] = nullptr;
    size_t off = 0;
    for (int p = 0; p < 3; p++)
    {
        Plane &g = h->pl[p];
        g.w = p == 0 ? cfg->width : -((-cfg->width) >> cfg->chroma_shift_w);
        g.h = p == 0 ? cfg->height : -((-cfg->height) >> cfg->chroma_shift_h);
        g.pitch_bytes = (g.w * h->bps + 63) / 64 * 64;                 // hb_image_stride
        g.off = off;
        off += (size_t)g.pitch_bytes * g.h;
    }
    h->picture_bytes = off;
    const Plane &m = h->pl[cfg->metric_plane];
    h->metric_w = (m.w - ((cfg->junk_left + cfg->junk_right) << 3)) >> 3;                 // :615
    h->metric_h = (m.h - ((cfg->junk_top + cfg->junk_bottom) << 1)) >> 3;                 // :616
    if (h->metric_w < 1 || h->metric_h < 1 || cfg->junk_top < 1 || cfg->junk_bottom < 1 || cfg->junk_left < 0 || cfg->junk_right < 0)
    {
        // the reference would walk zero or a negative number of blocks (or read above the plane with junk_top 0)
        set_error("detelecine_create: %dx%d leaves no metric blocks inside the junk margins", m.w, m.h);
        delete h;
        return -1;
    }
    h->metric_len = h->metric_w * h->metric_h;
    h->metric_off_bytes = (size_t)cfg->junk_left * 8 * h->bps + (size_t)(cfg->junk_top << 1) * m.pitch_bytes;
#define CK(expr)                                                                  \
    do {                                                                          \
        cudaError_t _e = (expr);                                                  \
        if (_e != cudaSuccess) {                                                  \
            set_error("%s failed: %s", #expr, cudaGetErrorString(_e));            \
            hbcu_detelecine_destroy(h);                                           \
            return -1;                                                            \
        }                                                                         \
    } while (0)
    CK(cudaStreamCreateWithFlags(&h->s, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&h->s_d2h, cudaStreamNonBlocking));
    CK(cudaEventCreateWithFlags(&h->ev_woven, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&h->ev_d2h, cudaEventDisableTiming));
    CK(cudaEventCreate(&h->ev_mark[0]));
    CK(cudaEventCreate(&h->ev_mark[1]));
    CK(cudaMalloc(&h->d_pictures, h->picture_bytes * cfg->pictures));
    CK(cudaMemset(h->d_pictures, 0, h->picture_bytes * cfg->pictures));
    CK(cudaMalloc(&h->d_staging, h->picture_bytes));
    CK(cudaMemset(h->d_staging, 0, h->picture_bytes));
    CK(cudaMalloc(&h->d_metrics, sizeof(int) * 3 * h->metric_len * cfg->fields));
    CK(cudaMemset(h->d_metrics, 0, sizeof(int) * 3 * h->metric_len * cfg->fields));        // calloc, :224-228
    CK(cudaMalloc(&h->d_results, sizeof(int) * 2 * cfg->results));
    CK(cudaMemset(h->d_results, 0, sizeof(int) * 2 * cfg->results));
    CK(cudaHostAlloc(&h->h_results, sizeof(int) * 2 * cfg->results, cudaHostAllocDefault));
    CK(cudaDeviceSynchronize());          // the memsets ran on the legacy default stream; h->s does not wait for it
#undef CK
    *out = h;
    return 0;
}

void hbcu_detelecine_destroy(hbcu_detelecine_t *h)
{
    if (h == nullptr) return;
    cudaSetDevice(h->cfg.device);
    if (h->s) cudaStreamSynchronize(h->s);
    if (h->s_d2h) cudaStreamSynchronize(h->s_d2h);
    if (h->d_pictures) cudaFree(h->d_pictures);
    if (h->d_staging) cudaFree(h->d_staging);
    if (h->d_metrics) cudaFree(h->d_metrics);
    if (h->d_results) cudaFree(h->d_results);
    if (h->h_results) cudaFreeHost(h->h_results);
    if (h->ev_mark[0]) cudaEventDestroy(h->ev_mark[0]);
    if (h->ev_mark[1]) cudaEventDestroy(h->ev_mark[1]);
    if (h->ev_woven) cudaEventDestroy(h->ev_woven);
    if (h->ev_d2h) cudaEventDestroy(h->ev_d2h);
    if (h->s_d2h) cudaStreamDestroy(h->s_d2h);
    if (h->s) cudaStreamDestroy(h->s);
    delete h;
}

int hbcu_detelecine_upload(hbcu_detelecine_t *h, int picture, const void *const planes[3], const int strides[3])
{
    if (h == nullptr || planes == nullptr || strides == nullptr || bad_picture(h, picture)) { set_error("detelecine_upload: bad argument"); return -1; }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    bool contiguous = true;
    for (int p = 0; p < 3; p++)
    {
        if (planes[p] == nullptr || strides[p] <= 0) { set_error("detelecine_upload: plane %d missing", p); return -1; }
        if (strides[p] != h->pl[p].pitch_bytes || (const uint8_t *)planes[p] != (const uint8_t *)planes[0] + h->pl[p].off) contiguous = false;
    }
    if (contiguous)
        HBCU_CHECK(cudaMemcpyAsync(picture_plane(h, picture, 0), planes[0], h->picture_bytes, cudaMemcpyHostToDevice, h->s));
    else
        for (int p = 0; p < 3; p++)
        {
            // hb_image_copy_plane: the shorter of the two strides per line
            const int row = strides[p] < h->pl[p].pitch_bytes ? strides[p] : h->pl[p].pitch_bytes;
            HBCU_CHECK(cudaMemcpy2DAsync(picture_plane(h, picture, p), h->pl[p].pitch_bytes, planes[p], strides[p], row, h->pl[p].h,
                                         cudaMemcpyHostToDevice, h->s));
        }
    return 0;
}

int hbcu_detelecine_metrics(hbcu_detelecine_t *h, int field, int picture, int parity, int diff_picture, int comb_top_picture, int comb_bottom_picture)
{
    if (h == nullptr || bad_field(h, field) || bad_picture(h, picture) || (parity != 0 && parity != 1) || diff_picture >= h->cfg.pictures ||
        comb_top_picture >= h->cfg.pictures || comb_bottom_picture >= h->cfg.pictures || (comb_top_picture < 0) != (comb_bottom_picture < 0))
    {
        set_error("detelecine_metrics: bad argument");
        return -1;
    }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    const int mp = h->cfg.metric_plane;
    const int pitch_bytes = h->pl[mp].pitch_bytes;
    auto field_base = [&](int pic, int par) { return picture_plane(h, pic, mp) + (size_t)par * pitch_bytes + h->metric_off_bytes; };
    const uint8_t *cur = field_base(picture, parity);
    const int diff_mode = diff_picture < 0 ? 0 : diff_picture == picture ? 1 : 2;
    const uint8_t *dprev = diff_mode == 2 ? field_base(diff_picture, parity) : nullptr;
    const uint8_t *ctop = comb_top_picture >= 0 ? field_base(comb_top_picture, 0) : nullptr;
    const uint8_t *cbot = comb_bottom_picture >= 0 ? field_base(comb_bottom_picture, 1) : nullptr;
    const dim3 blk(64, 4), grid((h->metric_w + 63) / 64, (h->metric_h + 3) / 4);
    int *diffs = metric_array(h, field, 0), *comb = metric_array(h, field, 1), *var = metric_array(h, field, 2);
    if (h->bps == 1)
        k_metrics<uint8_t><<<grid, blk, 0, h->s>>>(cur, dprev, diff_mode, ctop, cbot, diffs, comb, var, pitch_bytes, h->metric_w, h->metric_h);
    else
        k_metrics<uint16_t><<<grid, blk, 0, h->s>>>((const uint16_t *)cur, (const uint16_t *)dprev, diff_mode, (const uint16_t *)ctop,
                                                     (const uint16_t *)cbot, diffs, comb, var, pitch_bytes / 2, h->metric_w, h->metric_h);
    hbcu::count_launch();
    HBCU_CHECK(cudaGetLastError());
    return 0;
}

static int reduction_grid(const hbcu_detelecine_s *h)
{
    const int blocks = (h->metric_len + 255) / 256;
    return blocks < 264 ? blocks : 264;                       // 2 CTAs per SM of an H100 (132 SMs), grid-stride beyond that
}

int hbcu_detelecine_breaks(hbcu_detelecine_t *h, int field2, int field3, int slot)
{
    if (h == nullptr || bad_field(h, field2) || bad_field(h, field3) || slot < 0 || slot >= h->cfg.results) { set_error("detelecine_breaks: bad argument"); return -1; }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    HBCU_CHECK(cudaMemsetAsync(h->d_results + 2 * slot, 0, 2 * sizeof(int), h->s));
    k_breaks<<<reduction_grid(h), 256, 0, h->s>>>(metric_array(h, field2, 0), metric_array(h, field3, 0), h->metric_len, h->d_results + 2 * slot);
    hbcu::count_launch();
    HBCU_CHECK(cudaGetLastError());
    return 0;
}

int hbcu_detelecine_affinity(hbcu_detelecine_t *h, int field_prev, int field, int field_next, int slot)
{
    if (h == nullptr || bad_field(h, field_prev) || bad_field(h, field) || bad_field(h, field_next) || slot < 0 || slot >= h->cfg.results)
    {
        set_error("detelecine_affinity: bad argument");
        return -1;
    }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    HBCU_CHECK(cudaMemsetAsync(h->d_results + 2 * slot, 0, 2 * sizeof(int), h->s));
    k_affinity<<<reduction_grid(h), 256, 0, h->s>>>(metric_array(h, field_prev, 2), metric_array(h, field, 2), metric_array(h, field_next, 2),
                                                     metric_array(h, field, 1), metric_array(h, field_next, 1), h->metric_len, h->d_results + 2 * slot);
    hbcu::count_launch();
    HBCU_CHECK(cudaGetLastError());
    return 0;
}

int hbcu_detelecine_fetch(hbcu_detelecine_t *h, int *dst, int nslots)
{
    if (h == nullptr || nslots < 0 || nslots > h->cfg.results || (nslots > 0 && dst == nullptr)) { set_error("detelecine_fetch: bad argument"); return -1; }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    if (nslots > 0) HBCU_CHECK(cudaMemcpyAsync(h->h_results, h->d_results, sizeof(int) * 2 * nslots, cudaMemcpyDeviceToHost, h->s));
    HBCU_CHECK(cudaStreamSynchronize(h->s));
    if (nslots > 0) memcpy(dst, h->h_results, sizeof(int) * 2 * nslots);
    return 0;
}

int hbcu_detelecine_copy_field(hbcu_detelecine_t *h, int dst_picture, int src_picture, int parity)
{
    if (h == nullptr || bad_picture(h, dst_picture) || bad_picture(h, src_picture) || (parity != 0 && parity != 1)) { set_error("detelecine_copy_field: bad argument"); return -1; }
    if (dst_picture == src_picture) return 0;
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    for (int p = 0; p < 3; p++)
    {
        const int pitch = h->pl[p].pitch_bytes;
        HBCU_CHECK(cudaMemcpy2DAsync(picture_plane(h, dst_picture, p) + (size_t)parity * pitch, 2 * (size_t)pitch,
                                     picture_plane(h, src_picture, p) + (size_t)parity * pitch, 2 * (size_t)pitch,
                                     pitch, h->pl[p].h >> 1, cudaMemcpyDeviceToDevice, h->s));       // c->h[i] >> 1 lines, :307
    }
    return 0;
}

static int download_on(hbcu_detelecine_t *h, int picture, void *const planes[3], const int strides[3], bool staged, const char *who)
{
    if (h == nullptr || planes == nullptr || strides == nullptr || bad_picture(h, picture)) { set_error("%s: bad argument", who); return -1; }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    bool contiguous = true;
    for (int p = 0; p < 3; p++)
    {
        if (planes[p] == nullptr || strides[p] <= 0) { set_error("%s: plane %d missing", who, p); return -1; }
        if (strides[p] != h->pl[p].pitch_bytes || (uint8_t *)planes[p] != (uint8_t *)planes[0] + h->pl[p].off) contiguous = false;
    }
    cudaStream_t st = h->s;
    const uint8_t *base = picture_plane(h, picture, 0);
    if (staged)
    {
        // park the picture (the previous copy out of the staging buffer must be through), then copy out on the other stream
        HBCU_CHECK(cudaStreamWaitEvent(h->s, h->ev_d2h, 0));
        HBCU_CHECK(cudaMemcpyAsync(h->d_staging, base, h->picture_bytes, cudaMemcpyDeviceToDevice, h->s));
        HBCU_CHECK(cudaEventRecord(h->ev_woven, h->s));
        HBCU_CHECK(cudaStreamWaitEvent(h->s_d2h, h->ev_woven, 0));
        st = h->s_d2h;
        base = h->d_staging;
    }
    if (contiguous)
        HBCU_CHECK(cudaMemcpyAsync(planes[0], base, h->picture_bytes, cudaMemcpyDeviceToHost, st));
    else
        for (int p = 0; p < 3; p++)
        {
            const int row = strides[p] < h->pl[p].pitch_bytes ? strides[p] : h->pl[p].pitch_bytes;
            HBCU_CHECK(cudaMemcpy2DAsync(planes[p], strides[p], base + h->pl[p].off, h->pl[p].pitch_bytes, row, h->pl[p].h,
                                         cudaMemcpyDeviceToHost, st));
        }
    return 0;
}

int hbcu_detelecine_download(hbcu_detelecine_t *h, int picture, void *const planes[3], const int strides[3])
{
    if (download_on(h, picture, planes, strides, false, "detelecine_download") != 0) return -1;
    HBCU_CHECK(cudaStreamSynchronize(h->s));
    return 0;
}

int hbcu_detelecine_download_begin(hbcu_detelecine_t *h, int picture, void *const planes[3], const int strides[3])
{
    if (download_on(h, picture, planes, strides, true, "detelecine_download_begin") != 0) return -1;
    HBCU_CHECK(cudaEventRecord(h->ev_d2h, h->s_d2h));
    return 0;
}

int hbcu_detelecine_download_end(hbcu_detelecine_t *h)
{
    if (h == nullptr) { set_error("detelecine_download_end: null handle"); return -1; }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    HBCU_CHECK(cudaEventSynchronize(h->ev_d2h));
    return 0;
}

static bool frame_matches(const hbcu_detelecine_t *h, const hbcu_frame_t *f)
{
    if (f == nullptr || f->device != h->cfg.device) return false;
    for (int p = 0; p < 3; p++)
        if (f->rows[p] != h->pl[p].h || f->row_bytes[p] > h->pl[p].pitch_bytes) return false;
    return true;
}

int hbcu_detelecine_upload_frame(hbcu_detelecine_t *h, int picture, hbcu_frame_t *in)
{
    if (h == nullptr || bad_picture(h, picture) || !frame_matches(h, in)) { set_error("detelecine_upload_frame: bad argument or frame geometry"); return -1; }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    if (hbcu::frame_begin_read(in, h->s) != 0) return -1;
    for (int p = 0; p < 3; p++)
    {
        // hb_image_copy_plane: the shorter of the two strides per line
        const int row = in->stride[p] < h->pl[p].pitch_bytes ? in->stride[p] : h->pl[p].pitch_bytes;
        HBCU_CHECK(cudaMemcpy2DAsync(picture_plane(h, picture, p), h->pl[p].pitch_bytes, in->plane[p], in->stride[p], row, h->pl[p].h,
                                     cudaMemcpyDeviceToDevice, h->s));
    }
    return hbcu::frame_end_read(in, h->s);
}

int hbcu_detelecine_download_frame(hbcu_detelecine_t *h, int picture, hbcu_frame_t *out)
{
    if (h == nullptr || bad_picture(h, picture) || !frame_matches(h, out)) { set_error("detelecine_download_frame: bad argument or frame geometry"); return -1; }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    if (hbcu::frame_begin_write(out, h->s) != 0) return -1;
    for (int p = 0; p < 3; p++)
    {
        const int row = out->stride[p] < h->pl[p].pitch_bytes ? out->stride[p] : h->pl[p].pitch_bytes;
        HBCU_CHECK(cudaMemcpy2DAsync(out->plane[p], out->stride[p], picture_plane(h, picture, p), h->pl[p].pitch_bytes, row, h->pl[p].h,
                                     cudaMemcpyDeviceToDevice, h->s));
    }
    return hbcu::frame_end_write(out, h->s);      // no host wait: the consumer orders itself behind the frame's `ready`
}

int hbcu_detelecine_mark(hbcu_detelecine_t *h, int which)
{
    if (h == nullptr || which < 0 || which > 1) { set_error("detelecine_mark: bad argument"); return -1; }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    HBCU_CHECK(cudaEventRecord(h->ev_mark[which], h->s));
    return 0;
}

int hbcu_detelecine_elapsed_ms(hbcu_detelecine_t *h, float *ms)
{
    if (h == nullptr || ms == nullptr) { set_error("detelecine_elapsed_ms: bad argument"); return -1; }
    HBCU_CHECK(cudaEventSynchronize(h->ev_mark[1]));
    HBCU_CHECK(cudaEventElapsedTime(ms, h->ev_mark[0], h->ev_mark[1]));
    return 0;
}

}  // extern "C"
