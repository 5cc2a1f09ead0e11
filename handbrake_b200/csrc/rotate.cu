// rotate.cu -- rotations by 90, 180 and 270 degrees and mirrors for sm_90a behind the C-ABI of include/hbcu.h
// (hbcu_rotate_*).
//
// What the reference's rotate filter (rotate.c) asks FFmpeg's avfilter graph for: hflip, vflip, both, or a transpose
// (clock, cclock, clock_flip, cclock_flip).  Each is a pure permutation of every plane's elements within the plane's own
// size, where an element is a sample of a planar format or the Cb/Cr pair of a semi-planar chroma plane, which moves as
// one unit.  For an input plane of pw x ph elements, output element (x, y) is
//   flips       in[fy ? ph-1-y : y][fx ? pw-1-x : x]                      (output pw x ph)
//   transposes  in[fx ? ph-1-x : x][fy ? pw-1-y : y]                      (output ph x pw)
// Element sizes are 1 byte (8-bit planar), 2 (9-16-bit planar, NV12 pairs) and 4 (P010 / P016 pairs); the kernels are
// templated on the element size of the luma plane and of the chroma planes, so one launch covers every plane.
//
// Flips: every thread owns one 16-byte chunk of an output row.  The 16 source bytes are fetched with one aligned load,
// or with the two aligned loads that cover them and a funnel shift when the mirrored source does not line up with the
// output chunk (pw * elem not a multiple of 16, or a source pitch that breaks the alignment); a mirror then reverses
// the elements in registers (__byte_perm for bytes, half-word swaps for 16-bit elements, word order for 32-bit ones).
//
// Transposes: one CTA moves one square tile of N = 128 / elem elements (128 bytes a row) through shared memory.  Each
// thread reads 16 bytes of 4 / elem consecutive source rows (an output-row-aligned window, fetched as above, mirrored
// when fy), transposes them in registers into 32-bit words that each hold 4 / elem elements of one source column (4 x 4
// byte blocks by __byte_perm for 1-byte elements, 2 x 2 half-word blocks for 2-byte ones), and stores those words;
// after the barrier each thread reads 4 words of one tile column and writes them as 16 bytes of an output row.  Global
// reads and writes are full 128-byte row segments.  The word array is [N columns][32 row groups], with the row group
// index XOR-swizzled by ((col / (16 / elem)) & 7) << 2 | (col & 3): the stores (a warp = 8 column chunks x 4 row groups)
// and the loads (a warp = 4 columns x 8 row-group quads) each hit 32 different banks.
//
// Edges and pitches: every row computes its own pointers.  A chunk that would pass a row's end, or whose output row is
// not 16-byte aligned (an odd device pitch), is done element by element over the same samples, so nothing outside a
// row's samples is written; partial edge tiles are predicated the same way.  An aligned 16-byte load never leaves the
// 16-byte block of a byte the row owns.  HBM bound: read one frame, write one frame.
#include "hbcu_common.h"
#include "hbcu_frames.h"
#include "hbcu_staging.h"
#include "../../include/hbcu.h"

#include <climits>
#include <new>

namespace {

using hbcu::set_error;

constexpr int kThreads = 256;

struct RotPlane
{
    const uint8_t *src;
    uint8_t *dst;
    int spitch, dpitch;          // bytes
    int pw, ph;                  // the source plane in elements
};

struct RotateArgs
{
    RotPlane p[3];
    unsigned first[4];           // first work unit of each plane (flips: output chunk, transposes: tile); [3] = total
    int units_x[3];              // flips: 16-byte chunks per output row; transposes: tiles per output row
    int fx, fy;                  // see the mapping above
};

__device__ __forceinline__ bool aligned(const void *p, unsigned a) { return ((uintptr_t)p & (a - 1)) == 0; }

// the 16 bytes at p, any alignment: one aligned load, or the two that cover them and a funnel shift
__device__ __forceinline__ uint4 load16(const uint8_t *p)
{
    const unsigned s = (unsigned)((uintptr_t)p & 15);
    const uint4 *q = (const uint4 *)(p - s);
    const uint4 lo = __ldg(q);
    if (s == 0) return lo;
    const uint4 hi = __ldg(q + 1);
    uint32_t v0 = lo.x, v1 = lo.y, v2 = lo.z, v3 = lo.w, v4 = hi.x, v5 = hi.y, v6 = hi.z, v7 = hi.w;
    if (s & 8) { v0 = v2; v1 = v3; v2 = v4; v3 = v5; v4 = v6; v5 = v7; }     // words s/4 .. s/4+4 into v0 .. v4
    if (s & 4) { v0 = v1; v1 = v2; v2 = v3; v3 = v4; v4 = v5; }
    const unsigned b = (s & 3) * 8;
    return make_uint4(__funnelshift_r(v0, v1, b), __funnelshift_r(v1, v2, b), __funnelshift_r(v2, v3, b),
                      __funnelshift_r(v3, v4, b));
}

// the E-byte elements of 16 bytes in reverse order
template <int E>
__device__ __forceinline__ uint4 reverse16(uint4 v)
{
    if (E == 4) return make_uint4(v.w, v.z, v.y, v.x);
    constexpr unsigned sel = E == 2 ? 0x1032 : 0x0123;
    return make_uint4(__byte_perm(v.w, 0, sel), __byte_perm(v.z, 0, sel), __byte_perm(v.y, 0, sel), __byte_perm(v.x, 0, sel));
}

template <int E>
__device__ __forceinline__ uint32_t load_elem(const uint8_t *p)
{
    if (E == 1) return *p;
    if (aligned(p, E)) return E == 2 ? (uint32_t)*(const uint16_t *)p : *(const uint32_t *)p;
    uint32_t v = 0;
#pragma unroll
    for (int b = 0; b < E; b++) v |= (uint32_t)p[b] << (8 * b);
    return v;
}

template <int E>
__device__ __forceinline__ void store_elem(uint8_t *p, uint32_t v)
{
    if (E == 1) { *p = (uint8_t)v; return; }
    if (aligned(p, E))
    {
        if (E == 2) *(uint16_t *)p = (uint16_t)v;
        else        *(uint32_t *)p = v;
        return;
    }
#pragma unroll
    for (int b = 0; b < E; b++) p[b] = (uint8_t)(v >> (8 * b));
}

__device__ __forceinline__ uint32_t word_of(const uint4 &v, int i) { return i == 0 ? v.x : i == 1 ? v.y : i == 2 ? v.z : v.w; }

// element e of 16 bytes (e a compile-time index after unrolling)
template <int E>
__device__ __forceinline__ uint32_t elem_of(const uint4 &v, int e)
{
    const uint32_t w = word_of(v, e * E / 4);
    return E == 4 ? w : E == 2 ? (w >> (16 * (e & 1))) & 0xFFFFu : (w >> (8 * (e & 3))) & 0xFFu;
}

template <int E>
__device__ __forceinline__ void set_elem(uint4 &v, int e, uint32_t x)
{
    uint32_t *w = e * E / 4 == 0 ? &v.x : e * E / 4 == 1 ? &v.y : e * E / 4 == 2 ? &v.z : &v.w;
    if (E == 4) *w = x;
    else if (E == 2) *w |= x << (16 * (e & 1));
    else *w |= x << (8 * (e & 3));
}

// ---------------------------------------------------------------------------------------------------------- flips
template <int E>
__device__ __forceinline__ void flip_chunk(const RotPlane &P, int row, int c, bool hf, bool vf)
{
    constexpr int NE = 16 / E;
    const int rb = P.pw * E;
    const uint8_t *s = P.src + (size_t)(vf ? P.ph - 1 - row : row) * P.spitch;
    uint8_t *d = P.dst + (size_t)row * P.dpitch;
    const int b0 = c * 16;
    if (b0 + 16 <= rb && aligned(d, 16))
    {
        uint4 v = load16(s + (hf ? rb - b0 - 16 : b0));
        if (hf) v = reverse16<E>(v);
        *(uint4 *)(d + b0) = v;
        return;
    }
    const int x0 = c * NE, x1 = min(x0 + NE, P.pw);
    for (int x = x0; x < x1; x++)
        store_elem<E>(d + x * E, load_elem<E>(s + (hf ? P.pw - 1 - x : x) * E));
}

__device__ __forceinline__ int plane_of(const RotateArgs &a, unsigned u)
{
    return u >= a.first[1] ? (u >= a.first[2] ? 2 : 1) : 0;
}

// plane p's fields by selects, so the kernel parameters are never indexed at run time
__device__ __forceinline__ unsigned first_of(const RotateArgs &a, int p) { return p == 0 ? a.first[0] : p == 1 ? a.first[1] : a.first[2]; }
__device__ __forceinline__ unsigned units_of(const RotateArgs &a, int p) { return (unsigned)(p == 0 ? a.units_x[0] : p == 1 ? a.units_x[1] : a.units_x[2]); }
__device__ __forceinline__ RotPlane chroma_of(const RotateArgs &a, int p) { return p == 1 ? a.p[1] : a.p[2]; }

template <int E0, int E1>
__global__ void __launch_bounds__(kThreads) flip_kernel(const RotateArgs a)
{
    const unsigned g = blockIdx.x * kThreads + threadIdx.x;
    if (g >= a.first[3]) return;
    const int p = plane_of(a, g);
    const unsigned u = g - first_of(a, p), n = units_of(a, p);
    const int row = (int)(u / n), c = (int)(u % n);
    if (p == 0) flip_chunk<E0>(a.p[0], row, c, a.fx, a.fy);
    else        flip_chunk<E1>(chroma_of(a, p), row, c, a.fx, a.fy);
}

// ---------------------------------------------------------------------------------------------------------- transposes
// word index of (tile column col, row group g) in the swizzled [N][32] array; B = 4 / E elements per word
template <int E>
__device__ __forceinline__ int tidx(int col, int g)
{
    constexpr int CPC = 16 / E;                                // tile columns per 16-byte chunk
    return col * 32 + (g ^ ((((col / CPC) & 7) << 2) | (col & 3)));
}

template <int E>
__device__ __forceinline__ void transpose_tile(uint32_t *T, const RotPlane &P, int ox0, int oy0, bool fx, bool fy)
{
    constexpr int N = 128 / E, B = 4 / E, CPC = 16 / E;
    const int OW = P.ph, OH = P.pw;                             // output plane
    const int t = threadIdx.x;
    // ---- load: row group g (tile rows g*B .. g*B+B-1 = output columns), chunk k (tile columns k*CPC .. = output rows)
    {
        const int k = t & 7, g = t >> 3;
        const int j0 = k * CPC;                                 // first tile column of the chunk
        const bool full = oy0 + j0 + CPC <= OH;
        uint4 r[B];
#pragma unroll
        for (int b = 0; b < B; b++)
        {
            r[b] = make_uint4(0, 0, 0, 0);
            const int x = ox0 + g * B + b;                      // output column
            if (x >= OW) continue;
            const uint8_t *srow = P.src + (size_t)(fx ? OW - 1 - x : x) * P.spitch;
            if (full)
            {
                const uint4 v = load16(srow + (size_t)(fy ? OH - (oy0 + j0 + CPC) : oy0 + j0) * E);
                r[b] = fy ? reverse16<E>(v) : v;
            }
            else
            {
#pragma unroll
                for (int e = 0; e < CPC; e++)
                {
                    const int y = oy0 + j0 + e;
                    if (y < OH) set_elem<E>(r[b], e, load_elem<E>(srow + (size_t)(fy ? OH - 1 - y : y) * E));
                }
            }
        }
        // r[b] holds elements (tile row g*B+b, tile columns j0 ..); make one word per tile column, rows in byte order
#pragma unroll
        for (int w = 0; w < 4; w++)
        {
            if (E == 4)
            {
                T[tidx<E>(j0 + w, g)] = word_of(r[0], w);
            }
            else if (E == 2)
            {
                const uint32_t a = word_of(r[0], w), c = word_of(r[B - 1], w);
                T[tidx<E>(j0 + 2 * w, g)]     = __byte_perm(a, c, 0x5410);
                T[tidx<E>(j0 + 2 * w + 1, g)] = __byte_perm(a, c, 0x7632);
            }
            else
            {
                const uint32_t r0 = word_of(r[0], w), r1 = word_of(r[1 % B], w), r2 = word_of(r[2 % B], w), r3 = word_of(r[3 % B], w);
                const uint32_t lo01 = __byte_perm(r0, r1, 0x5140), hi01 = __byte_perm(r0, r1, 0x7362);
                const uint32_t lo23 = __byte_perm(r2, r3, 0x5140), hi23 = __byte_perm(r2, r3, 0x7362);
                T[tidx<E>(j0 + 4 * w, g)]     = __byte_perm(lo01, lo23, 0x5410);
                T[tidx<E>(j0 + 4 * w + 1, g)] = __byte_perm(lo01, lo23, 0x7632);
                T[tidx<E>(j0 + 4 * w + 2, g)] = __byte_perm(hi01, hi23, 0x5410);
                T[tidx<E>(j0 + 4 * w + 3, g)] = __byte_perm(hi01, hi23, 0x7632);
            }
        }
    }
    __syncthreads();
    // ---- store: tile column c is output row oy0 + c; thread k writes its 16 bytes (row groups 4k .. 4k+3)
#pragma unroll
    for (int pass = 0; pass < N / 32; pass++)
    {
        const int c = pass * 32 + (t >> 3), k = t & 7;
        const int y = oy0 + c;
        if (y >= OH) continue;
        const uint4 v = make_uint4(T[tidx<E>(c, 4 * k)], T[tidx<E>(c, 4 * k + 1)], T[tidx<E>(c, 4 * k + 2)], T[tidx<E>(c, 4 * k + 3)]);
        uint8_t *d = P.dst + (size_t)y * P.dpitch;
        const int x0 = ox0 + k * CPC;
        if (x0 + CPC <= OW && aligned(d, 16))
        {
            *(uint4 *)(d + (size_t)x0 * E) = v;
        }
        else
        {
#pragma unroll
            for (int e = 0; e < CPC; e++)
                if (x0 + e < OW) store_elem<E>(d + (size_t)(x0 + e) * E, elem_of<E>(v, e));
        }
    }
}

template <int E0, int E1>
__global__ void __launch_bounds__(kThreads) transpose_kernel(const RotateArgs a)
{
    constexpr int EMIN = E0 < E1 ? E0 : E1;
    __shared__ uint32_t T[(128 / EMIN) * 32];
    const int p = plane_of(a, blockIdx.x);
    const unsigned u = blockIdx.x - first_of(a, p), n = units_of(a, p);
    const int tx = (int)(u % n), ty = (int)(u / n);
    if (p == 0) transpose_tile<E0>(T, a.p[0], tx * (128 / E0), ty * (128 / E0), a.fx, a.fy);
    else        transpose_tile<E1>(T, chroma_of(a, p), tx * (128 / E1), ty * (128 / E1), a.fx, a.fy);
}

// transform -> (transpose, fx, fy)
struct Mapping { bool transpose; int fx, fy; };
bool mapping_of(int transform, Mapping *m)
{
    switch (transform)
    {
        case HBCU_ROTATE_HFLIP:       *m = {false, 1, 0}; return true;
        case HBCU_ROTATE_VFLIP:       *m = {false, 0, 1}; return true;
        case HBCU_ROTATE_180:         *m = {false, 1, 1}; return true;
        case HBCU_ROTATE_CLOCK:       *m = {true, 1, 0}; return true;
        case HBCU_ROTATE_CLOCK_FLIP:  *m = {true, 1, 1}; return true;
        case HBCU_ROTATE_CCLOCK:      *m = {true, 0, 1}; return true;
        case HBCU_ROTATE_CCLOCK_FLIP: *m = {true, 0, 0}; return true;
        default:                      return false;
    }
}

}  // namespace

struct hbcu_rotate_s
{
    hbcu_rotate_config_t cfg;
    Mapping map;
    int e0, e1;
    RotateArgs geom;             // everything but the plane pointers and pitches
    unsigned blocks;
    hbcu::Staging st;            // in / out: the planes before and after the transform; an absent third plane has 0 rows
};

namespace {

template <int E0, int E1>
void launch_pair(const hbcu_rotate_s *h, const RotateArgs &a)
{
    if (h->map.transpose) transpose_kernel<E0, E1><<<h->blocks, kThreads, 0, h->st.s_compute>>>(a);
    else                  flip_kernel<E0, E1><<<h->blocks, kThreads, 0, h->st.s_compute>>>(a);
}

int launch(hbcu_rotate_s *h, const uint8_t *const src[3], const int spitch[3], uint8_t *const dst[3], const int dpitch[3])
{
    RotateArgs a = h->geom;
    for (int p = 0; p < h->cfg.planes; p++)
    {
        a.p[p].src = src[p]; a.p[p].dst = dst[p];
        a.p[p].spitch = spitch[p]; a.p[p].dpitch = dpitch[p];
    }
    const int key = h->e0 * 10 + h->e1;
    switch (key)
    {
        case 11: launch_pair<1, 1>(h, a); break;
        case 22: launch_pair<2, 2>(h, a); break;
        case 12: launch_pair<1, 2>(h, a); break;
        case 24: launch_pair<2, 4>(h, a); break;
        default: set_error("rotate_frame: element sizes %d / %d", h->e0, h->e1); return -1;
    }
    hbcu::count_launch();
    HBCU_CHECK(cudaGetLastError());
    return 0;
}

}  // namespace

extern "C" {

int hbcu_rotate_create(hbcu_rotate_t **out, const hbcu_rotate_config_t *cfg)
{
    if (out == nullptr || cfg == nullptr) { set_error("rotate_create: null argument"); return -1; }
    *out = nullptr;
    Mapping map;
    if (!mapping_of(cfg->transform, &map)) { set_error("rotate_create: unknown transform %d", cfg->transform); return -1; }
    if (cfg->planes != 2 && cfg->planes != 3)
    {
        set_error("rotate_create: %d planes (2: semi-planar, 3: planar)", cfg->planes);
        return -1;
    }
    const int e0 = cfg->elem_bytes[0], e1 = cfg->elem_bytes[1];
    const bool pair_ok = (e0 == 1 && (e1 == 1 || e1 == 2)) || (e0 == 2 && (e1 == 2 || e1 == 4));
    if (!pair_ok || (cfg->planes == 3 && cfg->elem_bytes[2] != e1))
    {
        set_error("rotate_create: element sizes %d / %d / %d (1 / 1 / 1, 2 / 2 / 2, 1 / 2 and 2 / 4)", e0, e1,
                  cfg->planes == 3 ? cfg->elem_bytes[2] : 0);
        return -1;
    }
    for (int p = 0; p < cfg->planes; p++)
        if (cfg->width[p] < 1 || cfg->height[p] < 1 || cfg->width[p] > (1 << 16) || cfg->height[p] > (1 << 16))
        {
            set_error("rotate_create: plane %d is %dx%d elements", p, cfg->width[p], cfg->height[p]);
            return -1;
        }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || cfg->device < 0 || cfg->device >= ndev)
    {
        cudaGetLastError();
        set_error("rotate_create: CUDA device %d not available (%d devices); there is no CPU fallback", cfg->device, ndev);
        return -1;
    }
    HBCU_CHECK(cudaSetDevice(cfg->device));
    cudaDeviceProp prop;
    HBCU_CHECK(cudaGetDeviceProperties(&prop, cfg->device));
    if (prop.major != 9 || prop.minor != 0)
    {
        set_error("rotate_create: device %d is sm_%d%d; this library is built for sm_90a only", cfg->device, prop.major, prop.minor);
        return -1;
    }
    hbcu_rotate_s *h = new (std::nothrow) hbcu_rotate_s();
    if (h == nullptr) { set_error("rotate_create: out of memory"); return -1; }
    h->cfg = *cfg;
    h->map = map;
    h->e0 = e0;
    h->e1 = e1;
    RotateArgs &g = h->geom;
    g = RotateArgs();
    g.fx = map.fx;
    g.fy = map.fy;
    int in_rb[3] = {0, 0, 0}, in_rows[3] = {0, 0, 0}, out_rb[3] = {0, 0, 0}, out_rows[3] = {0, 0, 0};
    size_t total = 0;
    for (int p = 0; p < 3; p++)
    {
        g.first[p] = (unsigned)total;
        if (p >= cfg->planes) continue;
        const int E = cfg->elem_bytes[p], pw = cfg->width[p], ph = cfg->height[p];
        const int ow = map.transpose ? ph : pw, oh = map.transpose ? pw : ph;
        g.p[p].pw = pw;
        g.p[p].ph = ph;
        in_rb[p] = pw * E; in_rows[p] = ph;
        out_rb[p] = ow * E; out_rows[p] = oh;
        if (map.transpose)
        {
            const int n = 128 / E;
            g.units_x[p] = (ow + n - 1) / n;
            total += (size_t)g.units_x[p] * ((oh + n - 1) / n);
        }
        else
        {
            g.units_x[p] = (ow * E + 15) / 16;
            total += (size_t)g.units_x[p] * oh;
        }
    }
    g.first[3] = (unsigned)total;
    h->blocks = (unsigned)(map.transpose ? total : (total + kThreads - 1) / kThreads);
    h->st.in_bytes = hbcu::stage_layout(h->st.in, in_rb, in_rows);
    h->st.out_bytes = hbcu::stage_layout(h->st.out, out_rb, out_rows);
    if (total > (size_t)INT_MAX)
    {
        set_error("rotate_create: frame too large");
        delete h;
        return -1;
    }
    if (hbcu::stage_init(&h->st, "rotate", cfg->device, cfg->slots >= 2 ? cfg->slots : 4) != 0)
    {
        hbcu_rotate_destroy(h);
        return -1;
    }
    *out = h;
    return 0;
}

void hbcu_rotate_destroy(hbcu_rotate_t *h)
{
    if (h == nullptr) return;
    hbcu::stage_destroy(&h->st);
    delete h;
}

int hbcu_rotate_frame(hbcu_rotate_t *h, int64_t ticket,
                      hbcu_frame_t *in_frame, const void *const in_planes[3], const int in_strides[3],
                      hbcu_frame_t *out_frame, void *const out_planes[3], const int out_strides[3])
{
    if (h == nullptr) { set_error("rotate_frame: bad argument"); return -1; }
    return hbcu::stage_submit(&h->st, "frame", ticket, in_frame, in_planes, in_strides, out_frame, out_planes, out_strides,
                              [h](const uint8_t *const src[3], const int spitch[3], uint8_t *const dst[3], const int dpitch[3])
                              { return launch(h, src, spitch, dst, dpitch); });
}

int hbcu_rotate_wait(hbcu_rotate_t *h, int64_t ticket)
{
    if (h == nullptr) { set_error("rotate_wait: null handle"); return -1; }
    return hbcu::stage_wait(&h->st, ticket);
}

int hbcu_rotate_poll(hbcu_rotate_t *h, int64_t ticket)
{
    if (h == nullptr) { set_error("rotate_poll: null handle"); return -1; }
    return hbcu::stage_poll(&h->st, ticket);
}

int hbcu_rotate_sync(hbcu_rotate_t *h)
{
    if (h == nullptr) { set_error("rotate_sync: null handle"); return -1; }
    return hbcu::stage_sync(&h->st);
}

int hbcu_rotate_mark(hbcu_rotate_t *h, int which)
{
    if (h == nullptr || which < 0 || which > 1) { set_error("rotate_mark: bad argument"); return -1; }
    return hbcu::stage_mark(&h->st, which);
}

int hbcu_rotate_elapsed_ms(hbcu_rotate_t *h, float *ms)
{
    if (h == nullptr || ms == nullptr) { set_error("rotate_elapsed_ms: bad argument"); return -1; }
    return hbcu::stage_elapsed_ms(&h->st, ms);
}

}  // extern "C"
