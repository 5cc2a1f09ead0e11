// hqdn3d.cu -- hqdn3d ("high quality 3-D denoise") for sm_90a behind the C-ABI of include/hbcu.h (SURVEY.md 8 f4).
//
// Replaces hqdn3d_denoise_spatial / _temporal / _depth (reference libhb/denoise.c:102-201).
// The reference sweeps a plane once, carrying three recursive low-passes: along the row (pixel_ant), down the column
// (line_ant[]) and through time (frame_ant[]).  lowpass(prev, cur) = cur + coef[(prev - cur) >> (8 - LUT_BITS)] is a table
// lookup, not a linear filter, so the recursions cannot be turned into scans -- but they separate:
//   H  rows are independent of each other        -> one thread per row marches along x      (hqdn3d_h_kernel)
//   V  columns are independent once H is known    -> one thread per column marches down y,
//   T  the temporal step is per sample               fused into the same march               (hqdn3d_vt_kernel)
// (oracle/port/hqdn3d_port.c restates the filter in exactly this three-pass form and is pinned against the compiled
// reference.)  Parallelism is the plane's height resp. width, each thread a dependent chain of table lookups: the kernels
// are latency bound by construction; tiles go through shared memory so that global accesses stay coalesced although a
// thread owns a row.  The 16-bit fixed-point domain, the bias of LOAD, the uint16 truncation of the stored states and the
// first-row special case (h(0) = lowpass(LOAD(0), LOAD(0)) only in row 0) are reproduced: bit-exact.
#include "hbcu_common.h"
#include "hbcu_frames.h"
#include "../../include/hbcu.h"

#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>

namespace {

using hbcu::set_error;

__device__ __forceinline__ int lowpass(int prev, int cur, const int16_t *__restrict__ coef, int shift)
{
    return cur + (int)coef[(prev - cur) >> shift];          // coef points at the table's centre
}

template <typename PIX>
__device__ __forceinline__ int load16(const PIX *p, int sh, int bias) { return ((int)*p << sh) + bias; }

// H pass: warp = 32 rows, lane = row; 32 x 32 tiles staged through shared memory (pitch 33: conflict free both ways)
template <typename PIX, bool SMEM_LUT>
__global__ void __launch_bounds__(128) hqdn3d_h_kernel(const PIX *__restrict__ src, int spitch, uint16_t *__restrict__ hbuf,
                                                      int w, int h, int depth, const int16_t *__restrict__ table, int half)
{
    extern __shared__ int16_t s_lut[];
    __shared__ uint16_t tile[4][32][33];
    const int16_t *coef = table + half;
    if (SMEM_LUT)
    {
        for (int i = threadIdx.x; i < 2 * half; i += blockDim.x) s_lut[i] = table[i];
        __syncthreads();
        coef = s_lut + half;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int row0 = (blockIdx.x * 4 + warp) * 32, row = row0 + lane;
    if (row0 >= h) return;
    const int sh = 16 - depth, bias = ((1 << sh) - 1) >> 1, lsh = depth == 16 ? 0 : 4;
    int p = 0;
    // The chain of dependent table lookups is the kernel's critical path; the global loads of the NEXT 32 x 32 tile are
    // issued before the chain of the current one starts and land in registers while it runs (round 2: the loads used to
    // sit exposed between two chains -- ~2000 cycles per tile at one warp per 32 rows).
    uint16_t nxt[32];
#pragma unroll
    for (int r = 0; r < 32; r++)
    {
        const int y = row0 + r, x = lane;
        nxt[r] = (y < h && x < w) ? (uint16_t)load16(src + (size_t)y * spitch + x, sh, bias) : 0;
    }
    for (int x0 = 0; x0 < w; x0 += 32)
    {
#pragma unroll
        for (int r = 0; r < 32; r++) tile[warp][r][lane] = nxt[r];
        __syncwarp();
        if (x0 + 32 < w)
        {
#pragma unroll
            for (int r = 0; r < 32; r++)
            {
                const int y = row0 + r, x = x0 + 32 + lane;
                nxt[r] = (y < h && x < w) ? (uint16_t)load16(src + (size_t)y * spitch + x, sh, bias) : 0;
            }
        }
        if (row < h)
        {
            // the row's 32 samples first (independent loads), then the dependent chain: one table lookup per step
            const int n = min(32, w - x0);
            int v[32];
#pragma unroll
            for (int c = 0; c < 32; c++) v[c] = tile[warp][lane][c];
#pragma unroll
            for (int c = 0; c < 32; c++)
            {
                if (c < n)
                {
                    if (c == 0 && x0 == 0) p = row == 0 ? lowpass(v[0], v[0], coef, lsh) : v[0];   // denoise.c:140-143 vs :152
                    else                   p = lowpass(p, v[c], coef, lsh);
                    v[c] = p;
                }
            }
#pragma unroll
            for (int c = 0; c < 32; c++) tile[warp][lane][c] = (uint16_t)v[c];
        }
        __syncwarp();
#pragma unroll 8
        for (int r = 0; r < 32; r++)
        {
            const int y = row0 + r, x = x0 + lane;
            if (y < h && x < w) hbuf[(size_t)y * w + x] = tile[warp][r][lane];
        }
        __syncwarp();
    }
}

// V + T pass: thread = column.  SPATIAL = false is the temporal-only mode (denoise.c:102-124): v = LOAD(src).
template <typename PIX, bool SMEM_LUT, bool SPATIAL>
__global__ void __launch_bounds__(128) hqdn3d_vt_kernel(const PIX *__restrict__ src, int spitch, const uint16_t *__restrict__ hbuf,
                                                       uint16_t *__restrict__ ant, int first, PIX *__restrict__ dst, int dpitch,
                                                       int w, int h, int depth, const int16_t *__restrict__ stable,
                                                       const int16_t *__restrict__ ttable, int half)
{
    extern __shared__ int16_t s_lut[];
    const int16_t *scoef = stable + half, *tcoef = ttable + half;
    if (SMEM_LUT)
    {
        for (int i = threadIdx.x; i < 2 * half; i += blockDim.x)
        {
            s_lut[i] = stable[i];
            s_lut[2 * half + i] = ttable[i];
        }
        __syncthreads();
        scoef = s_lut + half;
        tcoef = s_lut + 3 * half;
    }
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= w) return;
    const int sh = 16 - depth, bias = ((1 << sh) - 1) >> 1, lsh = depth == 16 ? 0 : 4;
    constexpr int U = 16;                                  // rows per batch: the NEXT batch is fetched while this one's chain runs
    int v = 0;
    int ncur[U], na[U];
    auto fetch = [&](int y0) {
#pragma unroll
        for (int k = 0; k < U; k++)
        {
            const int y = min(y0 + k, h - 1);
            const int s = load16(src + (size_t)y * spitch + x, sh, bias);
            ncur[k] = SPATIAL ? (int)hbuf[(size_t)y * w + x] : s;
            na[k] = first ? s : (int)ant[(size_t)y * w + x];           // denoise.c:175-189: the state starts as the first frame
        }
    };
    fetch(0);
    for (int y0 = 0; y0 < h; y0 += U)
    {
        int cur[U], a[U];
#pragma unroll
        for (int k = 0; k < U; k++) { cur[k] = ncur[k]; a[k] = na[k]; }
        // rows y0+U .. y0+2U-1 are not written before this batch's stores (a thread owns its column), so fetching `ant`
        // ahead of them is safe
        if (y0 + U < h) fetch(y0 + U);
#pragma unroll
        for (int k = 0; k < U; k++)
        {
            const int y = y0 + k;
            if (y >= h) break;
            if (SPATIAL) v = y == 0 ? cur[k] : lowpass(v, cur[k], scoef, lsh);
            else         v = cur[k];
            v &= 0xffff;                                   // line_ant[] is uint16_t
            const int t = lowpass(a[k], v, tcoef, lsh);
            ant[(size_t)y * w + x] = (uint16_t)t;
            dst[(size_t)y * dpitch + x] = (PIX)((unsigned)t >> sh);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Round 2: warp-specialised kernels.  ncu showed the kernels above at 6-14 cycles per instruction: one warp per scheduler
// executes ~50 instructions per sample (address arithmetic, guards, conversions, stores) in series with its lookup chain.
// Here the chain warp does nothing but the chain -- samples come from and go back to shared memory as 16-bit values, 8 at
// a time -- and helper warps of the same CTA move the tiles (16-byte global accesses, conversion, and in the V+T pass the
// temporal low-pass, which is not recursive within a frame).  A three-deep ring of tiles is handed on with one
// __syncthreads per step: helper loads tile s, chain works on tile s-1, helper retires tile s-2.
// Requirements (checked by the launcher, the kernels above remain for everything else): depth < 16 (tables in shared
// memory, index shift 4), width a multiple of 8, 16-byte aligned planes and pitches.
constexpr int kTileW = 128, kTilePitch = kTileW * 2 + 16;       // bytes per tile row: 17 x 16 B, conflict free for LDS.128 by row

__device__ __forceinline__ int lut_at(const int16_t *centre, int d)
{
    // centre[d >> 4] with the index scaled to bytes in two instructions: (d >> 3) & ~1
    return *reinterpret_cast<const int16_t *>(reinterpret_cast<const char *>(centre) + ((d >> 3) & ~1));
}

template <typename PIX>
__device__ __forceinline__ void widen_store(unsigned char *dst, const uint4 q, bool inside, int sh, int bias)
{
    // 16 (8-bit) or 8 (16-bit) samples -> LOAD()'s 16-bit fixed point (denoise.c:33), stored as 16-byte vectors
    const uint32_t b2 = inside ? (uint32_t)bias * 0x10001u : 0u;
    if (sizeof(PIX) == 1)
    {
        const uint32_t w[4] = { q.x, q.y, q.z, q.w };
        uint32_t o[8];
#pragma unroll
        for (int i = 0; i < 4; i++)
        {
            o[2 * i]     = __byte_perm(w[i], 0, 0x1404) + b2;        // bytes 0, 1 -> the high bytes of two halves (sh = 8)
            o[2 * i + 1] = __byte_perm(w[i], 0, 0x3424) + b2;
        }
        *reinterpret_cast<uint4 *>(dst)      = make_uint4(o[0], o[1], o[2], o[3]);
        *reinterpret_cast<uint4 *>(dst + 16) = make_uint4(o[4], o[5], o[6], o[7]);
    }
    else
        *reinterpret_cast<uint4 *>(dst) = make_uint4((q.x << sh) + b2, (q.y << sh) + b2, (q.z << sh) + b2, (q.w << sh) + b2);
}

__device__ __forceinline__ void stage_lut(int16_t *dst, const int16_t *__restrict__ table, int entries)
{
    const uint4 *s4 = reinterpret_cast<const uint4 *>(table);
    uint4 *d4 = reinterpret_cast<uint4 *>(dst);
    for (int i = threadIdx.x; i < entries / 8; i += blockDim.x) d4[i] = __ldg(s4 + i);
}

// H pass: CTA = 32 rows; warp 0 = chain (lane = row), warps 1-3 = helpers (one helper alone took longer over a tile than
// the chain: 6 us per 128 columns against 3)
constexpr int kHHelpers = 3 * 32;
template <typename PIX>
__global__ void __launch_bounds__(32 + kHHelpers, 1) hqdn3d_h2_kernel(const PIX *__restrict__ src, int spitch, uint16_t *__restrict__ hbuf,
                                                                   int w, int h, int depth, const int16_t *__restrict__ table, int half)
{
    extern __shared__ __align__(16) unsigned char smem2[];
    int16_t *s_lut = reinterpret_cast<int16_t *>(smem2);
    unsigned char *tiles = smem2 + (size_t)2 * half * sizeof(int16_t);
    stage_lut(s_lut, table, 2 * half);
    __syncthreads();
    const int16_t *coef = s_lut + half;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int row0 = blockIdx.x * 32;
    const int sh = 16 - depth, bias = ((1 << sh) - 1) >> 1;
    const int ntiles = (w + kTileW - 1) / kTileW;
    constexpr int SPV = 16 / (int)sizeof(PIX);            // samples per 16-byte global load
    int p = 0;
    for (int s = 0; s < ntiles + 2; s++)
    {
        if (warp >= 1)
        {
            const int ht = threadIdx.x - 32;
            constexpr int LPR = kTileW / SPV;             // chunks per row
            constexpr int NCH = 32 * LPR, IT = (NCH + kHHelpers - 1) / kHHelpers;
            uint4 q[IT];
            unsigned ok = 0;
            if (s < ntiles)                               // all loads of the tile first, then conversion and stores
            {
#pragma unroll
                for (int it = 0; it < IT; it++)
                {
                    const int idx = it * kHHelpers + ht, r = idx / LPR, c = (idx % LPR) * SPV;
                    const int y = row0 + r, x = s * kTileW + c;
                    q[it] = make_uint4(0, 0, 0, 0);
                    if (idx < NCH && y < h && x < w)
                    {
                        q[it] = __ldg(reinterpret_cast<const uint4 *>(src + (size_t)y * spitch + x));
                        ok |= 1u << it;
                    }
                }
            }
            if (s >= 2)
            {
                const unsigned char *buf = tiles + (size_t)((s - 2) % 3) * 32 * kTilePitch;
#pragma unroll
                for (int it = 0; it < (32 * 16 + kHHelpers - 1) / kHHelpers; it++)
                {
                    const int idx = it * kHHelpers + ht, r = idx >> 4, c = (idx & 15) * 8;
                    const int y = row0 + r, x = (s - 2) * kTileW + c;
                    if (idx < 32 * 16 && y < h && x < w)
                        *reinterpret_cast<uint4 *>(hbuf + (size_t)y * w + x) = *reinterpret_cast<const uint4 *>(buf + r * kTilePitch + c * 2);
                }
            }
            if (s < ntiles)
            {
                unsigned char *buf = tiles + (size_t)(s % 3) * 32 * kTilePitch;
#pragma unroll
                for (int it = 0; it < IT; it++)
                {
                    const int idx = it * kHHelpers + ht, r = idx / LPR, c = (idx % LPR) * SPV;
                    if (idx >= NCH) continue;
                    // samples outside the plane are zeros: the chain walks over them (results dropped) and must stay inside the table
                    widen_store<PIX>(buf + r * kTilePitch + c * 2, q[it], (ok >> it) & 1, sh, bias);
                }
            }
        }
        else if (s >= 1 && s <= ntiles)
        {
            unsigned char *rowp = tiles + (size_t)((s - 1) % 3) * 32 * kTilePitch + lane * kTilePitch;
            uint4 q = *reinterpret_cast<const uint4 *>(rowp);
#pragma unroll 2
            for (int g = 0; g < kTileW / 8; g++)
            {
                const uint4 qn = *reinterpret_cast<const uint4 *>(rowp + (g + 1 < kTileW / 8 ? g + 1 : g) * 16);
                const uint32_t wv[4] = { q.x, q.y, q.z, q.w };
                int cur[8], out[8];
#pragma unroll
                for (int i = 0; i < 4; i++) { cur[2 * i] = (int)(wv[i] & 0xffffu); cur[2 * i + 1] = (int)(wv[i] >> 16); }
                int d, l;
                if (s == 1 && g == 0)
                {
                    // first column: lowpass(LOAD(0), LOAD(0)) in row 0, the plain sample elsewhere (denoise.c:140-143 vs :152)
                    out[0] = (row0 + lane == 0) ? cur[0] + lut_at(coef, 0) : cur[0];
                }
                else
                {
                    d = p - cur[0];
                    l = lut_at(coef, d);
                    out[0] = cur[0] + l;
                }
                // out[c] = cur[c] + l_c;  the next index needs only l_c + (cur[c] - cur[c+1]): one add between two lookups
                d = out[0] - cur[1];
#pragma unroll
                for (int c = 1; c < 8; c++)
                {
                    l = lut_at(coef, d);
                    out[c] = cur[c] + l;
                    // (an opaque add: the compiler otherwise re-associates this into out[c] - cur[c+1], two adds on the chain)
                    if (c < 7) asm("add.s32 %0, %1, %2;" : "=r"(d) : "r"(l), "r"(cur[c] - cur[c + 1]));
                }
                p = out[7];
                uint4 o;
                o.x = __byte_perm(out[0], out[1], 0x5410); o.y = __byte_perm(out[2], out[3], 0x5410);
                o.z = __byte_perm(out[4], out[5], 0x5410); o.w = __byte_perm(out[6], out[7], 0x5410);
                *reinterpret_cast<uint4 *>(rowp + g * 16) = o;
                q = qn;
            }
        }
        __syncthreads();
    }
}

// V + T pass: CTA = 128 columns; warps 0-3 = chains (lane = column), warps 4-11 = helpers (with four, the helpers' share of a
// tile -- 32 temporal lookups per thread -- took twice as long as the chain).  Tiles are 32 rows deep.
template <typename PIX>
__global__ void __launch_bounds__(384, 1) hqdn3d_vt2_kernel(const PIX *__restrict__ src, int spitch, const uint16_t *__restrict__ hbuf,
                                                        uint16_t *__restrict__ ant, int first, PIX *__restrict__ dst, int dpitch,
                                                        int w, int h, int depth, const int16_t *__restrict__ stable,
                                                        const int16_t *__restrict__ ttable, int half)
{
    extern __shared__ __align__(16) unsigned char smem2[];
    int16_t *s_lut = reinterpret_cast<int16_t *>(smem2);
    unsigned char *tiles = smem2 + (size_t)4 * half * sizeof(int16_t);
    stage_lut(s_lut, stable, 2 * half);
    stage_lut(s_lut + 2 * half, ttable, 2 * half);
    __syncthreads();
    const int16_t *scoef = s_lut + half, *tcoef = s_lut + 3 * half;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int x0 = blockIdx.x * kTileW;
    const int sh = 16 - depth, bias = ((1 << sh) - 1) >> 1;
    const int ntiles = (h + 31) / 32;
    int v = 0;
    // helper registers, one step ahead of their use: the H tile that enters the ring next step, and the `ant` / `src`
    // samples of the tile that retires next step (every global load has a whole step -- a chain over 32 rows -- to land)
    const int ht = threadIdx.x - 128;                     // helper thread 0..255
    uint4 qh[2], qa[2], qs[2];
    auto fetch_h = [&](int t) {
#pragma unroll
        for (int it = 0; it < 2; it++)
        {
            const int r = it * 16 + (ht >> 4), c = (ht & 15) * 8;
            const int y = t * 32 + r, x = x0 + c;
            // samples outside the plane are zeros: the chain walks over them (results dropped) and must stay inside the table
            qh[it] = (y < h && x < w) ? __ldg(reinterpret_cast<const uint4 *>(hbuf + (size_t)y * w + x)) : make_uint4(0, 0, 0, 0);
        }
    };
    auto fetch_retiring = [&](int t) {
#pragma unroll
        for (int it = 0; it < 2; it++)
        {
            const int r = it * 16 + (ht >> 4), c = (ht & 15) * 8;
            const int y = t * 32 + r, x = x0 + c;
            qa[it] = make_uint4(0, 0, 0, 0); qs[it] = make_uint4(0, 0, 0, 0);
            if (y < h && x < w)
            {
                if (!first) qa[it] = *reinterpret_cast<const uint4 *>(ant + (size_t)y * w + x);
                if (sizeof(PIX) == 1)
                {
                    const uint2 t2 = __ldg(reinterpret_cast<const uint2 *>(src + (size_t)y * spitch + x));
                    qs[it].x = t2.x; qs[it].y = t2.y;
                }
                else qs[it] = __ldg(reinterpret_cast<const uint4 *>(src + (size_t)y * spitch + x));
            }
        }
    };
    if (warp >= 4) fetch_h(0);
    for (int s = 0; s < ntiles + 2; s++)
    {
        if (warp >= 4)
        {
            const int rt0 = (s - 2) * 32;
            if (s < ntiles)
            {
                unsigned char *buf = tiles + (size_t)(s % 3) * 32 * kTilePitch;
#pragma unroll
                for (int it = 0; it < 2; it++)
                {
                    const int r = it * 16 + (ht >> 4), c = (ht & 15) * 8;
                    *reinterpret_cast<uint4 *>(buf + r * kTilePitch + c * 2) = qh[it];
                }
            }
            if (s + 1 < ntiles) fetch_h(s + 1);
            if (s >= 2)
            {
                const unsigned char *buf = tiles + (size_t)((s - 2) % 3) * 32 * kTilePitch;
#pragma unroll
                for (int it = 0; it < 2; it++)
                {
                    const int r = it * 16 + (ht >> 4), c = (ht & 15) * 8;
                    const int y = rt0 + r, x = x0 + c;
                    if (!(y < h && x < w)) continue;
                    const uint4 qv = *reinterpret_cast<const uint4 *>(buf + r * kTilePitch + c * 2);
                    const uint32_t vw[4] = { qv.x, qv.y, qv.z, qv.w }, aw[4] = { qa[it].x, qa[it].y, qa[it].z, qa[it].w },
                                   sw[4] = { qs[it].x, qs[it].y, qs[it].z, qs[it].w };
                    uint32_t tw[4], ow[4];
                    int t[8];
#pragma unroll
                    for (int i = 0; i < 8; i++)
                    {
                        const int vv = (int)((i & 1) ? (vw[i >> 1] >> 16) : (vw[i >> 1] & 0xffffu));
                        int a;
                        if (first)                         // denoise.c:175-189: the state starts as the first frame
                        {
                            const int px = sizeof(PIX) == 1 ? (int)((sw[i >> 2] >> (8 * (i & 3))) & 0xffu)
                                                            : (int)((i & 1) ? (sw[i >> 1] >> 16) : (sw[i >> 1] & 0xffffu));
                            a = (px << sh) + bias;
                        }
                        else a = (int)((i & 1) ? (aw[i >> 1] >> 16) : (aw[i >> 1] & 0xffffu));
                        t[i] = vv + lut_at(tcoef, a - vv);
                    }
#pragma unroll
                    for (int i = 0; i < 4; i++) tw[i] = __byte_perm(t[2 * i], t[2 * i + 1], 0x5410);
                    *reinterpret_cast<uint4 *>(ant + (size_t)y * w + x) = make_uint4(tw[0], tw[1], tw[2], tw[3]);
                    if (sizeof(PIX) == 1)
                    {
#pragma unroll
                        for (int i = 0; i < 2; i++)
                            ow[i] = (((unsigned)t[4 * i] >> sh) & 0xffu) | ((((unsigned)t[4 * i + 1] >> sh) & 0xffu) << 8)
                                  | ((((unsigned)t[4 * i + 2] >> sh) & 0xffu) << 16) | ((((unsigned)t[4 * i + 3] >> sh) & 0xffu) << 24);
                        *reinterpret_cast<uint2 *>(dst + (size_t)y * dpitch + x) = make_uint2(ow[0], ow[1]);
                    }
                    else
                    {
#pragma unroll
                        for (int i = 0; i < 4; i++)
                            ow[i] = (((unsigned)t[2 * i] >> sh) & 0xffffu) | ((((unsigned)t[2 * i + 1] >> sh) & 0xffffu) << 16);
                        *reinterpret_cast<uint4 *>(dst + (size_t)y * dpitch + x) = make_uint4(ow[0], ow[1], ow[2], ow[3]);
                    }
                }
            }
            if (s >= 1 && s <= ntiles) fetch_retiring(s - 1);      // tile s-1 retires in step s+1 (this thread writes its `ant` then)
        }
        else if (s >= 1 && s <= ntiles)
        {
            unsigned char *colp = tiles + (size_t)((s - 1) % 3) * 32 * kTilePitch + (warp * 32 + lane) * 2;
            const int y0 = (s - 1) * 32;
            int cur[32];
#pragma unroll
            for (int r = 0; r < 32; r++) cur[r] = *reinterpret_cast<const uint16_t *>(colp + r * kTilePitch);
#pragma unroll
            for (int r = 0; r < 32; r++)
            {
                if (y0 + r == 0) v = cur[0];
                else             v = (cur[r] + lut_at(scoef, v - cur[r])) & 0xffff;      // line_ant[] is uint16_t
                *reinterpret_cast<uint16_t *>(colp + r * kTilePitch) = (uint16_t)v;
            }
        }
        __syncthreads();
    }
}

struct Geom { int w, h, pitch; size_t bytes; };

}  // namespace

struct hbcu_hqdn3d_s
{
    hbcu_hqdn3d_config_t cfg;
    int bps, slots, next, half;
    Geom g[3];
    size_t frame_bytes, plane_off[3];
    std::vector<uint8_t *> in_base, out_base;
    std::vector<int64_t> ticket;
    int16_t *d_coef[6];
    uint16_t *d_ant[3], *d_h[3];
    int first[3];
    bool spatial[3];
    cudaStream_t s_h2d, s_compute, s_d2h;
    cudaStream_t s_pl[3];                // the three planes are independent: they run side by side, forked from / joined to s_compute
    cudaEvent_t ev_fork, ev_join[3];
    std::vector<cudaEvent_t> ev_up, ev_k, ev_down;
    cudaEvent_t ev_mark[2];
};

namespace {

template <typename PIX>
int launch_plane_t(hbcu_hqdn3d_s *h, int pl, const void *src, void *dst, cudaStream_t st)
{
    const Geom &g = h->g[pl];
    const bool smem = h->cfg.depth < 16;
    const size_t lut1 = smem ? (size_t)2 * h->half * sizeof(int16_t) : 0;
    const int depth = h->cfg.depth;
    // round-2 kernels: tables in shared memory, vector accesses
    const bool v2 = smem && h->spatial[pl] && g.w % 8 == 0 && ((uintptr_t)src % 16 == 0) && ((uintptr_t)dst % 16 == 0)
                 && ((size_t)g.pitch * h->bps) % 16 == 0 && getenv("HBCU_HQDN3D_V1") == nullptr;
    if (v2)
    {
        const size_t tiles = (size_t)3 * 32 * kTilePitch;
        hqdn3d_h2_kernel<PIX><<<(g.h + 31) / 32, 32 + kHHelpers, lut1 + tiles, st>>>((const PIX *)src, g.pitch, h->d_h[pl], g.w, g.h, depth, h->d_coef[2 * pl], h->half);
        hbcu::count_launch();
        hqdn3d_vt2_kernel<PIX><<<(g.w + kTileW - 1) / kTileW, 384, 2 * lut1 + tiles, st>>>((const PIX *)src, g.pitch, h->d_h[pl], h->d_ant[pl], h->first[pl],
                       (PIX *)dst, g.pitch, g.w, g.h, depth, h->d_coef[2 * pl], h->d_coef[2 * pl + 1], h->half);
        hbcu::count_launch();
        h->first[pl] = 0;
        HBCU_CHECK(cudaGetLastError());
        return 0;
    }
    if (h->spatial[pl])
    {
        const int hgrid = (g.h + 127) / 128;
        if (smem) hqdn3d_h_kernel<PIX, true><<<hgrid, 128, lut1, st>>>((const PIX *)src, g.pitch, h->d_h[pl], g.w, g.h, depth, h->d_coef[2 * pl], h->half);
        else      hqdn3d_h_kernel<PIX, false><<<hgrid, 128, 0, st>>>((const PIX *)src, g.pitch, h->d_h[pl], g.w, g.h, depth, h->d_coef[2 * pl], h->half);
        hbcu::count_launch();
    }
    const int vgrid = (g.w + 127) / 128;
#define VT(SM, SP) hqdn3d_vt_kernel<PIX, SM, SP><<<vgrid, 128, 2 * lut1, st>>>((const PIX *)src, g.pitch, h->d_h[pl], h->d_ant[pl], h->first[pl], \
                       (PIX *)dst, g.pitch, g.w, g.h, depth, h->d_coef[2 * pl], h->d_coef[2 * pl + 1], h->half)
    if (smem) { if (h->spatial[pl]) VT(true, true); else VT(true, false); }
    else      { if (h->spatial[pl]) VT(false, true); else VT(false, false); }
#undef VT
    hbcu::count_launch();
    h->first[pl] = 0;
    HBCU_CHECK(cudaGetLastError());
    return 0;
}

bool same_layout(const hbcu_hqdn3d_s *h, const void *const planes[3], const int strides[3])
{
    for (int pl = 0; pl < 3; pl++)
    {
        if ((size_t)strides[pl] != (size_t)h->g[pl].pitch * h->bps) return false;
        if ((const uint8_t *)planes[pl] != (const uint8_t *)planes[0] + h->plane_off[pl]) return false;
    }
    return true;
}

bool frame_fits(const hbcu_hqdn3d_s *h, const hbcu_frame_t *f)
{
    if (f->device != h->cfg.device) return false;
    for (int pl = 0; pl < 3; pl++)
        if (f->row_bytes[pl] != h->g[pl].w * h->bps || f->rows[pl] != h->g[pl].h || f->stride[pl] != h->g[pl].pitch * h->bps) return false;
    return true;
}

int find_slot(const hbcu_hqdn3d_s *h, int64_t ticket)
{
    for (int s = 0; s < h->slots; s++)
        if (h->ticket[s] == ticket) return s;
    return -1;
}

}  // namespace

extern "C" {

int hbcu_hqdn3d_create(hbcu_hqdn3d_t **out, const hbcu_hqdn3d_config_t *cfg)
{
    if (out == nullptr || cfg == nullptr) { set_error("hqdn3d_create: null argument"); return -1; }
    *out = nullptr;
    for (int i = 0; i < 6; i++)
        if (cfg->coef[i] == nullptr) { set_error("hqdn3d_create: coefficient table %d missing", i); return -1; }
    if (cfg->width < 1 || cfg->height < 1 || cfg->depth < 8 || cfg->depth > 16)
    {
        set_error("hqdn3d_create: unsupported geometry %dx%d depth %d", cfg->width, cfg->height, cfg->depth);
        return -1;
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || cfg->device < 0 || cfg->device >= ndev)
    {
        cudaGetLastError();
        set_error("hqdn3d_create: CUDA device %d not available (%d devices); there is no CPU fallback", cfg->device, ndev);
        return -1;
    }
    HBCU_CHECK(cudaSetDevice(cfg->device));
    cudaDeviceProp prop;
    HBCU_CHECK(cudaGetDeviceProperties(&prop, cfg->device));
    if (prop.major != 9 || prop.minor != 0)
    {
        set_error("hqdn3d_create: device %d is sm_%d%d; this library is built for sm_90a only", cfg->device, prop.major, prop.minor);
        return -1;
    }
    hbcu_hqdn3d_s *h = new (std::nothrow) hbcu_hqdn3d_s();
    if (h == nullptr) { set_error("hqdn3d_create: out of memory"); return -1; }
    h->cfg = *cfg;
    h->bps = cfg->depth > 8 ? 2 : 1;
    h->slots = cfg->slots >= 2 ? cfg->slots : 4;
    h->next = 0;
    h->half = 256 << (cfg->depth == 16 ? 8 : 4);             // LUT_BITS, denoise.c:30
    h->s_h2d = h->s_compute = h->s_d2h = nullptr;
    h->ev_mark[0] = h->ev_mark[1] = nullptr;
    h->ev_fork = nullptr;
    for (int pl = 0; pl < 3; pl++) { h->s_pl[pl] = nullptr; h->ev_join[pl] = nullptr; }
    for (int i = 0; i < 6; i++) h->d_coef[i] = nullptr;
    for (int pl = 0; pl < 3; pl++)
    {
        h->d_ant[pl] = h->d_h[pl] = nullptr;
        h->first[pl] = 1;
        h->spatial[pl] = cfg->coef[2 * pl][0] != 0;         // ct[0] = !!dist25 (denoise.c:93, :192)
        Geom &g = h->g[pl];
        g.w = pl == 0 ? cfg->width : -((-cfg->width) >> cfg->chroma_shift_w);
        g.h = pl == 0 ? cfg->height : -((-cfg->height) >> cfg->chroma_shift_h);
        g.pitch = ((g.w * h->bps + 63) / 64 * 64) / h->bps;
        g.bytes = (size_t)g.pitch * g.h * h->bps;
        h->plane_off[pl] = pl == 0 ? 0 : h->plane_off[pl - 1] + h->g[pl - 1].bytes;
        h->frame_bytes = h->plane_off[pl] + g.bytes;
    }
#define CK(expr)                                                                  \
    do {                                                                          \
        cudaError_t _e = (expr);                                                  \
        if (_e != cudaSuccess) {                                                  \
            set_error("%s failed: %s", #expr, cudaGetErrorString(_e));            \
            hbcu_hqdn3d_destroy(h);                                               \
            return -1;                                                            \
        }                                                                         \
    } while (0)
    CK(cudaStreamCreateWithFlags(&h->s_h2d, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&h->s_compute, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&h->s_d2h, cudaStreamNonBlocking));
    CK(cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming));
    for (int pl = 0; pl < 3; pl++)
    {
        CK(cudaStreamCreateWithFlags(&h->s_pl[pl], cudaStreamNonBlocking));
        CK(cudaEventCreateWithFlags(&h->ev_join[pl], cudaEventDisableTiming));
    }
    for (int i = 0; i < 6; i++)
    {
        CK(cudaMalloc(&h->d_coef[i], (size_t)2 * h->half * sizeof(int16_t)));
        CK(cudaMemcpy(h->d_coef[i], cfg->coef[i], (size_t)2 * h->half * sizeof(int16_t), cudaMemcpyHostToDevice));
        h->cfg.coef[i] = nullptr;                           // the caller's tables are not kept
    }
    if (cfg->depth < 16)
    {
        // per device (a second handle on another GPU needs its own opt-in)
        const int v2smem = 4 * h->half * (int)sizeof(int16_t) + 3 * 32 * kTilePitch;
        CK(cudaFuncSetAttribute(hqdn3d_vt2_kernel<uint8_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, v2smem));
        CK(cudaFuncSetAttribute(hqdn3d_vt2_kernel<uint16_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, v2smem));
        CK(cudaFuncSetAttribute(hqdn3d_h2_kernel<uint8_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, v2smem));
        CK(cudaFuncSetAttribute(hqdn3d_h2_kernel<uint16_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, v2smem));
    }
    if (cfg->depth < 16)
    {
        const int lut = 4 * h->half * (int)sizeof(int16_t);
        if (lut > 48 * 1024)
        {
            CK(cudaFuncSetAttribute(hqdn3d_vt_kernel<uint8_t, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, lut));
            CK(cudaFuncSetAttribute(hqdn3d_vt_kernel<uint8_t, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, lut));
            CK(cudaFuncSetAttribute(hqdn3d_vt_kernel<uint16_t, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, lut));
            CK(cudaFuncSetAttribute(hqdn3d_vt_kernel<uint16_t, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, lut));
        }
    }
    for (int pl = 0; pl < 3; pl++)
    {
        CK(cudaMalloc(&h->d_ant[pl], (size_t)h->g[pl].w * h->g[pl].h * sizeof(uint16_t)));
        CK(cudaMalloc(&h->d_h[pl], (size_t)h->g[pl].w * h->g[pl].h * sizeof(uint16_t)));
    }
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

void hbcu_hqdn3d_destroy(hbcu_hqdn3d_t *h)
{
    if (h == nullptr) return;
    cudaSetDevice(h->cfg.device);
    cudaDeviceSynchronize();
    for (auto p : h->in_base) if (p) cudaFree(p);
    for (auto p : h->out_base) if (p) cudaFree(p);
    for (int i = 0; i < 6; i++) if (h->d_coef[i]) cudaFree(h->d_coef[i]);
    for (int pl = 0; pl < 3; pl++) { if (h->d_ant[pl]) cudaFree(h->d_ant[pl]); if (h->d_h[pl]) cudaFree(h->d_h[pl]); }
    for (auto e : h->ev_up) if (e) cudaEventDestroy(e);
    for (auto e : h->ev_k) if (e) cudaEventDestroy(e);
    for (auto e : h->ev_down) if (e) cudaEventDestroy(e);
    if (h->ev_mark[0]) cudaEventDestroy(h->ev_mark[0]);
    if (h->ev_mark[1]) cudaEventDestroy(h->ev_mark[1]);
    if (h->ev_fork) cudaEventDestroy(h->ev_fork);
    for (int pl = 0; pl < 3; pl++)
    {
        if (h->ev_join[pl]) cudaEventDestroy(h->ev_join[pl]);
        if (h->s_pl[pl]) cudaStreamDestroy(h->s_pl[pl]);
    }
    if (h->s_h2d) cudaStreamDestroy(h->s_h2d);
    if (h->s_compute) cudaStreamDestroy(h->s_compute);
    if (h->s_d2h) cudaStreamDestroy(h->s_d2h);
    delete h;
}

// frames MUST be submitted in display order: the temporal state makes every frame depend on the previous one
int hbcu_hqdn3d_filter_frames(hbcu_hqdn3d_t *h, int64_t ticket,
                              hbcu_frame_t *in_frame, const void *const in_planes[3], const int in_strides[3],
                              hbcu_frame_t *out_frame, void *const out_planes[3], const int out_strides[3])
{
    if (h == nullptr || (in_frame == nullptr && (in_planes == nullptr || in_strides == nullptr)) ||
        (out_frame == nullptr && (out_planes == nullptr || out_strides == nullptr)) ||
        (in_frame && !frame_fits(h, in_frame)) || (out_frame && !frame_fits(h, out_frame)))
    {
        set_error("hqdn3d_filter_frames: bad argument or frame geometry");
        return -1;
    }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    const int s = h->next;
    h->next = (h->next + 1) % h->slots;
    if (in_frame == nullptr)
    {
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
    // fork: every plane on its own stream (stream order per plane also chains the plane's temporal state frame to frame)
    HBCU_CHECK(cudaEventRecord(h->ev_fork, h->s_compute));
    for (int pl = 0; pl < 3; pl++)
    {
        const void *src = in_frame ? (const void *)in_frame->plane[pl] : (const void *)(h->in_base[s] + h->plane_off[pl]);
        void *dst = out_frame ? (void *)out_frame->plane[pl] : (void *)(h->out_base[s] + h->plane_off[pl]);
        HBCU_CHECK(cudaStreamWaitEvent(h->s_pl[pl], h->ev_fork, 0));
        const int rc = h->bps == 1 ? launch_plane_t<uint8_t>(h, pl, src, dst, h->s_pl[pl]) : launch_plane_t<uint16_t>(h, pl, src, dst, h->s_pl[pl]);
        if (rc != 0) return -1;
        HBCU_CHECK(cudaEventRecord(h->ev_join[pl], h->s_pl[pl]));
        HBCU_CHECK(cudaStreamWaitEvent(h->s_compute, h->ev_join[pl], 0));
    }
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

int hbcu_hqdn3d_wait(hbcu_hqdn3d_t *h, int64_t ticket)
{
    if (h == nullptr) { set_error("hqdn3d_wait: null handle"); return -1; }
    const int s = find_slot(h, ticket);
    if (s < 0) { set_error("hqdn3d_wait: ticket %lld is not in flight", (long long)ticket); return -1; }
    HBCU_CHECK(cudaEventSynchronize(h->ev_down[s]));
    return 0;
}

int hbcu_hqdn3d_poll(hbcu_hqdn3d_t *h, int64_t ticket)
{
    if (h == nullptr) { set_error("hqdn3d_poll: null handle"); return -1; }
    const int s = find_slot(h, ticket);
    if (s < 0) { set_error("hqdn3d_poll: ticket %lld is not in flight", (long long)ticket); return -1; }
    cudaError_t e = cudaEventQuery(h->ev_down[s]);
    if (e == cudaSuccess) return 1;
    if (e == cudaErrorNotReady) return 0;
    set_error("hqdn3d_poll: %s", cudaGetErrorString(e));
    return -1;
}

int hbcu_hqdn3d_sync(hbcu_hqdn3d_t *h)
{
    if (h == nullptr) { set_error("hqdn3d_sync: null handle"); return -1; }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    HBCU_CHECK(cudaStreamSynchronize(h->s_h2d));
    for (int pl = 0; pl < 3; pl++) HBCU_CHECK(cudaStreamSynchronize(h->s_pl[pl]));
    HBCU_CHECK(cudaStreamSynchronize(h->s_compute));
    HBCU_CHECK(cudaStreamSynchronize(h->s_d2h));
    return 0;
}

int hbcu_hqdn3d_mark(hbcu_hqdn3d_t *h, int which)
{
    if (h == nullptr || which < 0 || which > 1) { set_error("hqdn3d_mark: bad argument"); return -1; }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    HBCU_CHECK(cudaEventRecord(h->ev_mark[which], h->s_compute));
    return 0;
}

int hbcu_hqdn3d_elapsed_ms(hbcu_hqdn3d_t *h, float *ms)
{
    if (h == nullptr || ms == nullptr) { set_error("hqdn3d_elapsed_ms: bad argument"); return -1; }
    HBCU_CHECK(cudaEventSynchronize(h->ev_mark[1]));
    HBCU_CHECK(cudaEventElapsedTime(ms, h->ev_mark[0], h->ev_mark[1]));
    return 0;
}

}  // extern "C"
