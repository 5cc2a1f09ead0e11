// decomb.cu -- decomb (yadif / cubic / blend line filters, bob, per-frame mode) for sm_90a
// behind the C-ABI of include/hbcu.h.
//
// Replaces (reference: HandBrake's libhb):
//   cubic_interpolate_pixel/line  templates/decomb_template.c:43-107
//   blend_filter_pixel/line       templates/decomb_template.c:279-361
//   yadif_filter_line/YADIF_CHECK templates/decomb_template.c:482-710
//   yadif_decomb_filter_work      templates/decomb_template.c:714-808   (cpu_count row segments)
//   filter_{8,16}                 templates/decomb_template.c:810-898
// The reference splits every plane into cpu_count row segments joined by a taskset barrier; rows
// are independent, so here one kernel covers a whole plane: a thread produces four adjacent
// output pixels of one row (kept rows are straight copies, rebuilt rows run the line filter).
// Integer arithmetic only -> bit-exact.  The kernel is HBM-bound: it reads the three input
// frames once (rows are re-touched through L1/L2) and writes one.
#include "hbcu_common.h"
#include "hbcu_frames.h"
#include "../../include/hbcu.h"
#include "eedi2.cuh"

#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>

namespace {

using hbcu::set_error;

struct FieldParams
{
    const void *prev, *cur, *next;   // plane base pointers
    const void *eedi;                // EEDI2 full-height interpolation of this plane or nullptr
    void *dst;
    int w, h;
    int pitch;                       // input planes, elements
    int dpitch;                      // output plane, elements
    int epitch;
    int mode;                        // per-frame mode (EEDI2 bit kept: selects the spatial predictor)
    int parity, tff;
    int maxv;
};

__device__ __forceinline__ int crop(int v, int maxv) { return min(max(v, 0), maxv); }

// template :43-49 (C division truncates toward zero, as does CUDA's)
__device__ __forceinline__ int cubic_px(int maxv, int y0, int y1, int y2, int y3)
{
    const int r = (y0 * -3) + (y1 * 23) + (y2 * 23) + (y3 * -3);
    return crop(r / 40, maxv);
}

template <typename PIX>
__device__ __forceinline__ int cubic_line_px(const PIX *c, int pitch, int h, int x, int y, int maxv)
{
    const PIX *p = c + (size_t)y * pitch + x;
    int a = 0, b = 0, cc = 0, d = 0;
    if (y >= 3)                { a = p[-3 * pitch]; b = p[-pitch]; }
    else if (y == 2 || y == 1) { a = p[-pitch]; b = a; }
    else if (y == 0)           { a = p[pitch]; b = a; }
    if (y <= h - 4)                     { cc = p[pitch]; d = p[3 * pitch]; }
    else if (y == h - 3 || y == h - 2)  { cc = p[pitch]; d = cc; }
    else if (y == h - 1)                { cc = p[-pitch]; d = cc; }
    return cubic_px(maxv, a, b, cc, d);
}

template <typename PIX>
__device__ __forceinline__ int blend_line_px(const PIX *c, int pitch, int h, int x, int y, int maxv)
{
    const PIX *p = c + (size_t)y * pitch + x;
    int u1, u2, d1, d2;
    if (y > 1 && y < h - 2) { u1 = -pitch; u2 = -2 * pitch; d1 = pitch; d2 = 2 * pitch; }
    else if (y == 0)        { u1 = u2 = 0; d1 = pitch; d2 = 2 * pitch; }
    else if (y == 1)        { u1 = u2 = -pitch; d1 = pitch; d2 = 2 * pitch; }
    else if (y == h - 2)    { u1 = -pitch; u2 = -2 * pitch; d1 = d2 = pitch; }
    else                    { u1 = -pitch; u2 = -2 * pitch; d1 = d2 = 0; }
    int r = -(int)p[u2] + 2 * (int)p[u1] + 6 * (int)p[0] + 2 * (int)p[d1] - (int)p[d2];
    r >>= 3;
    return crop(r, maxv);
}

template <typename PIX>
__device__ __forceinline__ int yadif_px(const FieldParams &fp, int x, int y)
{
    const PIX *prev = (const PIX *)fp.prev, *cur = (const PIX *)fp.cur, *next = (const PIX *)fp.next;
    const int pitch = fp.pitch, w = fp.w, h = fp.h, maxv = fp.maxv;
    const int par = fp.parity ^ fp.tff;
    const PIX *prev2 = par ? prev : cur, *next2 = par ? cur : next;
    const int sp = y ? -pitch : pitch;                       // mirrored at the first / last line
    const int sn = y + 1 < h ? pitch : -pitch;
    const bool vertical_edge = (y < 3) || (y > h - 4);
    const bool cubic = (fp.mode & HBCU_DECOMB_CUBIC) != 0;
    const int margin = cubic ? 3 : 2;
    const size_t o = (size_t)y * pitch + x;

    const int c = cur[o + sp];
    const int p2 = prev2[o], n2 = next2[o];
    const int d = (p2 + n2) >> 1;
    const int e = cur[o + sn];
    const int td0 = abs(p2 - n2);
    const int td1 = (abs((int)prev[o + sp] - c) + abs((int)prev[o + sn] - e)) >> 1;
    const int td2 = (abs((int)next[o + sp] - c) + abs((int)next[o + sn] - e)) >> 1;
    int diff = max(max(td0 >> 1, td1), td2);
    int spatial_pred;

    if (fp.eedi != nullptr)
    {
        spatial_pred = ((const PIX *)fp.eedi)[(size_t)y * fp.epitch + x];
    }
    else
    {
        const PIX *q = cur + o;
        if (cubic && !vertical_edge)
            spatial_pred = cubic_px(maxv, q[-3 * pitch], q[-pitch], q[pitch], q[3 * pitch]);
        else
            spatial_pred = (c + e) >> 1;
        if (x > margin && x < w - (margin + 1))
        {
            int score = abs((int)q[sp - 1] - (int)q[sn - 1]) + abs(c - e) + abs((int)q[sp + 1] - (int)q[sn + 1]) - 1;
#pragma unroll
            for (int dir = -1; dir <= 1; dir += 2)
            {
#pragma unroll
                for (int step = 1; step <= 2; step++)
                {
                    const int j = dir * step;
                    const int s = abs((int)q[sp - 1 + j] - (int)q[sn - 1 - j]) + abs((int)q[sp + j] - (int)q[sn - j]) +
                                  abs((int)q[sp + 1 + j] - (int)q[sn + 1 - j]);
                    if (!(s < score)) break;                 // the +-2 probe lives inside a successful +-1 probe
                    score = s;
                    if (cubic && !vertical_edge)
                    {
                        if (step == 1)
                            spatial_pred = cubic_px(maxv, q[-3 * pitch + 3 * j], q[-pitch + j], q[pitch - j], q[3 * pitch - 3 * j]);
                        else
                            spatial_pred = cubic_px(maxv, ((int)q[-3 * pitch + 2 * j] + (int)q[-pitch + 2 * j]) / 2, q[-pitch + j],
                                                    q[pitch - j], ((int)q[3 * pitch - 2 * j] + (int)q[pitch - 2 * j]) / 2);
                    }
                    else
                    {
                        spatial_pred = ((int)q[sp + j] + (int)q[sn - j]) >> 1;
                    }
                }
            }
        }
    }
    if (!vertical_edge)
    {
        const int b = ((int)prev2[o - 2 * pitch] + (int)next2[o - 2 * pitch]) >> 1;
        const int f = ((int)prev2[o + 2 * pitch] + (int)next2[o + 2 * pitch]) >> 1;
        const int mx = max(max(d - e, d - c), min(b - c, f - e));
        const int mn = min(min(d - e, d - c), max(b - c, f - e));
        diff = max(max(diff, mn), -mx);
    }
    if (spatial_pred > d + diff) spatial_pred = d + diff;
    else if (spatial_pred < d - diff) spatial_pred = d - diff;
    return spatial_pred;
}

// 4 / 12 consecutive samples starting at a 4-sample-aligned position, as one or three vector loads
template <typename PIX> __device__ __forceinline__ void load4(const PIX *__restrict__ p, int *v);
template <> __device__ __forceinline__ void load4<uint8_t>(const uint8_t *__restrict__ p, int *v)
{
    const uchar4 t = *reinterpret_cast<const uchar4 *>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
template <> __device__ __forceinline__ void load4<uint16_t>(const uint16_t *__restrict__ p, int *v)
{
    const ushort4 t = *reinterpret_cast<const ushort4 *>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
template <typename PIX> __device__ __forceinline__ void load12(const PIX *__restrict__ p, int *v)
{
    load4<PIX>(p, v); load4<PIX>(p + 4, v + 4); load4<PIX>(p + 8, v + 8);
}

// yadif for the 4 pixels x0..x0+3 of row y, everything read once into registers (same arithmetic as
// yadif_px, which stays the reference formulation and handles the groups next to the left/right edge).
// Requires 4 <= x0 and x0 + 8 <= w.
// CUBIC / EEDI: fp.mode & HBCU_DECOMB_CUBIC and fp.eedi != nullptr, known per launch -- as run-time values both sides of every
// `use_cubic` / `eedi` choice were compiled into the pixel loop as predicated code
template <typename PIX, bool CUBIC, bool EEDI>
__device__ __forceinline__ void yadif_px4(const FieldParams &fp, int x0, int y, int *out)
{
    const PIX *prev = (const PIX *)fp.prev, *cur = (const PIX *)fp.cur, *next = (const PIX *)fp.next;
    const int pitch = fp.pitch, w = fp.w, h = fp.h, maxv = fp.maxv;
    const int par = fp.parity ^ fp.tff;
    const PIX *prev2 = par ? prev : cur, *next2 = par ? cur : next;
    const int yp = y ? y - 1 : y + 1, yn = y + 1 < h ? y + 1 : y - 1;
    const bool vertical_edge = (y < 3) || (y > h - 4);
    constexpr bool cubic = CUBIC;
    constexpr int margin = cubic ? 3 : 2;
    const int o = y * pitch + x0, op = yp * pitch + x0, on = yn * pitch + x0;

    int P[12], N[12], A[12], D[12];                   // cur rows yp, yn, y-3, y+3 over x0-4 .. x0+7
    load12<PIX>(cur + op - 4, P);
    load12<PIX>(cur + on - 4, N);
    const bool use_cubic = cubic && !vertical_edge && !EEDI;
    if (use_cubic)
    {
        load12<PIX>(cur + o - 3 * pitch - 4, A);
        load12<PIX>(cur + o + 3 * pitch - 4, D);
    }
    int p2[4], n2[4], pp[4], pn[4], np_[4], nn[4], b2p[4], b2n[4], f2p[4], f2n[4], ee[4];
    load4<PIX>(prev2 + o, p2);
    load4<PIX>(next2 + o, n2);
    load4<PIX>(prev + op, pp);
    load4<PIX>(prev + on, pn);
    load4<PIX>(next + op, np_);
    load4<PIX>(next + on, nn);
    if (!vertical_edge)
    {
        load4<PIX>(prev2 + o - 2 * pitch, b2p);
        load4<PIX>(next2 + o - 2 * pitch, b2n);
        load4<PIX>(prev2 + o + 2 * pitch, f2p);
        load4<PIX>(next2 + o + 2 * pitch, f2n);
    }
    if (EEDI) load4<PIX>((const PIX *)fp.eedi + y * fp.epitch + x0, ee);

#pragma unroll
    for (int i = 0; i < 4; i++)
    {
        const int x = x0 + i, li = 4 + i;
        const int c = P[li], e = N[li];
        const int d = (p2[i] + n2[i]) >> 1;
        const int td0 = abs(p2[i] - n2[i]);
        const int td1 = (abs(pp[i] - c) + abs(pn[i] - e)) >> 1;
        const int td2 = (abs(np_[i] - c) + abs(nn[i] - e)) >> 1;
        int diff = max(max(td0 >> 1, td1), td2);
        int spatial_pred;
        if (EEDI)
        {
            spatial_pred = ee[i];
        }
        else
        {
            if (use_cubic) spatial_pred = cubic_px(maxv, A[li], P[li], N[li], D[li]);
            else           spatial_pred = (c + e) >> 1;
            if (x > margin && x < w - (margin + 1))
            {
                int score = abs(P[li - 1] - N[li - 1]) + abs(c - e) + abs(P[li + 1] - N[li + 1]) - 1;
#pragma unroll
                for (int dir = -1; dir <= 1; dir += 2)
                {
                    bool go = true;
#pragma unroll
                    for (int step = 1; step <= 2; step++)
                    {
                        const int j = dir * step;
                        const int sc = abs(P[li - 1 + j] - N[li - 1 - j]) + abs(P[li + j] - N[li - j]) + abs(P[li + 1 + j] - N[li + 1 - j]);
                        go = go && (sc < score);
                        if (go)
                        {
                            score = sc;
                            if (use_cubic)
                            {
                                if (step == 1) spatial_pred = cubic_px(maxv, A[li + 3 * j], P[li + j], N[li - j], D[li - 3 * j]);
                                else           spatial_pred = cubic_px(maxv, (A[li + 2 * j] + P[li + 2 * j]) / 2, P[li + j], N[li - j],
                                                                       (D[li - 2 * j] + N[li - 2 * j]) / 2);
                            }
                            else
                                spatial_pred = (P[li + j] + N[li - j]) >> 1;
                        }
                    }
                }
            }
        }
        if (!vertical_edge)
        {
            const int b = (b2p[i] + b2n[i]) >> 1, f = (f2p[i] + f2n[i]) >> 1;
            const int mx = max(max(d - e, d - c), min(b - c, f - e));
            const int mn = min(min(d - e, d - c), max(b - c, f - e));
            diff = max(max(diff, mn), -mx);
        }
        if (spatial_pred > d + diff) spatial_pred = d + diff;
        else if (spatial_pred < d - diff) spatial_pred = d - diff;
        out[i] = spatial_pred;
    }
}

// one thread = 4 adjacent pixels of two consecutive output rows (one kept, one rebuilt): every warp carries the same
// amount of work.  With one row per thread half of the warps (kept rows) retire at once and the SM runs at half its
// already register-limited occupancy.
template <typename PIX, bool CUBIC, bool EEDI>
__device__ __forceinline__ void decomb_row4(const FieldParams &fp, int x0, int y)
{
    const PIX *cur = (const PIX *)fp.cur;
    PIX *dst = (PIX *)fp.dst + (size_t)y * fp.dpitch;
    const bool filtered = fp.parity ? !(y & 1) : (y & 1);     // template :744, :796
    int v[4];
    if (filtered && fp.mode != HBCU_DECOMB_BLEND && fp.mode != HBCU_DECOMB_CUBIC && (fp.mode & HBCU_DECOMB_YADIF) &&
        x0 >= 4 && x0 + 8 <= fp.w)
    {
        yadif_px4<PIX, CUBIC, EEDI>(fp, x0, y, v);
        if (sizeof(PIX) == 1) *reinterpret_cast<uchar4 *>(dst + x0) = make_uchar4(v[0], v[1], v[2], v[3]);
        else                  *reinterpret_cast<ushort4 *>(dst + x0) = make_ushort4(v[0], v[1], v[2], v[3]);
        return;
    }
    if (!filtered && x0 + 3 < fp.w)
    {
        // kept rows are straight copies: one vector load, one vector store
        if (sizeof(PIX) == 1) *reinterpret_cast<uchar4 *>(dst + x0) = *reinterpret_cast<const uchar4 *>(cur + (size_t)y * fp.pitch + x0);
        else                  *reinterpret_cast<ushort4 *>(dst + x0) = *reinterpret_cast<const ushort4 *>(cur + (size_t)y * fp.pitch + x0);
        return;
    }
#pragma unroll
    for (int i = 0; i < 4; i++)
    {
        const int x = min(x0 + i, fp.w - 1);
        if (!filtered)                           v[i] = cur[(size_t)y * fp.pitch + x];
        else if (fp.mode == HBCU_DECOMB_BLEND)   v[i] = blend_line_px<PIX>(cur, fp.pitch, fp.h, x, y, fp.maxv);
        else if (fp.mode == HBCU_DECOMB_CUBIC)   v[i] = cubic_line_px<PIX>(cur, fp.pitch, fp.h, x, y, fp.maxv);
        else if (fp.mode & HBCU_DECOMB_YADIF)    v[i] = yadif_px<PIX>(fp, x, y);
        else                                     v[i] = 0;    // no line filter runs: a fresh (zeroed) buffer row
    }
    if (x0 + 3 < fp.w)
    {
        if (sizeof(PIX) == 1) *reinterpret_cast<uchar4 *>(dst + x0) = make_uchar4(v[0], v[1], v[2], v[3]);
        else                  *reinterpret_cast<ushort4 *>(dst + x0) = make_ushort4(v[0], v[1], v[2], v[3]);
    }
    else
    {
        for (int i = 0; i < 4; i++)
            if (x0 + i < fp.w) dst[x0 + i] = (PIX)v[i];
    }
}

template <typename PIX, int MINB, bool CUBIC, bool EEDI>
__global__ void __launch_bounds__(256, MINB) decomb_field_kernel(FieldParams fp)
{
    const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    const int y0 = (blockIdx.y * blockDim.y + threadIdx.y) * 2;
    if (x0 >= fp.w || y0 >= fp.h) return;
    decomb_row4<PIX, CUBIC, EEDI>(fp, x0, y0);
    if (y0 + 1 < fp.h) decomb_row4<PIX, CUBIC, EEDI>(fp, x0, y0 + 1);
}

template <typename PIX>
__global__ void __launch_bounds__(256) copy_rows_kernel(const PIX *__restrict__ src, int spitch, PIX *__restrict__ dst, int dpitch, int w, int h)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x < w && y < h) dst[(size_t)y * dpitch + x] = src[(size_t)y * spitch + x];
}

struct Geom { int w, h, pitch; size_t bytes; };

}  // namespace

struct hbcu_decomb_s
{
    hbcu_decomb_config_t cfg;
    int bps, maxv;
    Geom g[3];
    int slots, out_slots;
    std::vector<uint8_t *> in_base, out_base;   // one allocation per frame, planes back to back at the reference stride:
    size_t frame_bytes, plane_off[3];            // the layout of a STANDARD hb_buffer_t, so a frame moves as one copy
    std::vector<uint8_t *> in_mem;       // [slot*3+plane]
    std::vector<int64_t> in_index;
    std::vector<cudaEvent_t> ev_upload, ev_readers;
    std::vector<uint8_t *> out_mem;      // [oslot*3+plane]
    std::vector<int64_t> out_ticket;
    std::vector<cudaEvent_t> ev_kernel, ev_d2h;
    int next_out;
    hbcu::Eedi2 *eedi;                   // EEDI2 state (mask carry-over) + scratch, one per handle
    cudaStream_t s_h2d, s_compute, s_d2h;
    cudaStream_t s_chroma[2];            // chroma field kernels run beside luma's (forked from / joined to s_compute)
    cudaEvent_t ev_fork, ev_join[2];
    cudaEvent_t ev_mark[2];
};

namespace {

int run_field(hbcu_decomb_s *h, int64_t ticket, int64_t prev, int64_t cur, int64_t next, int frame_mode, int parity, int tff, int oslot,
              uint8_t *const *ext_dst = nullptr)
{
    const int64_t idx[3] = { prev, cur, next };
    int slot[3];
    for (int k = 0; k < 3; k++)
    {
        slot[k] = (int)(idx[k] % h->slots);
        if (idx[k] < 0 || h->in_index[slot[k]] != idx[k])
        {
            set_error("decomb: frame %lld is not resident", (long long)idx[k]);
            return -1;
        }
        HBCU_CHECK(cudaStreamWaitEvent(h->s_compute, h->ev_upload[slot[k]], 0));
    }
    HBCU_CHECK(cudaStreamWaitEvent(h->s_compute, h->ev_d2h[oslot], 0));
    const bool use_eedi = (frame_mode & HBCU_DECOMB_EEDI2) != 0;
    if (use_eedi)
    {
        if (h->eedi == nullptr)
        {
            set_error("decomb: EEDI2 requested but the handle was created without mode bit 8");
            return -1;
        }
        // eedi2_planer (decomb template :455-473): field `!tff_eedi` of cur, tff_eedi = !parity (decomb.c:539-542)
        const void *planes[3] = { h->in_mem[slot[1] * 3 + 0], h->in_mem[slot[1] * 3 + 1], h->in_mem[slot[1] * 3 + 2] };
        if (hbcu::eedi2_run(h->eedi, planes, !parity, h->s_compute) != 0) return -1;
    }
    HBCU_CHECK(cudaEventRecord(h->ev_fork, h->s_compute));
    for (int pl = 0; pl < 3; pl++)
    {
        cudaStream_t st = pl == 0 ? h->s_compute : h->s_chroma[pl - 1];
        if (pl > 0) HBCU_CHECK(cudaStreamWaitEvent(st, h->ev_fork, 0));
        const Geom &g = h->g[pl];
        uint8_t *dst = ext_dst ? ext_dst[pl] : h->out_mem[oslot * 3 + pl];     // external planes share the reference stride
        if (frame_mode == 0 || (use_eedi && !(frame_mode & HBCU_DECOMB_YADIF)))
        {
            // pass-through (hb_buffer_copy) or "just EEDI2": whole-plane copy (decomb template :855-875, :893-896)
            const uint8_t *src = frame_mode == 0 ? h->in_mem[slot[1] * 3 + pl] : (const uint8_t *)hbcu::eedi2_output(h->eedi, pl);
            dim3 blk(64, 4), grid((g.w + 63) / 64, (g.h + 3) / 4);
            if (h->bps == 1) copy_rows_kernel<uint8_t><<<grid, blk, 0, st>>>(src, g.pitch, dst, g.pitch, g.w, g.h);
            else copy_rows_kernel<uint16_t><<<grid, blk, 0, st>>>((const uint16_t *)src, g.pitch, (uint16_t *)dst, g.pitch, g.w, g.h);
            hbcu::count_launch();
            HBCU_CHECK(cudaGetLastError());
            if (pl > 0) HBCU_CHECK(cudaEventRecord(h->ev_join[pl - 1], st));
            continue;
        }
        FieldParams fp;
        fp.prev = h->in_mem[slot[0] * 3 + pl];
        fp.cur  = h->in_mem[slot[1] * 3 + pl];
        fp.next = h->in_mem[slot[2] * 3 + pl];
        fp.eedi = use_eedi ? hbcu::eedi2_output(h->eedi, pl) : nullptr;
        fp.dst = dst;
        fp.w = g.w; fp.h = g.h; fp.pitch = g.pitch; fp.dpitch = g.pitch; fp.epitch = g.pitch;
        fp.mode = frame_mode; fp.parity = parity; fp.tff = tff; fp.maxv = h->maxv;
        dim3 blk(64, 4), grid(((g.w + 3) / 4 + 63) / 64, ((g.h + 1) / 2 + 3) / 4);   // 4 px x 2 rows per thread
        // 3 resident CTAs per SM (register cap 85) measured best of 2 / 3 / 4 in round 1
        const bool cub = (frame_mode & HBCU_DECOMB_CUBIC) != 0, ee = fp.eedi != nullptr;
#define FIELD(PIX)                                                                                          \
        do {                                                                                                \
            if (cub && ee)       decomb_field_kernel<PIX, 3, true, true><<<grid, blk, 0, st>>>(fp);    \
            else if (cub)        decomb_field_kernel<PIX, 3, true, false><<<grid, blk, 0, st>>>(fp);   \
            else if (ee)         decomb_field_kernel<PIX, 3, false, true><<<grid, blk, 0, st>>>(fp);   \
            else                 decomb_field_kernel<PIX, 3, false, false><<<grid, blk, 0, st>>>(fp);  \
        } while (0)
        if (h->bps == 1) FIELD(uint8_t);
        else             FIELD(uint16_t);
#undef FIELD
        hbcu::count_launch();
        HBCU_CHECK(cudaGetLastError());
        if (pl > 0) HBCU_CHECK(cudaEventRecord(h->ev_join[pl - 1], st));
    }
    for (int i = 0; i < 2; i++) HBCU_CHECK(cudaStreamWaitEvent(h->s_compute, h->ev_join[i], 0));
    HBCU_CHECK(cudaEventRecord(h->ev_kernel[oslot], h->s_compute));
    // prev leaves the window once the last field of this frame is done; recording after every field is harmless
    HBCU_CHECK(cudaEventRecord(h->ev_readers[slot[0]], h->s_compute));
    h->out_ticket[oslot] = ticket;
    return 0;
}

int find_ticket(hbcu_decomb_s *h, int64_t ticket)
{
    for (int s = 0; s < h->out_slots; s++)
        if (h->out_ticket[s] == ticket) return s;
    return -1;
}

}  // namespace

extern "C" {

int hbcu_decomb_create(hbcu_decomb_t **out, const hbcu_decomb_config_t *cfg)
{
    if (out == nullptr || cfg == nullptr) { set_error("decomb_create: null argument"); return -1; }
    *out = nullptr;
    if (cfg->width < 8 || cfg->height < 8 || cfg->depth < 8 || cfg->depth > 16)
    {
        set_error("decomb_create: unsupported geometry %dx%d depth %d", cfg->width, cfg->height, cfg->depth);
        return -1;
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || cfg->device < 0 || cfg->device >= ndev)
    {
        cudaGetLastError();
        set_error("decomb_create: CUDA device %d not available (%d devices); there is no CPU fallback", cfg->device, ndev);
        return -1;
    }
    HBCU_CHECK(cudaSetDevice(cfg->device));
    hbcu_decomb_s *h = new (std::nothrow) hbcu_decomb_s();
    if (h == nullptr) { set_error("decomb_create: out of memory"); return -1; }
    h->cfg = *cfg;
    h->bps = cfg->depth > 8 ? 2 : 1;
    h->maxv = (1 << cfg->depth) - 1;
    h->slots = cfg->slots >= 4 ? cfg->slots : 4;
    h->out_slots = cfg->out_slots >= 2 ? cfg->out_slots : 4;
    h->next_out = 0;
    h->eedi = nullptr;
    h->s_h2d = h->s_compute = h->s_d2h = nullptr;
    h->s_chroma[0] = h->s_chroma[1] = nullptr;
    h->ev_fork = h->ev_join[0] = h->ev_join[1] = nullptr;
    h->ev_mark[0] = h->ev_mark[1] = nullptr;
    for (int pl = 0; pl < 3; pl++)
    {
        Geom &g = h->g[pl];
        g.w = pl == 0 ? cfg->width : -((-cfg->width) >> cfg->chroma_shift_w);
        g.h = pl == 0 ? cfg->height : -((-cfg->height) >> cfg->chroma_shift_h);
        // the reference's planes have stride == hb_image_stride (64-byte multiple); EEDI2 reads across row ends
        // (SURVEY.md 8a/a26), so the device pitch reproduces exactly that stride
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
            hbcu_decomb_destroy(h);                                               \
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
    h->in_mem.assign(h->slots * 3, nullptr);
    h->in_base.assign(h->slots, nullptr);
    h->out_base.assign(h->out_slots, nullptr);
    h->in_index.assign(h->slots, -1);
    h->ev_upload.assign(h->slots, nullptr);
    h->ev_readers.assign(h->slots, nullptr);
    h->out_mem.assign(h->out_slots * 3, nullptr);
    h->out_ticket.assign(h->out_slots, -1);
    h->ev_kernel.assign(h->out_slots, nullptr);
    h->ev_d2h.assign(h->out_slots, nullptr);
    for (int s = 0; s < h->slots; s++)
    {
        CK(cudaEventCreateWithFlags(&h->ev_upload[s], cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&h->ev_readers[s], cudaEventDisableTiming));
        CK(cudaMalloc(&h->in_base[s], h->frame_bytes));
        CK(cudaMemset(h->in_base[s], 0, h->frame_bytes));
        for (int pl = 0; pl < 3; pl++) h->in_mem[s * 3 + pl] = h->in_base[s] + h->plane_off[pl];
    }
    for (int s = 0; s < h->out_slots; s++)
    {
        CK(cudaEventCreateWithFlags(&h->ev_kernel[s], cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&h->ev_d2h[s], cudaEventDisableTiming));
        CK(cudaMalloc(&h->out_base[s], h->frame_bytes));
        CK(cudaMemset(h->out_base[s], 0, h->frame_bytes));          // the stride padding is never written
        for (int pl = 0; pl < 3; pl++) h->out_mem[s * 3 + pl] = h->out_base[s] + h->plane_off[pl];
    }
    CK(cudaEventCreate(&h->ev_mark[0]));
    CK(cudaEventCreate(&h->ev_mark[1]));
#undef CK
    if (cfg->mode & HBCU_DECOMB_EEDI2)
    {
        hbcu::Eedi2Config ec;
        ec.depth = cfg->depth;
        for (int pl = 0; pl < 3; pl++) { ec.w[pl] = h->g[pl].w; ec.h[pl] = h->g[pl].h; ec.pitch[pl] = h->g[pl].pitch; }
        ec.mthresh = cfg->magnitude_threshold; ec.vthresh = cfg->variance_threshold; ec.lthresh = cfg->laplacian_threshold;
        ec.dstr = cfg->dilation_threshold; ec.estr = cfg->erosion_threshold; ec.nt = cfg->noise_threshold;
        ec.maxd = cfg->maximum_search_distance; ec.pp = cfg->post_processing;
        // decomb.c:291-296: the half-height EEDI2 buffers are frames of height/2 (chroma rounds up from that)
        ec.half_frame_height = cfg->height / 2;
        ec.chroma_shift_h = cfg->chroma_shift_h;
        h->eedi = hbcu::eedi2_create(ec);
        if (h->eedi == nullptr)
        {
            hbcu_decomb_destroy(h);
            return -1;
        }
    }
    // the clearing memsets above (and EEDI2's) ran on the legacy default stream; the handle's non-blocking streams do not wait for it
    if (cudaDeviceSynchronize() != cudaSuccess)
    {
        set_error("decomb_create: %s", cudaGetErrorString(cudaGetLastError()));
        hbcu_decomb_destroy(h);
        return -1;
    }
    *out = h;
    return 0;
}

void hbcu_decomb_destroy(hbcu_decomb_t *h)
{
    if (h == nullptr) return;
    cudaSetDevice(h->cfg.device);
    cudaDeviceSynchronize();
    if (h->eedi) hbcu::eedi2_destroy(h->eedi);
    for (auto p : h->in_base) if (p) cudaFree(p);
    for (auto p : h->out_base) if (p) cudaFree(p);
    for (auto e : h->ev_upload) if (e) cudaEventDestroy(e);
    for (auto e : h->ev_readers) if (e) cudaEventDestroy(e);
    for (auto e : h->ev_kernel) if (e) cudaEventDestroy(e);
    for (auto e : h->ev_d2h) if (e) cudaEventDestroy(e);
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

// the caller's planes have exactly the device layout (back to back, reference stride): the frame is one copy
static bool same_layout(const hbcu_decomb_t *h, const void *const planes[3], const int strides[3])
{
    for (int pl = 0; pl < 3; pl++)
    {
        if ((size_t)strides[pl] != (size_t)h->g[pl].pitch * h->bps) return false;
        if ((const uint8_t *)planes[pl] != (const uint8_t *)planes[0] + h->plane_off[pl]) return false;
    }
    return true;
}

static int decomb_upload(hbcu_decomb_t *h, int64_t index, const void *const planes[3], const int strides[3], cudaMemcpyKind kind)
{
    if (h == nullptr || planes == nullptr || strides == nullptr || index < 0) { set_error("decomb_upload: bad argument"); return -1; }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    const int slot = (int)(index % h->slots);
    HBCU_CHECK(cudaStreamWaitEvent(h->s_h2d, h->ev_readers[slot], 0));
    const bool whole = same_layout(h, planes, strides);
    if (whole) HBCU_CHECK(cudaMemcpyAsync(h->in_base[slot], planes[0], h->frame_bytes, kind, h->s_h2d));
    for (int pl = 0; pl < 3 && !whole; pl++)
    {
        const Geom &g = h->g[pl];
        // copy whole strides when the layouts agree (the stride padding is part of what EEDI2 may read)
        const size_t row = (size_t)strides[pl] == (size_t)g.pitch * h->bps ? (size_t)g.pitch * h->bps : (size_t)g.w * h->bps;
        HBCU_CHECK(cudaMemcpy2DAsync(h->in_mem[slot * 3 + pl], (size_t)g.pitch * h->bps, planes[pl], (size_t)strides[pl],
                                     row, (size_t)g.h, kind, h->s_h2d));
    }
    HBCU_CHECK(cudaEventRecord(h->ev_upload[slot], h->s_h2d));
    h->in_index[slot] = index;
    return 0;
}

int hbcu_decomb_upload(hbcu_decomb_t *h, int64_t index, const void *const planes[3], const int strides[3])
{
    return decomb_upload(h, index, planes, strides, cudaMemcpyHostToDevice);
}

int hbcu_decomb_upload_device(hbcu_decomb_t *h, int64_t index, const void *const dplanes[3], const int strides[3])
{
    return decomb_upload(h, index, dplanes, strides, cudaMemcpyDeviceToDevice);
}

int hbcu_decomb_wait_upload(hbcu_decomb_t *h, int64_t index)
{
    if (h == nullptr || index < 0) { set_error("decomb_wait_upload: bad argument"); return -1; }
    const int slot = (int)(index % h->slots);
    if (h->in_index[slot] != index) return 0;     // overwritten since: that upload waited for its readers, which waited for ours
    HBCU_CHECK(cudaEventSynchronize(h->ev_upload[slot]));
    return 0;
}

int hbcu_decomb_filter(hbcu_decomb_t *h, int64_t ticket, int64_t prev, int64_t cur, int64_t next,
                       int frame_mode, int parity, int tff, void *const planes[3], const int strides[3])
{
    if (h == nullptr || planes == nullptr || strides == nullptr) { set_error("decomb_filter: bad argument"); return -1; }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    const int oslot = h->next_out;
    h->next_out = (h->next_out + 1) % h->out_slots;
    if (run_field(h, ticket, prev, cur, next, frame_mode, parity, tff, oslot) != 0) return -1;
    HBCU_CHECK(cudaStreamWaitEvent(h->s_d2h, h->ev_kernel[oslot], 0));
    const bool whole = same_layout(h, planes, strides);
    if (whole) HBCU_CHECK(cudaMemcpyAsync(planes[0], h->out_base[oslot], h->frame_bytes, cudaMemcpyDeviceToHost, h->s_d2h));
    for (int pl = 0; pl < 3 && !whole; pl++)
    {
        const Geom &g = h->g[pl];
        HBCU_CHECK(cudaMemcpy2DAsync(planes[pl], (size_t)strides[pl], h->out_mem[oslot * 3 + pl], (size_t)g.pitch * h->bps,
                                     (size_t)g.w * h->bps, (size_t)g.h, cudaMemcpyDeviceToHost, h->s_d2h));
    }
    HBCU_CHECK(cudaEventRecord(h->ev_d2h[oslot], h->s_d2h));
    return 0;
}

int hbcu_decomb_filter_device(hbcu_decomb_t *h, int64_t ticket, int64_t prev, int64_t cur, int64_t next,
                              int frame_mode, int parity, int tff, void *out_planes[3], int out_strides[3])
{
    if (h == nullptr) { set_error("decomb_filter_device: null handle"); return -1; }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    const int oslot = h->next_out;
    h->next_out = (h->next_out + 1) % h->out_slots;
    if (run_field(h, ticket, prev, cur, next, frame_mode, parity, tff, oslot) != 0) return -1;
    HBCU_CHECK(cudaEventRecord(h->ev_d2h[oslot], h->s_compute));
    for (int pl = 0; pl < 3; pl++)
    {
        if (out_planes) out_planes[pl] = h->out_mem[oslot * 3 + pl];
        if (out_strides) out_strides[pl] = h->g[pl].pitch * h->bps;
    }
    return 0;
}

static bool frame_fits(const hbcu_decomb_t *h, const hbcu_frame_t *f)
{
    if (f == nullptr || f->device != h->cfg.device) return false;
    for (int pl = 0; pl < 3; pl++)
        if (f->row_bytes[pl] != h->g[pl].w * h->bps || f->rows[pl] != h->g[pl].h || f->stride[pl] != h->g[pl].pitch * h->bps) return false;
    return true;
}

int hbcu_decomb_upload_frame(hbcu_decomb_t *h, int64_t index, hbcu_frame_t *in)
{
    if (h == nullptr || index < 0 || !frame_fits(h, in)) { set_error("decomb_upload_frame: bad argument or frame geometry"); return -1; }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    if (hbcu::frame_begin_read(in, h->s_h2d) != 0) return -1;
    const void *planes[3] = { in->plane[0], in->plane[1], in->plane[2] };
    if (decomb_upload(h, index, planes, in->stride, cudaMemcpyDeviceToDevice) != 0) return -1;
    return hbcu::frame_end_read(in, h->s_h2d);
}

int hbcu_decomb_filter_frame(hbcu_decomb_t *h, int64_t ticket, int64_t prev, int64_t cur, int64_t next,
                             int frame_mode, int parity, int tff, hbcu_frame_t *out)
{
    if (h == nullptr || !frame_fits(h, out)) { set_error("decomb_filter_frame: bad argument or frame geometry"); return -1; }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    const int oslot = h->next_out;
    h->next_out = (h->next_out + 1) % h->out_slots;
    if (hbcu::frame_begin_write(out, h->s_compute) != 0) return -1;
    if (run_field(h, ticket, prev, cur, next, frame_mode, parity, tff, oslot, out->plane) != 0) return -1;
    HBCU_CHECK(cudaEventRecord(h->ev_d2h[oslot], h->s_compute));
    return hbcu::frame_end_write(out, h->s_compute);
}

int hbcu_decomb_wait(hbcu_decomb_t *h, int64_t ticket)
{
    if (h == nullptr) { set_error("decomb_wait: null handle"); return -1; }
    const int s = find_ticket(h, ticket);
    if (s < 0) { set_error("decomb_wait: ticket %lld is not in flight", (long long)ticket); return -1; }
    HBCU_CHECK(cudaEventSynchronize(h->ev_d2h[s]));
    return 0;
}

int hbcu_decomb_poll(hbcu_decomb_t *h, int64_t ticket)
{
    if (h == nullptr) { set_error("decomb_poll: null handle"); return -1; }
    const int s = find_ticket(h, ticket);
    if (s < 0) { set_error("decomb_poll: ticket %lld is not in flight", (long long)ticket); return -1; }
    cudaError_t e = cudaEventQuery(h->ev_d2h[s]);
    if (e == cudaSuccess) return 1;
    if (e == cudaErrorNotReady) return 0;
    set_error("decomb_poll: %s", cudaGetErrorString(e));
    return -1;
}

int hbcu_decomb_debug_eedi2(hbcu_decomb_t *h, int which, void *host, size_t host_bytes)
{
    if (h == nullptr || h->eedi == nullptr) { set_error("decomb_debug_eedi2: no EEDI2 state"); return -1; }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    HBCU_CHECK(cudaDeviceSynchronize());
    return hbcu::eedi2_debug_read(h->eedi, which, host, host_bytes);
}

int hbcu_decomb_sync(hbcu_decomb_t *h)
{
    if (h == nullptr) { set_error("decomb_sync: null handle"); return -1; }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    HBCU_CHECK(cudaStreamSynchronize(h->s_h2d));
    HBCU_CHECK(cudaStreamSynchronize(h->s_compute));
    HBCU_CHECK(cudaStreamSynchronize(h->s_d2h));
    return 0;
}

int hbcu_decomb_mark(hbcu_decomb_t *h, int which)
{
    if (h == nullptr || which < 0 || which > 1) { set_error("decomb_mark: bad argument"); return -1; }
    HBCU_CHECK(cudaSetDevice(h->cfg.device));
    HBCU_CHECK(cudaEventRecord(h->ev_mark[which], h->s_compute));
    return 0;
}

int hbcu_decomb_elapsed_ms(hbcu_decomb_t *h, float *ms)
{
    if (h == nullptr || ms == nullptr) { set_error("decomb_elapsed_ms: bad argument"); return -1; }
    HBCU_CHECK(cudaEventSynchronize(h->ev_mark[1]));
    HBCU_CHECK(cudaEventElapsedTime(ms, h->ev_mark[0], h->ev_mark[1]));
    return 0;
}

}  // extern "C"
