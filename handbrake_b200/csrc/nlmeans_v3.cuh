// nlmeans_v3.cuh -- third generation of the fused 8-bit NLMeans tile kernel (included by nlmeans.cu).
//
// Same arithmetic contract as nlmeans_fast8_kernel (bit-identical to templates/nlmeans_template.c:593-717), same
// tiling idea (TMA tile in shared memory, a lane marches down a 4-pixel-wide column strip keeping the vertical running
// sum of horizontal patch-row sums and its N-row history in registers).  What changed, each item aimed at the
// instruction count per pixel and displacement:
//   * group shape (NG displacements), byte offset of the compare window and the origin slot are template parameters:
//     no per-row predicate/branch chains, and for the range-3 presets the three compare windows come straight out of
//     the raw words with 6 funnel shifts per row instead of 13 (the source window is never re-aligned: only the
//     relative alignment of source and compare matters to VABSDIFF4);
//   * the running sum V is kept as the integer 0x4B000000 + V: as a float that is 2^23 + V, so
//     fma.rn.sat(2^23 + V, wfact/128, -2^23 * wfact/128) = rn(V * wfact/128) exactly -- I2F and FMUL.SAT collapse into
//     one FFMA on the idle FMA pipe;
//   * the three-row delay line of compare words is indexed by the unrolled row slot instead of being shifted: no MOVs;
//   * warm-up rows are peeled: the steady-state loop has no "row >= NH" test;
//   * the compare tile of frame 1 is in flight while frame 0 is compared with itself (second mbarrier);
//   * accumulators (weight sum, pixel sum; 8 bytes per pixel) live in shared memory, a float4 per lane and array and row.
//     Together with the tiles they bound the tile height: 120 rows (12 warps x 10) keep the largest variant (16-bit
//     tiles, or the four tiles of the prefilter variant) inside the 227 KB an H100 block can have;
//   * range 3 without a prefilter (the SYM instantiation): frame 0, the current frame compared with itself, is one march
//     over four displacements instead of three over eight -- the other four weights are the same floats read one column
//     left or one row up (V3Sym) -- and it stores the accumulators instead of adding to zero-filled ones;
//   * range 3 with one or two frames (nlmeans_v3f_kernel): frame 1 advances in V3Sym's row step, every pixel is finished
//     in registers (V3Fused), and without accumulators the tile is twice as tall.
#pragma once

template <int NW, int RS, int NBUF, int BPS = 1, bool PRE = false>
struct V3Layout
{
    static constexpr int kTH        = NW * RS;
    static constexpr int kLoads     = kTH + 2 * kHalo > 256 ? 2 : 1;                     // a TMA box has at most 256 rows
    static constexpr int kBoxRows   = ((kTH + 2 * kHalo + kLoads - 1) / kLoads + 3) / 4 * 4;   // 4 rows x 160 B keep every box 128-byte aligned
    static constexpr int kRows      = kBoxRows * kLoads;                                 // >= kTH + 2 * kHalo; surplus rows are loaded, never used
    static constexpr int kRowBytes  = kTilePW * BPS;
    static constexpr int kTileBytes = kRows * kRowBytes;
    static constexpr int kAccBytes  = kTH * kTileW * (int)sizeof(float);                 // per accumulator array
    static constexpr int kLutBytes  = kLutEntries * 32 * (int)sizeof(float);
    static constexpr int kOffCur    = 0;
    static constexpr int kOffCmp    = kOffCur + kTileBytes;
    // prefilter variant: the pre-denoised current tile and ONE pre-denoised compare tile (patch distances are taken from
    // these, pixel values from the plain tiles)
    static constexpr int kOffPre0   = kOffCmp + NBUF * kTileBytes;
    static constexpr int kOffCmpPre = kOffPre0 + (PRE ? kTileBytes : 0);
    static constexpr int kOffWs     = kOffCmpPre + (PRE ? kTileBytes : 0);
    static_assert(!PRE || NBUF == 1, "the prefilter variant keeps one compare buffer pair");
    static constexpr int kOffPs     = kOffWs + kAccBytes;
    static constexpr int kOffLut    = kOffPs + kAccBytes;
    static constexpr int kOffBar    = kOffLut + kLutBytes;                               // 1 + NBUF mbarriers
    static constexpr int kUsed      = kOffBar + 64;
    // one CTA per SM by construction (every variant needs more than half of the SM's shared memory)
    static constexpr int kTotal     = kUsed < 117 * 1024 ? 117 * 1024 : kUsed;
    static_assert(kBoxRows <= 256, "TMA box rows");
    static_assert((kBoxRows * kRowBytes) % 128 == 0, "TMA destination must stay 128-byte aligned");
    static_assert(kTotal <= 227 * 1024, "shared memory");
};

// accumulator rows of one warp in shared memory (float4 per lane and array)
struct V3Acc
{
    float *ws, *ps;     // this lane's first row
    __device__ __forceinline__ void load(int r, uint32_t (&v)[8]) const
    {
        const uint4 a = *reinterpret_cast<const uint4 *>(ws + r * kTileW);
        const uint4 b = *reinterpret_cast<const uint4 *>(ps + r * kTileW);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    }
    __device__ __forceinline__ void wait_load(uint32_t (&)[8]) const {}
    __device__ __forceinline__ void store(int r, const uint32_t (&v)[8]) const
    {
        *reinterpret_cast<uint4 *>(ws + r * kTileW) = make_uint4(v[0], v[1], v[2], v[3]);
        *reinterpret_cast<uint4 *>(ps + r * kTileW) = make_uint4(v[4], v[5], v[6], v[7]);
    }
    __device__ __forceinline__ void wait_store() const {}
};

// fp32 pairs (pixels 0/2 and 1/3 of a lane's four): each half is one IEEE round-to-nearest (or toward-zero) fp32
// operation.  The _rn/_rz intrinsics are never contracted into an FMA (the reference rounds the product before it adds).
__device__ __forceinline__ float2 v3_pack2(float a, float b) { return make_float2(a, b); }
__device__ __forceinline__ void v3_unpack2(float2 v, float &a, float &b)
{
    a = v.x;
    b = v.y;
}
__device__ __forceinline__ float2 v3_add2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 v3_add2_rz(float2 a, float2 b) { return make_float2(__fadd_rz(a.x, b.x), __fadd_rz(a.y, b.y)); }
__device__ __forceinline__ float2 v3_mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
// position of pixel i of a lane's four in the accumulator words (pairs (0, 2) and (1, 3))
__device__ __forceinline__ constexpr int v3_acc_slot(int i) { return (i & 1) * 2 + (i >> 1); }

constexpr int kOrgNone = -1;
constexpr uint32_t kVBias = 0x4B000000u;     // bits of 2^23

// One group of NG horizontally adjacent displacements (dy, dx0 .. dx0+NG-1) over `rows` output rows of this warp's strip.
//   OBS  : (12 + dx0) & 3, the byte offset of the compare window inside its first word
//   ORG  : slot of the origin displacement inside the group, or kOrgNone
// A struct so that the row step can be a function template of its unrolled slot K (every index into hist / P is a
// compile-time constant; everything is force-inlined and the arrays live in registers).
template <int NH, int NG, int OBS, int ORG, bool PRE, class ACC>
struct V3Group
{
    static constexpr int N      = 2 * NH + 1;
    static constexpr int PW     = kTilePW / 4;       // tile pitch in words
    static constexpr int FIRSTB = 4 - NH;            // the source stream starts 4 pixels left of the lane's first pixel:
    static constexpr int LASTB  = 7 + NH;            // the four windows cover its bytes FIRSTB .. LASTB
    static constexpr int NWA    = LASTB / 4 + 1;     // source words (3 for every patch size <= 9)
    static constexpr int LASTC  = LASTB + NG - 1;    // last compare-stream byte any displacement of the group touches
    static constexpr int NAL    = LASTC / 4 + 1;     // compare-stream words
    static constexpr int NRAW   = NAL + 1;           // raw words that cover them at any byte offset
    static_assert(NWA == 3, "patch size");

    uint32_t V[NG][4];
    uint32_t hist[N][NG][4];
    uint32_t P[PRE ? 1 : N][2];                      // compare-stream words 1 and 2 of the last rows: the averaged pixels
    const uint32_t *arow, *brow, *orow, *prow;       // (prefilter variant: re-read from the PLAIN compare tile instead)
    const ACC &acc;
    uint32_t lut_lane_addr;
    float wscale, wbias;
    double origin_tune;

    // srcp / cmpd: the tiles the patch distances are taken from (source, compare); cmpv: the compare tile whose pixels are
    // averaged; cur: the plain current tile (origin term).  Without a prefilter srcp == cur and cmpd == cmpv.
    __device__ __forceinline__ V3Group(const uint32_t *srcp, const uint32_t *cmpd, const uint32_t *cmpv, const uint32_t *cur, const ACC &acc_,
                                       uint32_t lut_lane_addr_, float wscale_, float wbias_, double origin_tune_, int seg_y0, int lane, int dy, int dx0)
        : acc(acc_), lut_lane_addr(lut_lane_addr_), wscale(wscale_), wbias(wbias_), origin_tune(origin_tune_)
    {
        const int s   = 12 + dx0;                    // tile byte (relative to 4 * lane) of compare-stream byte 0
        const int wb0 = s >> 2;
#pragma unroll
        for (int g = 0; g < NG; g++)
#pragma unroll
            for (int i = 0; i < 4; i++)
            {
                V[g][i] = kVBias;
#pragma unroll
                for (int k = 0; k < N; k++) hist[k][g][i] = 0;
            }
#pragma unroll
        for (int k = 0; k < (PRE ? 1 : N); k++) P[k][0] = P[k][1] = 0;
        arow = srcp + (seg_y0 - NH + kHalo) * PW + lane + 3;
        brow = cmpd + (seg_y0 - NH + kHalo + dy) * PW + lane + wb0;
        orow = cur + (seg_y0 + kHalo) * PW + lane + kHaloX / 4;
        prow = cmpv + (seg_y0 + kHalo + dy) * PW + lane + wb0 + 1;
    }

    static __device__ __forceinline__ bool is_origin(int g) { return ORG >= 0 && g == ORG; }

    // one row step in unrolled slot K; OUT: the row NH above completes and is averaged into accumulator row r
    template <int K, bool OUT>
    __device__ __forceinline__ void step(int r)
    {
        uint32_t a[NWA], raw[NRAW], bg0[NAL];
#pragma unroll
        for (int j = 0; j < NWA; j++) a[j] = arow[j];
#pragma unroll
        for (int j = 0; j < NRAW; j++) raw[j] = brow[j];
        arow += PW;
        brow += PW;
        uint32_t accv[8];
        if (OUT) acc.load(r, accv);
        // compare stream aligned for displacement 0 of the group
#pragma unroll
        for (int j = 0; j < NAL; j++) bg0[j] = OBS == 0 ? raw[j] : __funnelshift_r(raw[j], raw[j + 1], 8 * OBS);
#pragma unroll
        for (int g = 0; g < NG; g++)
        {
            if (ORG != kOrgNone && is_origin(g)) continue;
            uint32_t D[NWA];
#pragma unroll
            for (int w = 0; w < NWA; w++)
            {
                uint32_t bw;
                if (g == 0) bw = bg0[w];
                else
                {
                    const int sh = (OBS + g) & 3, q = (OBS + g) >> 2;       // compile-time after unrolling
                    const int j1 = w + q + 1 < NRAW ? w + q + 1 : NRAW - 1;
                    bw = sh ? __funnelshift_r(raw[w + q], raw[j1], 8 * sh) : raw[w + q];
                }
                D[w] = __vabsdiffu4(a[w], bw);
            }
            if constexpr (NH == 3)
            {
                // patch 7: the windows are bytes 1+i .. 7+i of the D stream = word 1 (bytes 4..7, shared) plus exactly
                // three more bytes.  Byte 0 of the stream belongs to no window: cleared, it is the zero that pads those
                // three bytes (gathered by PRMT from words 0 and 2) to a word, so every window is IDP4A(X, X, T1).
                const uint32_t T1 = __dp4a(D[1], D[1], 0u);
                const uint32_t Z  = D[0] & 0xFFFFFF00u;
                uint32_t X[4];
                X[0] = Z;                                   // bytes 1, 2, 3
                X[1] = __byte_perm(Z, D[2], 0x0432);        // bytes 2, 3, 8
                X[2] = __byte_perm(Z, D[2], 0x0543);        // bytes 3, 8, 9
                X[3] = __byte_perm(Z, D[2], 0x0654);        // bytes 8, 9, 10
#pragma unroll
                for (int i = 0; i < 4; i++)
                {
                    const uint32_t hs = __dp4a(X[i], X[i], T1);
                    V[g][i] = V[g][i] + hs - hist[K][g][i];
                    hist[K][g][i] = hs;
                }
            }
            else
            {
            // patch-row sums over bytes FIRSTB+i .. FIRSTB+i+N-1 of the D stream: whole words by IDP4A(D, D), partial
            // words by IDP4A(D & mask, D); the first whole word is shared by the four windows
            uint32_t T[NWA];
#pragma unroll
            for (int w = 0; w < NWA; w++) T[w] = __dp4a(D[w], D[w], 0u);
#pragma unroll
            for (int i = 0; i < 4; i++)
            {
                const int b0 = FIRSTB + i, b1 = FIRSTB + i + N - 1;
                uint32_t hs = 0;
                bool started = false;
#pragma unroll
                for (int w = 0; w < NWA; w++)
                {
                    const int lo = b0 > 4 * w ? b0 : 4 * w, hi = b1 < 4 * w + 3 ? b1 : 4 * w + 3;
                    if (lo == 4 * w && hi == 4 * w + 3 && !started) { hs = T[w]; started = true; }
                }
                bool used_full = false;
#pragma unroll
                for (int w = 0; w < NWA; w++)
                {
                    const int lo = b0 > 4 * w ? b0 : 4 * w, hi = b1 < 4 * w + 3 ? b1 : 4 * w + 3;
                    if (lo > hi) continue;
                    if (lo == 4 * w && hi == 4 * w + 3)
                    {
                        if (started && !used_full) { used_full = true; continue; }   // already in hs
                        hs = __dp4a(D[w], D[w], hs);
                    }
                    else
                    {
                        uint32_t m = 0;
#pragma unroll
                        for (int bb = 0; bb < 4; bb++)
                            if (4 * w + bb >= lo && 4 * w + bb <= hi) m |= 0xFFu << (8 * bb);
                        hs = __dp4a(D[w] & m, D[w], hs);
                    }
                }
                V[g][i] = V[g][i] + hs - hist[K][g][i];
                hist[K][g][i] = hs;
            }
            }
        }
        if (OUT)
        {
            constexpr int KP = PRE ? 0 : (K + N - NH) % N;   // the compare row of the output row was loaded NH steps ago
            uint32_t p0, p1;
            if constexpr (PRE)
            {
                const uint32_t q0 = prow[r * PW], q1 = prow[r * PW + 1], q2 = prow[r * PW + 2];
                p0 = OBS == 0 ? q0 : __funnelshift_r(q0, q1, 8 * OBS);
                p1 = OBS == 0 ? q1 : __funnelshift_r(q1, q2, 8 * OBS);
            }
            else
            {
                p0 = P[KP][0];
                p1 = P[KP][1];
            }
            // pixels 0/2 and 1/3 of the lane's four travel as pairs; accumulator words are stored in that order:
            // {ws0, ws2, ws1, ws3, ps0, ps2, ps1, ps3}
            float2 pix2[NG + 1];                          // (compare pixel j, compare pixel j + 2) as floats
#pragma unroll
            for (int j = 0; j < NG + 1; j++)
                pix2[j] = v3_add2(v3_pack2(byte_as_biased_float(j < 4 ? p0 : p1, j & 3), byte_as_biased_float(j + 2 < 4 ? p0 : p1, (j + 2) & 3)),
                                  v3_pack2(-8388608.0f, -8388608.0f));
            acc.wait_load(accv);                          // issued at the top of the step: the patch-row sums covered its latency
            float2 W[NG][2];                              // weights of pixels (0, 2) and (1, 3)
#pragma unroll
            for (int g = 0; g < NG; g++)
            {
                if (ORG != kOrgNone && is_origin(g)) continue;
                float t[4];
#pragma unroll
                for (int i = 0; i < 4; i++)
                    asm("fma.rn.sat.f32 %0, %1, %2, %3;" : "=f"(t[i]) : "f"(__uint_as_float(V[g][i])), "f"(wscale), "f"(wbias));
#pragma unroll
                for (int h = 0; h < 2; h++)
                {
                    float u0, u1, w0, w1;
                    v3_unpack2(v3_add2_rz(v3_pack2(t[h], t[h + 2]), v3_pack2(65536.0f, 65536.0f)), u0, u1);   // 65536 + floor(128 t)
                    asm("ld.shared.f32 %0, [%1];" : "=f"(w0) : "r"((__float_as_uint(u0) << 7) + lut_lane_addr));
                    asm("ld.shared.f32 %0, [%1];" : "=f"(w1) : "r"((__float_as_uint(u1) << 7) + lut_lane_addr));
                    W[g][h] = v3_pack2(w0, w1);
                }
            }
            float2 ws2[2], ps2[2];
#pragma unroll
            for (int h = 0; h < 2; h++)
            {
                ws2[h] = v3_pack2(__uint_as_float(accv[2 * h]), __uint_as_float(accv[2 * h + 1]));
                ps2[h] = v3_pack2(__uint_as_float(accv[4 + 2 * h]), __uint_as_float(accv[4 + 2 * h + 1]));
            }
#pragma unroll
            for (int g = 0; g < NG; g++)
            {
                if (ORG != kOrgNone && is_origin(g))
                {
                    const uint32_t cw = orow[r * PW];
#pragma unroll
                    for (int h = 0; h < 2; h++)
                    {
                        float wa, wb, pa, pb;
                        v3_unpack2(ws2[h], wa, wb);
                        v3_unpack2(ps2[h], pa, pb);
                        add_origin(wa, pa, origin_tune, (int)((cw >> (8 * h)) & 0xffu));
                        add_origin(wb, pb, origin_tune, (int)((cw >> (8 * (h + 2))) & 0xffu));
                        ws2[h] = v3_pack2(wa, wb);
                        ps2[h] = v3_pack2(pa, pb);
                    }
                }
                else
                {
#pragma unroll
                    for (int h = 0; h < 2; h++)
                    {
                        ws2[h] = v3_add2(ws2[h], W[g][h]);
                        ps2[h] = v3_add2(ps2[h], v3_mul2(W[g][h], pix2[g + h]));
                    }
                }
            }
#pragma unroll
            for (int h = 0; h < 2; h++)
            {
                float a, b;
                v3_unpack2(ws2[h], a, b);
                accv[2 * h] = __float_as_uint(a); accv[2 * h + 1] = __float_as_uint(b);
                v3_unpack2(ps2[h], a, b);
                accv[4 + 2 * h] = __float_as_uint(a); accv[4 + 2 * h + 1] = __float_as_uint(b);
            }
            acc.store(r, accv);
        }
        if constexpr (!PRE)
        {
            P[K][0] = bg0[1];
            P[K][1] = bg0[2];
        }
    }

    template <int... Ks>
    __device__ __forceinline__ void warm_up(std::integer_sequence<int, Ks...>)
    {
        (step<Ks, false>(0), ...);
    }
    template <int... Ms>
    __device__ __forceinline__ void rows_from(int r0, int rows, std::integer_sequence<int, Ms...>)
    {
        ((r0 + Ms < rows ? step<(2 * NH + Ms) % N, true>(r0 + Ms) : (void)0), ...);
    }
    template <int... Ms>
    __device__ __forceinline__ void batch(int r0, std::integer_sequence<int, Ms...>)
    {
        (step<(2 * NH + Ms) % N, true>(r0 + Ms), ...);
    }

    // EXACT: `rows` is a multiple of N -- batches of N rows without a per-row test (and without the register moves the
    // merge points of those tests cost)
    template <bool EXACT>
    __device__ __forceinline__ void run(int rows)
    {
        // warm-up: the first 2*NH rows only build patch-row sums (slots 0 .. 2NH-1);
        // steady state: output row r completes at row step r + 2NH, slot (r + 2NH) % N
        warm_up(std::make_integer_sequence<int, 2 * NH>{});
        if (EXACT)
        {
#pragma unroll 1
            for (int r0 = 0; r0 < rows; r0 += N) batch(r0, std::make_integer_sequence<int, N>{});
        }
        else
        {
#pragma unroll 1
            for (int r0 = 0; r0 < rows; r0 += N) rows_from(r0, rows, std::make_integer_sequence<int, N>{});
        }
        acc.wait_store();
    }
};

template <int NH, int NG, int OBS, int ORG, bool EXACT, bool PRE, class ACC>
__device__ __forceinline__ void v3_group(const uint32_t *__restrict__ srcp, const uint32_t *__restrict__ cmpd, const uint32_t *__restrict__ cmpv,
                                         const uint32_t *__restrict__ cur, const ACC &acc,
                                         uint32_t lut_lane_addr, float wscale, float wbias, double origin_tune,
                                         int seg_y0, int rows, int lane, int dy, int dx0)
{
    V3Group<NH, NG, OBS, ORG, PRE, ACC> g(srcp, cmpd, cmpv, cur, acc, lut_lane_addr, wscale, wbias, origin_tune, seg_y0, lane, dy, dx0);
    g.template run<EXACT>(rows);
}

// Group shapes a displacement row can be cut into (three displacements per group, the remainder last), keyed by
// {displacements, (12 + dx0) & 3, origin slot}.  Every range 3 .. 15 decomposes into these eleven (v3_group_known()).
#define V3_GROUP_SHAPES(X) \
    X(3, 0, kOrgNone) X(3, 1, kOrgNone) X(3, 2, kOrgNone) X(3, 3, kOrgNone) \
    X(3, 3, 1) X(3, 2, 2) X(3, 0, 0) \
    X(2, 1, kOrgNone) X(2, 0, kOrgNone) X(1, 3, kOrgNone) X(1, 2, kOrgNone)

__host__ __device__ inline bool v3_group_known(int ng, int ob, int org)
{
#define X(NG_, OB_, ORG_) if (ng == NG_ && ob == OB_ && org == ORG_) return true;
    V3_GROUP_SHAPES(X)
#undef X
    return false;
}

// Frame 0 of a range-3 search (r_half == 1) in one march.  Frame 0 compares the current tile with itself, and there the
// patch distance is symmetric: SSD_{-d}(p) == SSD_d(p - d), the same integer from the same tile bytes, so the weight
// (a function of that integer alone) is the same float.  Four "forward" displacements give all eight weights:
//   A = (0,+1), B = (+1,+1), C = (+1,0), D = (+1,-1);
//   (0,-1) at x is A at x-1;  (-1,-1) at (y, x) is B at (y-1, x-1);  (-1,0) is C at (y-1, x);  (-1,+1) is D at (y-1, x+1).
// A lane keeps the running sums of A and B at columns x-1 .. x+3, C at x .. x+3 and D at x .. x+4 (the windows at x-1
// and x+4 come out of the same D words as the lane's own four: no shuffles), starting one row above the strip so that
// row -1 has (+1, .) weights.  The weights of the (+1, .) displacements are kept for one row; the patch-row sum leaving
// a running sum is recomputed from the tile instead of kept (a 2NH+1-row history of 19 sums does not fit the register
// budget of 12 warps).  The nine frame-0 terms of an output pixel are added in registers in the reference's order --
// (-1,-1) (-1,0) (-1,1) (0,-1) origin (0,1) (1,-1) (1,0) (1,1) -- one IEEE operation each, as V3Group does, and stored
// with plain stores: the accumulators need no zero fill.  The first term is stored as is (0 + w == w, 0 + w*p == w*p:
// weights and pixels are never negative).
//
// Row slots: output row r (r = -1 .. rows-1) runs in slot K = (r + 1) % 6.  Its compare-row words are kept by parity
// (the words of row t + 1 are the source words of the next step), its pixel rows by row mod 3: every array index is a
// compile-time constant of the unrolled slot.
template <int NH, class ACC>
struct V3Sym
{
    static constexpr int PW = kTilePW / 4;           // tile pitch in words
    static_assert(NH >= 1 && NH <= 3, "patch size");

    uint32_t VA[5], VB[5], VC[4], VD[5];             // 2^23-biased running sums; A, B: columns x-1 .. x+3, C: x .. x+3, D: x .. x+4
    uint32_t qi[2][5], qo[2][5];                     // words lane+2 .. lane+6 of the compare row entering / leaving the sums
    float pix[3][6];                                 // pixels x-1 .. x+4 of a row, as floats
    float WB[2][5], WC[2][4], WD[2][5];              // weights of the (+1, .) displacements, same columns as their sums
    const uint32_t *base;                            // tile word `lane` of output row 0
    const ACC &acc;
    uint32_t lut_lane_addr;
    float wscale, wbias;
    double origin_tune;

    __device__ __forceinline__ V3Sym(const uint32_t *cur, const ACC &acc_, uint32_t lut_lane_addr_, float wscale_, float wbias_,
                                     double origin_tune_, int seg_y0, int lane)
        : acc(acc_), lut_lane_addr(lut_lane_addr_), wscale(wscale_), wbias(wbias_), origin_tune(origin_tune_)
    {
        base = cur + (seg_y0 + kHalo) * PW + lane;
    }

    // patch-row sum of window I (columns x+I-NH .. x+I+NH) from the D words of a row (byte j: column x-4+j); T[w] is
    // IDP4A(D[w], D[w])
    template <int I>
    static __device__ __forceinline__ uint32_t window(const uint32_t (&D)[3], const uint32_t (&T)[3])
    {
        constexpr int b0 = 4 - NH + I, b1 = 4 + NH + I;
        static_assert(b0 >= 0 && b1 <= 11, "window outside the D words");
        if constexpr (NH == 3 && I >= 0 && I <= 3)
        {
            // V3Group's patch-7 form: bytes 4..7 shared, the other three gathered into one word (byte 0 cleared)
            const uint32_t Z = D[0] & 0xFFFFFF00u;
            const uint32_t X = I == 0 ? Z : __byte_perm(Z, D[2], I == 1 ? 0x0432 : I == 2 ? 0x0543 : 0x0654);
            return __dp4a(X, X, T[1]);
        }
        else
        {
            int full = -1;                           // the first whole word of the window starts the sum
#pragma unroll
            for (int w = 0; w < 3; w++)
                if (full < 0 && b0 <= 4 * w && 4 * w + 3 <= b1) full = w;
            uint32_t hs = full >= 0 ? T[full] : 0u;
#pragma unroll
            for (int w = 0; w < 3; w++)
            {
                const int lo = b0 > 4 * w ? b0 : 4 * w, hi = b1 < 4 * w + 3 ? b1 : 4 * w + 3;
                if (lo > hi || w == full) continue;
                if (lo == 4 * w && hi == 4 * w + 3) hs = __dp4a(D[w], D[w], hs);
                else
                {
                    uint32_t m = 0;
#pragma unroll
                    for (int bb = 0; bb < 4; bb++)
                        if (4 * w + bb >= lo && 4 * w + bb <= hi) m |= 0xFFu << (8 * bb);
                    hs = __dp4a(D[w] & m, D[w], hs);
                }
            }
            return hs;
        }
    }

    template <int LO, int... Is>
    static __device__ __forceinline__ void windows(const uint32_t (&D)[3], uint32_t (&hs)[sizeof...(Is)], std::integer_sequence<int, Is...>)
    {
        uint32_t T[3];
#pragma unroll
        for (int w = 0; w < 3; w++) T[w] = __dp4a(D[w], D[w], 0u);
        ((hs[Is] = window<LO + Is>(D, T)), ...);
    }

    // patch-row sums of one row: source words a = lane+3 .. lane+6 of row t, q = lane+2 .. lane+6 of row t+1
    static __device__ __forceinline__ void row_sums(const uint32_t (&a)[4], const uint32_t (&q)[5],
                                                    uint32_t (&hA)[5], uint32_t (&hB)[5], uint32_t (&hC)[4], uint32_t (&hD)[5])
    {
        uint32_t DA[3], DB[3], DC[3], DD[3];
#pragma unroll
        for (int w = 0; w < 3; w++)
        {
            DA[w] = __vabsdiffu4(a[w], __funnelshift_r(a[w], a[w + 1], 8));      // row t, one column right
            DB[w] = __vabsdiffu4(a[w], __funnelshift_r(q[w + 1], q[w + 2], 8));  // row t+1, one column right
            DC[w] = __vabsdiffu4(a[w], q[w + 1]);                                // row t+1
            DD[w] = __vabsdiffu4(a[w], __funnelshift_r(q[w], q[w + 1], 24));     // row t+1, one column left
        }
        windows<-1>(DA, hA, std::make_integer_sequence<int, 5>{});
        windows<-1>(DB, hB, std::make_integer_sequence<int, 5>{});
        windows<0>(DC, hC, std::make_integer_sequence<int, 4>{});
        windows<0>(DD, hD, std::make_integer_sequence<int, 5>{});
    }

    // compare row `row` (relative to output row 0) into q[P]; the sums of row - 1, whose source words are q[1 - P]
    template <int P>
    __device__ __forceinline__ void sums(uint32_t (&q)[2][5], int row, uint32_t (&hA)[5], uint32_t (&hB)[5], uint32_t (&hC)[4], uint32_t (&hD)[5])
    {
#pragma unroll
        for (int k = 0; k < 5; k++) q[P][k] = base[row * PW + 2 + k];
        const uint32_t a[4] = { q[1 - P][1], q[1 - P][2], q[1 - P][3], q[1 - P][4] };
        row_sums(a, q[P], hA, hB, hC, hD);
    }

    template <int S>
    __device__ __forceinline__ void load_pixels(int row)
    {
        const uint32_t *w = base + row * PW + 3;
        const uint32_t w0 = w[0], w1 = w[1], w2 = w[2];
        pix[S][0] = __fadd_rn(byte_as_biased_float(w0, 3), -8388608.0f);
#pragma unroll
        for (int i = 0; i < 4; i++) pix[S][1 + i] = __fadd_rn(byte_as_biased_float(w1, i), -8388608.0f);
        pix[S][5] = __fadd_rn(byte_as_biased_float(w2, 0), -8388608.0f);
    }

    __device__ __forceinline__ float weight(uint32_t v) const
    {
        float t, w;
        asm("fma.rn.sat.f32 %0, %1, %2, %3;" : "=f"(t) : "f"(__uint_as_float(v)), "f"(wscale), "f"(wbias));
        const float u = __fadd_rz(t, 65536.0f);                                  // 65536 + floor(128 t)
        asm("ld.shared.f32 %0, [%1];" : "=f"(w) : "r"((__float_as_uint(u) << 7) + lut_lane_addr));
        return w;
    }

    template <int P>
    __device__ __forceinline__ void plus_weights()
    {
#pragma unroll
        for (int k = 0; k < 5; k++) WB[P][k] = weight(VB[k]);
#pragma unroll
        for (int k = 0; k < 4; k++) WC[P][k] = weight(VC[k]);
#pragma unroll
        for (int k = 0; k < 5; k++) WD[P][k] = weight(VD[k]);
    }

    // output row r in slot K: the weight and pixel sums of its nine frame-0 terms
    template <int K>
    __device__ __forceinline__ void terms(int r, float (&ws4)[4], float (&ps4)[4])
    {
        constexpr int P = K % 2, Q = 1 - P;                                      // this row's and the previous row's weights
        constexpr int SM = (K + 1) % 3, S0 = (K + 2) % 3, SP = K % 3;           // pixel rows r-1, r, r+1
        {
            uint32_t iA[5], iB[5], iC[4], iD[5], oA[5], oB[5], oC[4], oD[5];
            sums<P>(qi, r + NH + 1, iA, iB, iC, iD);                            // patch row r+NH enters
            sums<P>(qo, r - NH, oA, oB, oC, oD);                                // patch row r-NH-1 leaves
#pragma unroll
            for (int k = 0; k < 5; k++)
            {
                VA[k] = VA[k] + iA[k] - oA[k];
                VB[k] = VB[k] + iB[k] - oB[k];
                VD[k] = VD[k] + iD[k] - oD[k];
            }
#pragma unroll
            for (int k = 0; k < 4; k++) VC[k] = VC[k] + iC[k] - oC[k];
        }
        load_pixels<SP>(r + 1);
        float WA[5];
#pragma unroll
        for (int k = 0; k < 5; k++) WA[k] = weight(VA[k]);
        plus_weights<P>();
#pragma unroll
        for (int i = 0; i < 4; i++)
        {
            const float *pm = pix[SM], *p0 = pix[S0], *pp = pix[SP];
            float ws = WB[Q][i];                                                  // (-1,-1) = B at (r-1, x+i-1)
            float ps = __fmul_rn(WB[Q][i], pm[i]);
            ws = __fadd_rn(ws, WC[Q][i]);                                         // (-1, 0) = C at (r-1, x+i)
            ps = __fadd_rn(ps, __fmul_rn(WC[Q][i], pm[i + 1]));
            ws = __fadd_rn(ws, WD[Q][i + 1]);                                     // (-1,+1) = D at (r-1, x+i+1)
            ps = __fadd_rn(ps, __fmul_rn(WD[Q][i + 1], pm[i + 2]));
            ws = __fadd_rn(ws, WA[i]);                                            // ( 0,-1) = A at (r, x+i-1)
            ps = __fadd_rn(ps, __fmul_rn(WA[i], p0[i]));
            ws = (float)__dadd_rn((double)ws, origin_tune);                       // origin (add_origin)
            ps = (float)__dadd_rn((double)ps, __dmul_rn(origin_tune, (double)p0[i + 1]));
            ws = __fadd_rn(ws, WA[i + 1]);                                        // ( 0,+1)
            ps = __fadd_rn(ps, __fmul_rn(WA[i + 1], p0[i + 2]));
            ws = __fadd_rn(ws, WD[P][i]);                                         // (+1,-1)
            ps = __fadd_rn(ps, __fmul_rn(WD[P][i], pp[i]));
            ws = __fadd_rn(ws, WC[P][i]);                                         // (+1, 0)
            ps = __fadd_rn(ps, __fmul_rn(WC[P][i], pp[i + 1]));
            ws = __fadd_rn(ws, WB[P][i + 1]);                                     // (+1,+1)
            ps = __fadd_rn(ps, __fmul_rn(WB[P][i + 1], pp[i + 2]));
            ws4[i] = ws;
            ps4[i] = ps;
        }
    }

    // output row r in slot K: its frame-0 sums into the accumulators
    template <int K>
    __device__ __forceinline__ void step(int r)
    {
        float ws[4], ps[4];
        terms<K>(r, ws, ps);
        uint32_t accv[8];
#pragma unroll
        for (int i = 0; i < 4; i++)
        {
            accv[v3_acc_slot(i)] = __float_as_uint(ws[i]);
            accv[4 + v3_acc_slot(i)] = __float_as_uint(ps[i]);
        }
        acc.store(r, accv);
    }

    template <int... Ms>
    __device__ __forceinline__ void rows_from(int r0, int rows, std::integer_sequence<int, Ms...>)
    {
        ((r0 + Ms < rows ? step<(Ms + 1) % 6>(r0 + Ms) : (void)0), ...);
    }

    // warm-up row j (patch row t = j - NH - 1) adds its sums
    template <int... Js>
    __device__ __forceinline__ void warm_up(std::integer_sequence<int, Js...>)
    {
        ((warm_row<Js % 2>(Js - NH - 1)), ...);
    }
    template <int P>
    __device__ __forceinline__ void warm_row(int t)
    {
        uint32_t hA[5], hB[5], hC[4], hD[5];
        sums<P>(qi, t + 1, hA, hB, hC, hD);
#pragma unroll
        for (int k = 0; k < 5; k++)
        {
            VA[k] += hA[k];
            VB[k] += hB[k];
            VD[k] += hD[k];
        }
#pragma unroll
        for (int k = 0; k < 4; k++) VC[k] += hC[k];
    }

    // the state of output row -1: slot 0 of the march comes next
    __device__ __forceinline__ void start()
    {
#pragma unroll
        for (int k = 0; k < 5; k++) VA[k] = VB[k] = VD[k] = kVBias;
#pragma unroll
        for (int k = 0; k < 4; k++) VC[k] = kVBias;
        // source words of patch row -NH-1: the first row of the warm-up, and the first row the march takes out again
#pragma unroll
        for (int k = 1; k < 5; k++) qo[0][k] = qi[1][k] = base[(-NH - 1) * PW + 2 + k];
        // row -1: the sums of patch rows -NH-1 .. NH-1 (the last one leaves its compare words in qi[0]), the (+1, .) weights
        warm_up(std::make_integer_sequence<int, 2 * NH + 1>{});
        plus_weights<0>();
        load_pixels<2>(-1);
        load_pixels<0>(0);
    }

    __device__ __forceinline__ void run(int rows)
    {
        start();
#pragma unroll 1
        for (int r0 = 0; r0 < rows; r0 += 6) rows_from(r0, rows, std::make_integer_sequence<int, 6>{});
        acc.wait_store();
    }
};

template <int NH, int NW, int RS, int NBUF, bool PRE = false, bool SYM = false>
__global__ void __launch_bounds__(NW * 32, 1) nlmeans_v3_kernel(const __grid_constant__ FusedParams fp)
{
    static_assert(!SYM || (!PRE && NH <= 3), "the symmetric frame-0 march: no prefilter, patch 3 .. 7");
    constexpr int kThreads = NW * 32;
    using L = V3Layout<NW, RS, NBUF, 1, PRE>;
    int pl = 0;
    while (pl + 1 < fp.nplanes && (int)blockIdx.x >= fp.first_tile[pl + 1]) pl++;
    const KernelParams &p = fp.k[pl];
    const CUtensorMap *maps = fp.maps[pl];
    const CUtensorMap *maps_pre = fp.maps_pre[pl];       // prefilter variant only
    const int tile = (int)blockIdx.x - fp.first_tile[pl];
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t *cur  = smem + L::kOffCur;
    float *lut    = reinterpret_cast<float *>(smem + L::kOffLut);
    uint64_t *bar = reinterpret_cast<uint64_t *>(smem + L::kOffBar);           // [0] current tile, [1 + b] compare buffer b

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int X0 = (tile % fp.tiles_x[pl]) * kTileW, Y0 = (tile / fp.tiles_x[pl]) * L::kTH;
    const int gx = X0 + kBorder - kHaloX, gy = Y0 + kBorder - kHalo;

    if (tid == 0)
    {
        for (int b = 0; b < 1 + NBUF; b++) mbar_init(bar + b, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid == 0)
    {
        mbar_expect_tx(bar, L::kTileBytes * (PRE ? 2 : 1));
        for (int l = 0; l < L::kLoads; l++) tma_load_2d(cur + l * L::kBoxRows * kTilePW, &maps[0], gx, gy + l * L::kBoxRows, bar);
        if (PRE)
            for (int l = 0; l < L::kLoads; l++) tma_load_2d(smem + L::kOffPre0 + l * L::kBoxRows * kTilePW, &maps_pre[0], gx, gy + l * L::kBoxRows, bar);
        // frame 0 is compared with itself: the compare buffers are free, fill them with the following frames now
        for (int b = 0; b < NBUF && 1 + b < p.nf; b++)
        {
            mbar_expect_tx(bar + 1 + b, L::kTileBytes * (PRE ? 2 : 1));
            for (int l = 0; l < L::kLoads; l++)
                tma_load_2d(smem + L::kOffCmp + b * L::kTileBytes + l * L::kBoxRows * kTilePW, &maps[1 + b], gx, gy + l * L::kBoxRows, bar + 1 + b);
            if (PRE)
                for (int l = 0; l < L::kLoads; l++)
                    tma_load_2d(smem + L::kOffCmpPre + l * L::kBoxRows * kTilePW, &maps_pre[1 + b], gx, gy + l * L::kBoxRows, bar + 1 + b);
        }
    }
    for (int i = tid; i < kLutEntries * 32; i += kThreads)
    {
        const int e = i >> 5;
        lut[i] = e < HBCU_NLMEANS_EXPSIZE ? p.exptable[e] : 0.f;
    }

    const int seg_y0 = warp * RS;
    int rows = p.h - (Y0 + seg_y0);                                     // rows of this warp's strip inside the plane
    rows = rows < 0 ? 0 : (rows > RS ? RS : rows);
    // range 3 without prefilter: frame 0 is one symmetric march (V3Sym) that stores every accumulator row it owns
    const bool sym = SYM && p.r_half == 1;
    V3Acc acc;
    float *acc_ws = reinterpret_cast<float *>(smem + L::kOffWs);
    float *acc_ps = reinterpret_cast<float *>(smem + L::kOffPs);
    if (!sym)
        for (int i = tid; i < L::kTH * kTileW; i += kThreads)
        {
            acc_ws[i] = 0.f;
            acc_ps[i] = 0.f;
        }
    acc.ws = acc_ws + seg_y0 * kTileW + lane * 4;
    acc.ps = acc_ps + seg_y0 * kTileW + lane * 4;
    mbar_wait(bar, 0);
    __syncthreads();

    const float wscale = p.wfact * 0.0078125f;                         // wfact / 128, exact
    const float wbias  = -8388608.0f * wscale;                         // exact (power-of-two scaling)
    // shared address of this lane's copy of table entry 0, pre-biased by -(0x47800000 << 7)
    const uint32_t lut_lane_addr = smem_u32(lut) + (uint32_t)lane * 4u - (0x47800000u << 7);
    const uint32_t *cw = reinterpret_cast<const uint32_t *>(cur);
    const uint32_t *pre0w = reinterpret_cast<const uint32_t *>(smem + L::kOffPre0);
    // the source patches: the pre-denoised current tile -- or the plain one where the reference's pointer is stale
    // (KernelParams::src_pre, the first frame of a stream)
    const uint32_t *srcw = (PRE && p.src_pre != p.planes[0]) ? pre0w : cw;
    for (int f = 0; f < p.nf; f++)
    {
        const uint32_t *bw = cw;
        const int buf = (f - 1) % NBUF;
        if (f > 0)
        {
            mbar_wait(bar + 1 + buf, (uint32_t)(((f - 1) / NBUF) & 1));
            bw = reinterpret_cast<const uint32_t *>(smem + L::kOffCmp + buf * L::kTileBytes);
        }
        // the tile the patch distances compare against: the pre-denoised twin of `bw` in the prefilter variant
        const uint32_t *bd = !PRE ? bw : (f == 0 ? pre0w : reinterpret_cast<const uint32_t *>(smem + L::kOffCmpPre));
        constexpr bool kExact = RS % (2 * NH + 1) == 0;                 // then partial strips run to their end (rows beyond the plane are never stored)
        const int nrows = kExact ? RS : rows;
        if constexpr (SYM)
        {
            if (sym && f == 0)
            {
                // every row the later frames' marches read and write (nrows) is stored here
                if (rows > 0) V3Sym<NH, V3Acc>(cw, acc, lut_lane_addr, wscale, wbias, p.origin_tune, seg_y0, lane).run(nrows);
                continue;
            }
        }
        if (rows > 0)
        {
            for (int dy = -p.r_half; dy <= p.r_half; dy++)
            {
                for (int dx0 = -p.r_half; dx0 <= p.r_half; dx0 += kGroup)
                {
                    const int ng  = min(kGroup, p.r_half - dx0 + 1);
                    const int org = (f == 0 && dy == 0 && dx0 <= 0 && dx0 + ng > 0) ? -dx0 : kOrgNone;
                    const int ob  = (12 + dx0) & 3;
#define X(NG_, OB_, ORG_)                                                                                                   \
                    if (ng == NG_ && ob == OB_ && org == ORG_)                                                              \
                        v3_group<NH, NG_, OB_, ORG_, kExact, PRE>(srcw, bd, bw, cw, acc, lut_lane_addr, wscale, wbias, p.origin_tune, seg_y0, nrows, lane, dy, dx0); \
                    else
                    V3_GROUP_SHAPES(X)
#undef X
                    { /* unreachable: the launcher checked v3_group_known() for every group of this range */ }
                }
            }
        }
        // the buffer just read takes frame f + NBUF (uniform condition: every warp reaches the barrier)
        if (f > 0 && f + NBUF < p.nf)
        {
            __syncthreads();
            if (tid == 0)
            {
                fence_proxy_async();
                mbar_expect_tx(bar + 1 + buf, L::kTileBytes * (PRE ? 2 : 1));
                for (int l = 0; l < L::kLoads; l++)
                    tma_load_2d(smem + L::kOffCmp + buf * L::kTileBytes + l * L::kBoxRows * kTilePW, &maps[f + NBUF], gx, gy + l * L::kBoxRows, bar + 1 + buf);
                if (PRE)
                    for (int l = 0; l < L::kLoads; l++)
                        tma_load_2d(smem + L::kOffCmpPre + l * L::kBoxRows * kTilePW, &maps_pre[f + NBUF], gx, gy + l * L::kBoxRows, bar + 1 + buf);
            }
        }
    }

    const int x = lane * 4;
    uint8_t *dst = reinterpret_cast<uint8_t *>(p.dst);
    for (int r = 0; r < rows; r++)
    {
        const int oy = seg_y0 + r;
        const int y = Y0 + oy;
        uint32_t accv[8];
        acc.load(r, accv);
        acc.wait_load(accv);
        const uint32_t cwd = cw[(oy + kHalo) * (kTilePW / 4) + lane + kHaloX / 4];
        uint8_t o[4];
#pragma unroll
        for (int i = 0; i < 4; i++)
            o[i] = finish_pixel<uint8_t>(__uint_as_float(accv[v3_acc_slot(i)]), __uint_as_float(accv[4 + v3_acc_slot(i)]), (uint8_t)((cwd >> (8 * i)) & 0xffu));
        uint8_t *drow = dst + (size_t)y * p.dpitch + X0 + x;
        if (X0 + x + 3 < p.w)
            *reinterpret_cast<uchar4 *>(drow) = make_uchar4(o[0], o[1], o[2], o[3]);
        else
        {
#pragma unroll
            for (int i = 0; i < 4; i++)
                if (X0 + x + i < p.w) drow[i] = o[i];
        }
    }
}

// Range 3 with one or two frames, patch 3 .. 7, no prefilter: the whole filter of a strip in one march (nlmeans_v3f_kernel).
// Frame 0 is V3Sym's march.  Frame 1 keeps the running sums of its nine displacements in registers and, like V3Sym,
// recomputes the patch-row sum leaving each of them from the tiles instead of keeping a history; the source words of
// the entering and the leaving row are the ones V3Sym has just loaded.  The terms of an output pixel are added in
// registers in the reference's order -- frame 0's nine as V3Sym adds them, then frame 1's, dy = -1, 0, +1 each with
// dx = -1, 0, +1, one IEEE operation each -- and the pixel is finished and stored at once: no accumulators in shared
// memory, so the tile is as tall as the registers allow and the strip's one warm-up is spread over twice the rows.
template <int NH, int NF>
struct V3Fused
{
    using Sym = V3Sym<NH, V3Acc>;
    static constexpr int PW = kTilePW / 4;           // tile pitch in words
    static_assert(NF == 1 || NF == 2, "frame count");

    Sym sym;
    uint32_t V1[3][3][4];                            // frame 1: 2^23-biased running sums of (dy, dx) at pixels x .. x+3
    float pix1[3][6];                                // frame 1: pixels x-1 .. x+4 of a compare row, slots as Sym::pix
    const uint32_t *cbase;                           // compare tile word `lane` of output row 0
    uint8_t *drow;                                   // output row 0 at pixel x
    int dpitch, xleft;                               // plane pixels from x on

    __device__ __forceinline__ V3Fused(const uint32_t *cur, const uint32_t *cmp, const V3Acc &none, uint32_t lut_lane_addr, float wscale,
                                       float wbias, double origin_tune, int seg_y0, int lane, uint8_t *drow_, int dpitch_, int xleft_)
        : sym(cur, none, lut_lane_addr, wscale, wbias, origin_tune, seg_y0, lane), drow(drow_), dpitch(dpitch_), xleft(xleft_)
    {
        cbase = cmp + (seg_y0 + kHalo) * PW + lane;
    }

    // frame-1 patch-row sums of source row t (words a: lane+3 .. lane+5) against compare row t + dy (words q: lane+2 ..
    // lane+6) for dx = -1, 0, +1: the compare stream one column left, in place and one column right
    static __device__ __forceinline__ void row_sums1(const uint32_t (&a)[3], const uint32_t (&q)[5], uint32_t (&h)[3][4])
    {
        uint32_t D[3][3];
#pragma unroll
        for (int w = 0; w < 3; w++)
        {
            D[0][w] = __vabsdiffu4(a[w], __funnelshift_r(q[w], q[w + 1], 24));
            D[1][w] = __vabsdiffu4(a[w], q[w + 1]);
            D[2][w] = __vabsdiffu4(a[w], __funnelshift_r(q[w + 1], q[w + 2], 8));
        }
#pragma unroll
        for (int dx = 0; dx < 3; dx++) Sym::template windows<0>(D[dx], h[dx], std::make_integer_sequence<int, 4>{});
    }

    __device__ __forceinline__ void cmp_words(int row, uint32_t (&q)[5]) const
    {
#pragma unroll
        for (int k = 0; k < 5; k++) q[k] = cbase[row * PW + 2 + k];
    }

    template <int S>
    __device__ __forceinline__ void load_pixels1(int row)
    {
        const uint32_t *w = cbase + row * PW + 3;
        const uint32_t w0 = w[0], w1 = w[1], w2 = w[2];
        pix1[S][0] = __fadd_rn(byte_as_biased_float(w0, 3), -8388608.0f);
#pragma unroll
        for (int i = 0; i < 4; i++) pix1[S][1 + i] = __fadd_rn(byte_as_biased_float(w1, i), -8388608.0f);
        pix1[S][5] = __fadd_rn(byte_as_biased_float(w2, 0), -8388608.0f);
    }

    // frame 1 moves from output row r-1 to r: patch rows r+NH (source words in Sym::qi[Q]) enter, r-NH-1 (Sym::qo[Q]) leave
    template <int Q>
    __device__ __forceinline__ void advance1(int r)
    {
        const uint32_t ai[3] = { sym.qi[Q][1], sym.qi[Q][2], sym.qi[Q][3] };
        const uint32_t ao[3] = { sym.qo[Q][1], sym.qo[Q][2], sym.qo[Q][3] };
#pragma unroll
        for (int dy = 0; dy < 3; dy++)
        {
            uint32_t q[5], hi[3][4], ho[3][4];
            cmp_words(r + NH + dy - 1, q);
            row_sums1(ai, q, hi);
            cmp_words(r - NH - 2 + dy, q);
            row_sums1(ao, q, ho);
#pragma unroll
            for (int dx = 0; dx < 3; dx++)
#pragma unroll
                for (int i = 0; i < 4; i++) V1[dy][dx][i] = V1[dy][dx][i] + hi[dx][i] - ho[dx][i];
        }
    }

    // output row r in slot K (Sym's slots)
    template <int K>
    __device__ __forceinline__ void step(int r)
    {
        float ws[4], ps[4];
        sym.template terms<K>(r, ws, ps);
        if constexpr (NF == 2)
        {
            constexpr int Q = 1 - K % 2;
            constexpr int S[3] = { (K + 1) % 3, (K + 2) % 3, K % 3 };            // compare pixel rows r-1, r, r+1
            advance1<Q>(r);
            load_pixels1<S[2]>(r + 1);
#pragma unroll
            for (int dy = 0; dy < 3; dy++)
#pragma unroll
                for (int dx = 0; dx < 3; dx++)
#pragma unroll
                    for (int i = 0; i < 4; i++)
                    {
                        const float w = sym.weight(V1[dy][dx][i]);
                        ws[i] = __fadd_rn(ws[i], w);
                        ps[i] = __fadd_rn(ps[i], __fmul_rn(w, pix1[S[dy]][i + dx]));
                    }
        }
        const uint32_t cwd = sym.base[r * PW + kHaloX / 4];
        uint8_t o[4];
#pragma unroll
        for (int i = 0; i < 4; i++) o[i] = finish_pixel<uint8_t>(ws[i], ps[i], (uint8_t)((cwd >> (8 * i)) & 0xffu));
        uint8_t *d = drow + (size_t)r * dpitch;
        if (xleft >= 4)
            *reinterpret_cast<uchar4 *>(d) = make_uchar4(o[0], o[1], o[2], o[3]);
        else
        {
#pragma unroll
            for (int i = 0; i < 4; i++)
                if (i < xleft) d[i] = o[i];
        }
    }

    template <int... Ms>
    __device__ __forceinline__ void rows_from(int r0, int rows, std::integer_sequence<int, Ms...>)
    {
        ((r0 + Ms < rows ? step<(Ms + 1) % 6>(r0 + Ms) : (void)0), ...);
    }

    __device__ __forceinline__ void run(int rows)
    {
        sym.start();
        if constexpr (NF == 2)
        {
            // the state of output row -1, as Sym's: the sums of patch rows -NH-1 .. NH-1, compare pixel rows -1 and 0
#pragma unroll
            for (int dy = 0; dy < 3; dy++)
#pragma unroll
                for (int dx = 0; dx < 3; dx++)
#pragma unroll
                    for (int i = 0; i < 4; i++) V1[dy][dx][i] = kVBias;
#pragma unroll 1
            for (int t = -NH - 1; t < NH; t++)
            {
                const uint32_t *s = sym.base + t * PW + 3;
                const uint32_t a[3] = { s[0], s[1], s[2] };
#pragma unroll
                for (int dy = 0; dy < 3; dy++)
                {
                    uint32_t q[5], h[3][4];
                    cmp_words(t + dy - 1, q);
                    row_sums1(a, q, h);
#pragma unroll
                    for (int dx = 0; dx < 3; dx++)
#pragma unroll
                        for (int i = 0; i < 4; i++) V1[dy][dx][i] += h[dx][i];
                }
            }
            load_pixels1<2>(-1);
            load_pixels1<0>(0);
        }
#pragma unroll 1
        for (int r0 = 0; r0 < rows; r0 += 6) rows_from(r0, rows, std::make_integer_sequence<int, 6>{});
    }
};

// Shared memory of nlmeans_v3f_kernel: the current tile, one compare tile, the weight table
template <int NW, int RS>
struct V3FusedLayout
{
    static constexpr int kTH        = NW * RS;
    static constexpr int kLoads     = (kTH + 2 * kHalo + 255) / 256;                    // a TMA box has at most 256 rows
    static constexpr int kBoxRows   = ((kTH + 2 * kHalo + kLoads - 1) / kLoads + 3) / 4 * 4;
    static constexpr int kTileBytes = kBoxRows * kLoads * kTilePW;
    static constexpr int kLutBytes  = kLutEntries * 32 * (int)sizeof(float);
    static constexpr int kOffCur    = 0;
    static constexpr int kOffCmp    = kOffCur + kTileBytes;
    static constexpr int kOffLut    = kOffCmp + kTileBytes;
    static constexpr int kOffBar    = kOffLut + kLutBytes;                               // 2 mbarriers
    static constexpr int kTotal     = kOffBar + 64;
    static_assert(kBoxRows <= 256, "TMA box rows");
    static_assert((kBoxRows * kTilePW) % 128 == 0, "TMA destination must stay 128-byte aligned");
    static_assert(kTotal <= 227 * 1024, "shared memory");
};

// Every plane of the launch at range 3 with nf <= 2, patch 3 .. 7 and no prefilter (launch_v3f): V3Fused per strip.
template <int NH, int NW, int RS>
__global__ void __launch_bounds__(NW * 32, 1) nlmeans_v3f_kernel(const __grid_constant__ FusedParams fp)
{
    static_assert(NH >= 1 && NH <= 3, "patch 3 .. 7");
    constexpr int kThreads = NW * 32;
    using L = V3FusedLayout<NW, RS>;
    int pl = 0;
    while (pl + 1 < fp.nplanes && (int)blockIdx.x >= fp.first_tile[pl + 1]) pl++;
    const KernelParams &p = fp.k[pl];
    const CUtensorMap *maps = fp.maps[pl];
    const int tile = (int)blockIdx.x - fp.first_tile[pl];
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t *cur  = smem + L::kOffCur;
    uint8_t *cmp  = smem + L::kOffCmp;
    float *lut    = reinterpret_cast<float *>(smem + L::kOffLut);
    uint64_t *bar = reinterpret_cast<uint64_t *>(smem + L::kOffBar);           // [0] current tile, [1] compare tile

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int X0 = (tile % fp.tiles_x[pl]) * kTileW, Y0 = (tile / fp.tiles_x[pl]) * L::kTH;
    const int gx = X0 + kBorder - kHaloX, gy = Y0 + kBorder - kHalo;

    if (tid == 0)
    {
        mbar_init(bar, 1);
        mbar_init(bar + 1, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid == 0)
    {
        mbar_expect_tx(bar, L::kTileBytes);
        for (int l = 0; l < L::kLoads; l++) tma_load_2d(cur + l * L::kBoxRows * kTilePW, &maps[0], gx, gy + l * L::kBoxRows, bar);
        if (p.nf > 1)
        {
            mbar_expect_tx(bar + 1, L::kTileBytes);
            for (int l = 0; l < L::kLoads; l++) tma_load_2d(cmp + l * L::kBoxRows * kTilePW, &maps[1], gx, gy + l * L::kBoxRows, bar + 1);
        }
    }
    for (int i = tid; i < kLutEntries * 32; i += kThreads)
    {
        const int e = i >> 5;
        lut[i] = e < HBCU_NLMEANS_EXPSIZE ? p.exptable[e] : 0.f;
    }

    const int seg_y0 = warp * RS;
    int rows = p.h - (Y0 + seg_y0);                                     // rows of this warp's strip inside the plane
    rows = rows < 0 ? 0 : (rows > RS ? RS : rows);
    mbar_wait(bar, 0);
    __syncthreads();
    if (rows == 0) return;

    const float wscale = p.wfact * 0.0078125f;                         // wfact / 128, exact
    const float wbias  = -8388608.0f * wscale;                         // exact (power-of-two scaling)
    // shared address of this lane's copy of table entry 0, pre-biased by -(0x47800000 << 7)
    const uint32_t lut_lane_addr = smem_u32(lut) + (uint32_t)lane * 4u - (0x47800000u << 7);
    const uint32_t *cw = reinterpret_cast<const uint32_t *>(cur);
    const uint32_t *bw = reinterpret_cast<const uint32_t *>(cmp);
    const V3Acc none = { nullptr, nullptr };
    uint8_t *drow = reinterpret_cast<uint8_t *>(p.dst) + (size_t)(Y0 + seg_y0) * p.dpitch + X0 + lane * 4;
    const int xleft = p.w - (X0 + lane * 4);
    if (p.nf == 1)
        V3Fused<NH, 1>(cw, bw, none, lut_lane_addr, wscale, wbias, p.origin_tune, seg_y0, lane, drow, p.dpitch, xleft).run(rows);
    else
    {
        mbar_wait(bar + 1, 0);
        V3Fused<NH, 2>(cw, bw, none, lut_lane_addr, wscale, wbias, p.origin_tune, seg_y0, lane, drow, p.dpitch, xleft).run(rows);
    }
}


// ---------------------------------------------------------------------------------------------------------------------
// 16-bit samples (yuv420p10 planes; every sample <= kFast16Max = 1023, checked by the border kernel -- see
// nlmeans_fast16_kernel for the contract and the integer stand-in that takes over otherwise).
//
// Same march as the 8-bit group: a lane owns 4 adjacent pixels and walks down its strip with the vertical running sum V
// of horizontal patch-row sums in registers.  The squared differences have no packed-integer instruction at this width;
// they are fp32 integers instead -- every value stays below 2^24, so every add/fma is exact in ANY order, which frees the
// grouping: the four windows of a row share their middle (27 fp32 operations per displacement and row instead of a
// 10-long prefix chain plus window differences).  V is a plain integer here
// (49 x 1023^2 does not fit the 2^23-biased-float trick of the 8-bit kernel): I2FP + FMUL.SAT.
// The compare pixels of the output row are re-read from shared memory (no 7-row delay line of words in registers).
template <int NH, int NG, int OB, int ORG, class ACC>
struct V3Group16
{
    static constexpr int N    = 2 * NH + 1;
    static constexpr int PW   = kTilePW / 2;          // tile pitch in words (two samples each)
    static constexpr int NA   = 4 + 2 * NH;           // source samples per row
    static constexpr int NB   = NA + NG - 1;          // compare samples per row
    static constexpr int OA   = (kHaloX - NH) & 3;    // sample offset of a[0] inside its first quad
    static constexpr int FB   = (OB - NH) & 3;        // sample offset of b[0] inside its first quad (OB = (12 + dx0) & 3)
    static constexpr int NWA  = (OA + NA + 1) / 2;    // words covering the source window
    static constexpr int NWB  = (FB + NB + 1) / 2;
    static constexpr int OP   = OB & 3;               // the output row's compare pixels start at sample kHaloX + dx0 of the row
    static constexpr int NWP  = (OP + NG + 3 + 1) / 2;
    static constexpr float kBias = 8388608.0f;
    static_assert(NH >= 1 && NH <= 3, "patch-row sums must stay below 2^23");

    int      V[NG][4];
    uint32_t hist[N][NG][4];                          // patch-row sums as bits of (2^23 + sum): the biases cancel in V
    const uint32_t *arow, *brow, *prow, *orow;
    const ACC &acc;
    uint32_t lut_lane_addr;
    float wscale;
    double origin_tune;

    __device__ __forceinline__ V3Group16(const uint32_t *cur, const uint32_t *cmp, const ACC &acc_, uint32_t lut_lane_addr_, float wscale_,
                                         double origin_tune_, int seg_y0, int lane, int dy, int dx0)
        : acc(acc_), lut_lane_addr(lut_lane_addr_), wscale(wscale_), origin_tune(origin_tune_)
    {
#pragma unroll
        for (int g = 0; g < NG; g++)
#pragma unroll
            for (int i = 0; i < 4; i++)
            {
                V[g][i] = 0;
#pragma unroll
                for (int k = 0; k < N; k++) hist[k][g][i] = kVBias;
            }
        const int fa = kHaloX - NH, fb = kHaloX - NH + dx0, fp = kHaloX + dx0;      // first sample of each window, relative to 4 * lane
        arow = cur + (seg_y0 - NH + kHalo) * PW + 2 * lane + 2 * (fa >> 2);
        brow = cmp + (seg_y0 - NH + kHalo + dy) * PW + 2 * lane + 2 * (fb >> 2);
        prow = cmp + (seg_y0 + kHalo + dy) * PW + 2 * lane + 2 * (fp >> 2);
        orow = cur + (seg_y0 + kHalo) * PW + 2 * lane + kHaloX / 2;
    }

    static __device__ __forceinline__ bool is_origin(int g) { return ORG >= 0 && g == ORG; }

    template <int K, bool OUT>
    __device__ __forceinline__ void step(int r)
    {
        uint32_t wa[NWA], wb[NWB];
#pragma unroll
        for (int j = 0; j < NWA; j++) wa[j] = arow[j];
#pragma unroll
        for (int j = 0; j < NWB; j++) wb[j] = brow[j];
        arow += PW;
        brow += PW;
        uint32_t accv[8];
        if (OUT) acc.load(r, accv);
        float a[NA], b[NB];
#pragma unroll
        for (int j = 0; j < NA; j++) a[j] = half_as_biased_float(wa[(OA + j) >> 1], (OA + j) & 1);
#pragma unroll
        for (int j = 0; j < NB; j++) b[j] = half_as_biased_float(wb[(FB + j) >> 1], (FB + j) & 1);

        // hs[i] = sum of d^2 over samples i .. i + 2NH of the row = the common middle M (samples 3 .. 2NH, carrying the
        // 2^23 bias of the stored sums) + L[i] (samples i .. 2, i <= 2) + R[i - 1] (samples 2NH+1 .. 2NH+i, i >= 1).
        // Every value is an integer below 2^24: all of it is exact in any order.
#pragma unroll
        for (int g = 0; g < NG; g++)
        {
            if (ORG != kOrgNone && is_origin(g)) continue;
            float d[NA];
#pragma unroll
            for (int j = 0; j < NA; j++) d[j] = __fsub_rn(a[j], b[j + g]);          // exact: both are 2^23 + sample
            float M = kBias;
#pragma unroll
            for (int j = 3; j <= 2 * NH; j++) M = __fmaf_rn(d[j], d[j], M);
            float L[3], R[3];
            L[2] = __fmul_rn(d[2], d[2]);
            L[1] = __fmaf_rn(d[1], d[1], L[2]);
            L[0] = __fmaf_rn(d[0], d[0], L[1]);
            R[0] = __fmul_rn(d[2 * NH + 1], d[2 * NH + 1]);
            R[1] = __fmaf_rn(d[2 * NH + 2], d[2 * NH + 2], R[0]);
            R[2] = __fmaf_rn(d[2 * NH + 3], d[2 * NH + 3], R[1]);
#pragma unroll
            for (int i = 0; i < 4; i++)
            {
                float h = M;
                if (i <= 2) h = __fadd_rn(h, L[i]);
                if (i >= 1) h = __fadd_rn(h, R[i - 1]);
                const uint32_t hb = __float_as_uint(h);
                V[g][i] = V[g][i] + (int)hb - (int)hist[K][g][i];
                hist[K][g][i] = hb;
            }
        }
        if (OUT)
        {
            uint32_t wp[NWP];
#pragma unroll
            for (int j = 0; j < NWP; j++) wp[j] = prow[r * PW + j];
            float2 pix2[NG + 1];                          // (compare pixel j, compare pixel j + 2) as floats
#pragma unroll
            for (int j = 0; j < NG + 1; j++)
                pix2[j] = v3_add2(v3_pack2(half_as_biased_float(wp[(OP + j) >> 1], (OP + j) & 1),
                                           half_as_biased_float(wp[(OP + j + 2) >> 1], (OP + j + 2) & 1)),
                                  v3_pack2(-kBias, -kBias));
            acc.wait_load(accv);
            float2 W[NG][2];
#pragma unroll
            for (int g = 0; g < NG; g++)
            {
                if (ORG != kOrgNone && is_origin(g)) continue;
                float t[4];
#pragma unroll
                for (int i = 0; i < 4; i++)
                    asm("mul.rn.sat.f32 %0, %1, %2;" : "=f"(t[i]) : "f"(__int2float_rn(V[g][i])), "f"(wscale));
#pragma unroll
                for (int h = 0; h < 2; h++)
                {
                    float u0, u1, w0, w1;
                    v3_unpack2(v3_add2_rz(v3_pack2(t[h], t[h + 2]), v3_pack2(65536.0f, 65536.0f)), u0, u1);
                    asm("ld.shared.f32 %0, [%1];" : "=f"(w0) : "r"((__float_as_uint(u0) << 7) + lut_lane_addr));
                    asm("ld.shared.f32 %0, [%1];" : "=f"(w1) : "r"((__float_as_uint(u1) << 7) + lut_lane_addr));
                    W[g][h] = v3_pack2(w0, w1);
                }
            }
            float2 ws2[2], ps2[2];
#pragma unroll
            for (int h = 0; h < 2; h++)
            {
                ws2[h] = v3_pack2(__uint_as_float(accv[2 * h]), __uint_as_float(accv[2 * h + 1]));
                ps2[h] = v3_pack2(__uint_as_float(accv[4 + 2 * h]), __uint_as_float(accv[4 + 2 * h + 1]));
            }
#pragma unroll
            for (int g = 0; g < NG; g++)
            {
                if (ORG != kOrgNone && is_origin(g))
                {
                    const uint32_t c0 = orow[r * PW], c1 = orow[r * PW + 1];
#pragma unroll
                    for (int h = 0; h < 2; h++)
                    {
                        float wa_, wb_, pa, pb;
                        v3_unpack2(ws2[h], wa_, wb_);
                        v3_unpack2(ps2[h], pa, pb);
                        add_origin(wa_, pa, origin_tune, (int)((c0 >> (16 * h)) & 0xffffu));      // pixel h
                        add_origin(wb_, pb, origin_tune, (int)((c1 >> (16 * h)) & 0xffffu));      // pixel h + 2
                        ws2[h] = v3_pack2(wa_, wb_);
                        ps2[h] = v3_pack2(pa, pb);
                    }
                }
                else
                {
#pragma unroll
                    for (int h = 0; h < 2; h++)
                    {
                        ws2[h] = v3_add2(ws2[h], W[g][h]);
                        ps2[h] = v3_add2(ps2[h], v3_mul2(W[g][h], pix2[g + h]));
                    }
                }
            }
#pragma unroll
            for (int h = 0; h < 2; h++)
            {
                float x, y;
                v3_unpack2(ws2[h], x, y);
                accv[2 * h] = __float_as_uint(x); accv[2 * h + 1] = __float_as_uint(y);
                v3_unpack2(ps2[h], x, y);
                accv[4 + 2 * h] = __float_as_uint(x); accv[4 + 2 * h + 1] = __float_as_uint(y);
            }
            acc.store(r, accv);
        }
    }

    template <int... Ks>
    __device__ __forceinline__ void warm_up(std::integer_sequence<int, Ks...>) { (step<Ks, false>(0), ...); }
    template <int... Ms>
    __device__ __forceinline__ void rows_from(int r0, int rows, std::integer_sequence<int, Ms...>)
    {
        ((r0 + Ms < rows ? step<(2 * NH + Ms) % N, true>(r0 + Ms) : (void)0), ...);
    }
    __device__ __forceinline__ void run(int rows)
    {
        warm_up(std::make_integer_sequence<int, 2 * NH>{});
#pragma unroll 1
        for (int r0 = 0; r0 < rows; r0 += N) rows_from(r0, rows, std::make_integer_sequence<int, N>{});
        acc.wait_store();
    }
};

template <int NH, int NG, int OB, int ORG, class ACC>
__device__ __forceinline__ void v3_group16(const uint32_t *__restrict__ cur, const uint32_t *__restrict__ cmp, const ACC &acc,
                                           uint32_t lut_lane_addr, float wscale, double origin_tune,
                                           int seg_y0, int rows, int lane, int dy, int dx0)
{
    V3Group16<NH, NG, OB, ORG, ACC> g(cur, cmp, acc, lut_lane_addr, wscale, origin_tune, seg_y0, lane, dy, dx0);
    g.run(rows);
}

template <int NH, int NW, int RS, int NBUF>
__global__ void __launch_bounds__(NW * 32, 1) nlmeans_v3w_kernel(const __grid_constant__ FusedParams fp)
{
    if (*fp.range_flag != 0u) return;               // samples above 10 bit seen: the integer kernel takes over
    constexpr int kThreads = NW * 32;
    using L = V3Layout<NW, RS, NBUF, 2>;
    int pl = 0;
    while (pl + 1 < fp.nplanes && (int)blockIdx.x >= fp.first_tile[pl + 1]) pl++;
    const KernelParams &p = fp.k[pl];
    const CUtensorMap *maps = fp.maps[pl];
    const int tile = (int)blockIdx.x - fp.first_tile[pl];
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t *cur  = smem + L::kOffCur;
    float *lut    = reinterpret_cast<float *>(smem + L::kOffLut);
    uint64_t *bar = reinterpret_cast<uint64_t *>(smem + L::kOffBar);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int X0 = (tile % fp.tiles_x[pl]) * kTileW, Y0 = (tile / fp.tiles_x[pl]) * L::kTH;
    const int gx = X0 + kBorder - kHaloX, gy = Y0 + kBorder - kHalo;

    if (tid == 0)
    {
        for (int b = 0; b < 1 + NBUF; b++) mbar_init(bar + b, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid == 0)
    {
        mbar_expect_tx(bar, L::kTileBytes);
        for (int l = 0; l < L::kLoads; l++) tma_load_2d(cur + l * L::kBoxRows * L::kRowBytes, &maps[0], gx, gy + l * L::kBoxRows, bar);
        for (int b = 0; b < NBUF && 1 + b < p.nf; b++)
        {
            mbar_expect_tx(bar + 1 + b, L::kTileBytes);
            for (int l = 0; l < L::kLoads; l++)
                tma_load_2d(smem + L::kOffCmp + b * L::kTileBytes + l * L::kBoxRows * L::kRowBytes, &maps[1 + b], gx, gy + l * L::kBoxRows, bar + 1 + b);
        }
    }
    for (int i = tid; i < kLutEntries * 32; i += kThreads)
    {
        const int e = i >> 5;
        lut[i] = e < HBCU_NLMEANS_EXPSIZE ? p.exptable[e] : 0.f;
    }

    const int seg_y0 = warp * RS;
    int rows = p.h - (Y0 + seg_y0);
    rows = rows < 0 ? 0 : (rows > RS ? RS : rows);
    V3Acc acc;
    float *acc_ws = reinterpret_cast<float *>(smem + L::kOffWs);
    float *acc_ps = reinterpret_cast<float *>(smem + L::kOffPs);
    for (int i = tid; i < L::kTH * kTileW; i += kThreads)
    {
        acc_ws[i] = 0.f;
        acc_ps[i] = 0.f;
    }
    acc.ws = acc_ws + seg_y0 * kTileW + lane * 4;
    acc.ps = acc_ps + seg_y0 * kTileW + lane * 4;
    mbar_wait(bar, 0);
    __syncthreads();

    const float wscale = p.wfact * 0.0078125f;                         // wfact / 128, exact
    const uint32_t lut_lane_addr = smem_u32(lut) + (uint32_t)lane * 4u - (0x47800000u << 7);
    const uint32_t *cw = reinterpret_cast<const uint32_t *>(cur);
    for (int f = 0; f < p.nf; f++)
    {
        const uint32_t *bw = cw;
        const int buf = (f - 1) % NBUF;
        if (f > 0)
        {
            mbar_wait(bar + 1 + buf, (uint32_t)(((f - 1) / NBUF) & 1));
            bw = reinterpret_cast<const uint32_t *>(smem + L::kOffCmp + buf * L::kTileBytes);
        }
        if (rows > 0)
        {
            for (int dy = -p.r_half; dy <= p.r_half; dy++)
            {
                for (int dx0 = -p.r_half; dx0 <= p.r_half; dx0 += kGroup)
                {
                    const int ng  = min(kGroup, p.r_half - dx0 + 1);
                    const int org = (f == 0 && dy == 0 && dx0 <= 0 && dx0 + ng > 0) ? -dx0 : kOrgNone;
                    const int ob  = (12 + dx0) & 3;
#define X(NG_, OB_, ORG_)                                                                                                   \
                    if (ng == NG_ && ob == OB_ && org == ORG_)                                                              \
                        v3_group16<NH, NG_, OB_, ORG_>(cw, bw, acc, lut_lane_addr, wscale, p.origin_tune, seg_y0, rows, lane, dy, dx0); \
                    else
                    V3_GROUP_SHAPES(X)
#undef X
                    { /* unreachable: the launcher checked v3_group_known() for every group of this range */ }
                }
            }
        }
        if (f > 0 && f + NBUF < p.nf)
        {
            __syncthreads();
            if (tid == 0)
            {
                fence_proxy_async();
                mbar_expect_tx(bar + 1 + buf, L::kTileBytes);
                for (int l = 0; l < L::kLoads; l++)
                    tma_load_2d(smem + L::kOffCmp + buf * L::kTileBytes + l * L::kBoxRows * L::kRowBytes, &maps[f + NBUF], gx, gy + l * L::kBoxRows, bar + 1 + buf);
            }
        }
    }

    const int x = lane * 4;
    uint16_t *dst = reinterpret_cast<uint16_t *>(p.dst);
    const uint16_t *cur16 = reinterpret_cast<const uint16_t *>(cur);
    for (int r = 0; r < rows; r++)
    {
        const int oy = seg_y0 + r;
        const int y = Y0 + oy;
        uint32_t accv[8];
        acc.load(r, accv);
        acc.wait_load(accv);
        uint16_t o[4];
#pragma unroll
        for (int i = 0; i < 4; i++)
            o[i] = finish_pixel<uint16_t>(__uint_as_float(accv[v3_acc_slot(i)]), __uint_as_float(accv[4 + v3_acc_slot(i)]),
                                          cur16[(oy + kHalo) * kTilePW + x + kHaloX + i]);
        uint16_t *drow = dst + (size_t)y * p.dpitch + X0 + x;
        if (X0 + x + 3 < p.w)
            *reinterpret_cast<ushort4 *>(drow) = make_ushort4(o[0], o[1], o[2], o[3]);
        else
        {
#pragma unroll
            for (int i = 0; i < 4; i++)
                if (X0 + x + i < p.w) drow[i] = o[i];
        }
    }
}
