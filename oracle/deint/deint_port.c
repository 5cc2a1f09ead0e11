/* deint_port.c -- TEST INFRASTRUCTURE: plain-C stand-in for the hbcu_deint_* group of include/hbcu.h, for
 * libhostlogic_deint.so (deint.mk), so that hb_filter_yadif_cuda and hb_filter_bwdif_cuda (deinterlace_cuda.c, compiled
 * untouched) run their host side -- init, pass-through, refusals, the frame window, the field order and field-end state,
 * timestamps, props, EOF, buffer ownership -- on a machine without a GPU.
 *
 * The per-sample arithmetic of Yadif and Bwdif restated sample by sample from the table in DESIGN.md 4.9, with the names
 * used there.  Each call finishes before it returns.  Never linked into the product.
 */
#include "../../include/hbcu.h"

#include <stdlib.h>
#include <string.h>

void oracle_hostlogic_set_error(const char *fmt, ...);

struct hbcu_deint_s { hbcu_deint_config_t cfg; };

typedef struct { const uint8_t *b; int pitch, bytes; } src_t;

static int at(const src_t *s, int y, int x)
{
    const uint8_t *r = s->b + (size_t)y * s->pitch;
    return s->bytes == 1 ? r[x] : ((const uint16_t *)r)[x];
}

static int imax(int a, int b) { return a > b ? a : b; }
static int imin(int a, int b) { return a < b ? a : b; }
static int max3(int a, int b, int c) { return imax(a, imax(b, c)); }
static int min3(int a, int b, int c) { return imin(a, imin(b, c)); }
static int clamp_to(int v, int lo, int hi) { return v > hi ? hi : v < lo ? lo : v; }

/* prev, cur, next, prev2, next2 */
enum { PV, CU, NX, P2, N2 };

static int yadif(const src_t *S, int x, int y, int w, int h, int spatial)
{
    const int m = y ? -1 : 1, n = y + 1 < h ? 1 : -1;
    const int c = at(&S[CU], y + m, x), e = at(&S[CU], y + n, x);
    const int d = (at(&S[P2], y, x) + at(&S[N2], y, x)) >> 1;
    const int td0 = abs(at(&S[P2], y, x) - at(&S[N2], y, x));
    const int td1 = (abs(at(&S[PV], y + m, x) - c) + abs(at(&S[PV], y + n, x) - e)) >> 1;
    const int td2 = (abs(at(&S[NX], y + m, x) - c) + abs(at(&S[NX], y + n, x) - e)) >> 1;
    int diff = max3(td0 >> 1, td1, td2);
    int pred = (c + e) >> 1;
    if (x >= 3 && x < w - 3)
    {
        int score = abs(at(&S[CU], y + m, x - 1) - at(&S[CU], y + n, x - 1)) + abs(c - e) +
                    abs(at(&S[CU], y + m, x + 1) - at(&S[CU], y + n, x + 1)) - 1;
        for (int side = -1; side <= 1; side += 2)
            for (int j = side; abs(j) <= 2; j += side)
            {
                int s = 0;
                for (int i = -1; i <= 1; i++)
                    s += abs(at(&S[CU], y + m, x + i + j) - at(&S[CU], y + n, x + i - j));
                if (s >= score) break;            /* CHECK(+-2) only after CHECK(+-1) improved the score */
                score = s;
                pred = (at(&S[CU], y + m, x + j) + at(&S[CU], y + n, x - j)) >> 1;
            }
    }
    if (spatial && y != 1 && y != h - 2)
    {
        const int b = (at(&S[P2], y + 2 * m, x) + at(&S[N2], y + 2 * m, x)) >> 1;
        const int f = (at(&S[P2], y + 2 * n, x) + at(&S[N2], y + 2 * n, x)) >> 1;
        diff = max3(diff, min3(d - e, d - c, imax(b - c, f - e)), -max3(d - e, d - c, imin(b - c, f - e)));
    }
    return clamp_to(pred, d - diff, d + diff);
}

static int bwdif(const src_t *S, int x, int y, int h, int intra, int df, int maxv)
{
    if (intra)
    {
        const int m = y > df - 1 ? -1 : 1, n = y + df < h ? 1 : -1;
        const int m3 = y > 3 * df - 1 ? -3 : 1, n3 = y + 3 * df < h ? 3 : -1;
        const int c = at(&S[CU], y + m, x), e = at(&S[CU], y + n, x);
        /* a row outside the plane (the row-step quirk on 4..6-row planes of 9-16-bit samples) is clamped to it */
        const int r3 = at(&S[CU], clamp_to(y + m3, 0, h - 1), x) + at(&S[CU], clamp_to(y + n3, 0, h - 1), x);
        return clamp_to((5077 * (c + e) - 981 * r3) >> 13, 0, maxv);
    }
    const int edge = y < 4 || y + 5 > h;
    const int m = edge ? (y > df - 1 ? -1 : 1) : -1, n = edge ? (y + df < h ? 1 : -1) : 1;
    const int c = at(&S[CU], y + m, x), e = at(&S[CU], y + n, x);
    const int p0 = at(&S[P2], y, x) + at(&S[N2], y, x);
    const int d = p0 >> 1;
    const int td0 = abs(at(&S[P2], y, x) - at(&S[N2], y, x));
    const int td1 = (abs(at(&S[PV], y + m, x) - c) + abs(at(&S[PV], y + n, x) - e)) >> 1;
    const int td2 = (abs(at(&S[NX], y + m, x) - c) + abs(at(&S[NX], y + n, x) - e)) >> 1;
    int diff = max3(td0 >> 1, td1, td2);
    if (diff == 0) return d;
    if (!edge || !(y < 2 || y + 3 > h))
    {
        const int b = ((at(&S[P2], y - 2, x) + at(&S[N2], y - 2, x)) >> 1) - c;
        const int f = ((at(&S[P2], y + 2, x) + at(&S[N2], y + 2, x)) >> 1) - e;
        diff = max3(diff, min3(d - e, d - c, imax(b, f)), -max3(d - e, d - c, imin(b, f)));
    }
    int interpol;
    if (edge)
        interpol = (c + e) >> 1;
    else
    {
        const int r3 = at(&S[CU], y - 3, x) + at(&S[CU], y + 3, x);
        if (abs(c - e) > td0)
        {
            const int p2 = at(&S[P2], y - 2, x) + at(&S[N2], y - 2, x) + at(&S[P2], y + 2, x) + at(&S[N2], y + 2, x);
            const int p4 = at(&S[P2], y - 4, x) + at(&S[N2], y - 4, x) + at(&S[P2], y + 4, x) + at(&S[N2], y + 4, x);
            interpol = (((5570 * p0 - 3801 * p2 + 1016 * p4) >> 2) + 4309 * (c + e) - 213 * r3) >> 13;
        }
        else
            interpol = (5077 * (c + e) - 981 * r3) >> 13;
    }
    return clamp_to(clamp_to(interpol, d - diff, d + diff), 0, maxv);
}

int oracle_hbcu_deint_create(hbcu_deint_t **out, const hbcu_deint_config_t *cfg)
{
    if ((cfg->algorithm != HBCU_DEINT_YADIF && cfg->algorithm != HBCU_DEINT_BWDIF) ||
        !((cfg->sample_bytes == 1 && cfg->depth == 8) || (cfg->sample_bytes == 2 && cfg->depth >= 9 && cfg->depth <= 16)))
    {
        oracle_hostlogic_set_error("deint_create: unsupported algorithm or sample format");
        return -1;
    }
    *out = calloc(1, sizeof(**out));
    (*out)->cfg = *cfg;
    return 0;
}

void oracle_hbcu_deint_destroy(hbcu_deint_t *h) { free(h); }

int oracle_hbcu_deint_frame(hbcu_deint_t *h, hbcu_frame_t *prev, hbcu_frame_t *cur, hbcu_frame_t *next, int tff, int spatial,
                            int npictures, hbcu_frame_t *const out[2], const int parity[2], const int intra[2])
{
    const hbcu_deint_config_t *g = &h->cfg;
    hbcu_frame_t *fr[3] = {prev, cur, next};
    for (int k = 0; k < npictures; k++)
        for (int p = 0; p < 3; p++)
        {
            src_t S[5];
            for (int f = 0; f < 3; f++)
                S[f] = (src_t){hbcu_frame_plane(fr[f], p), hbcu_frame_stride(fr[f], p), g->sample_bytes};
            const int par = parity[k] & 1, sel = par ^ (tff ? 1 : 0);
            S[P2] = sel ? S[PV] : S[CU];
            S[N2] = sel ? S[CU] : S[NX];
            uint8_t *dst = hbcu_frame_plane(out[k], p);
            const int ds = hbcu_frame_stride(out[k], p), w = g->width[p], hh = g->height[p];
            for (int y = 0; y < hh; y++)
                for (int x = 0; x < w; x++)
                {
                    int v = at(&S[CU], y, x);
                    if ((y ^ par) & 1)
                        v = g->algorithm == HBCU_DEINT_BWDIF
                                ? bwdif(S, x, y, hh, intra[k], g->sample_bytes, (1 << g->depth) - 1)
                                : yadif(S, x, y, w, hh, spatial);
                    if (g->sample_bytes == 1) dst[(size_t)y * ds + x] = (uint8_t)v;
                    else ((uint16_t *)(dst + (size_t)y * ds))[x] = (uint16_t)v;
                }
        }
    return 0;
}

int oracle_hbcu_deint_sync(hbcu_deint_t *h) { (void)h; return 0; }
int oracle_hbcu_deint_mark(hbcu_deint_t *h, int which) { (void)h; (void)which; return 0; }
int oracle_hbcu_deint_elapsed_ms(hbcu_deint_t *h, float *ms) { (void)h; *ms = 0; return 0; }
