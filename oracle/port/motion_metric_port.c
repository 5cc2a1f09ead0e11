/* motion_metric_port.c -- TEST INFRASTRUCTURE: plain-C restatement of the x86 motion metric of libhb/motion_metric.c
 * and, on top of it, CPU stand-ins for the hbcu_motion_metric_* calls of the product's framerate shaper
 * (handbrake_b200/libhb/vfr_cuda.c; see hostlogic_nlmeans.c for the idea).
 *
 * Per 16x16 block a uint32 sum of squared gamma differences that wraps, the block sums added into a uint64; on the
 * fast path both images are first reduced 4x4 by nested rounding averages.  A slot keeps a copy of what the device
 * keeps (the reduced image, or the luma), and a result is computed when it is queued.  The shaper over these stand-ins
 * (oracle/_ref/libhostlogic_vfr.so) must reproduce the reference vfr's recorded outputs and metrics
 * (tests/test_vfr_gpu.py).  Never linked into the product.
 */
#include "../../include/hbcu.h"

#include <stdlib.h>
#include <string.h>

void oracle_hostlogic_set_error(const char *fmt, ...);
const void *const *oracle_hostlogic_frame_planes(const hbcu_frame_t *f);      /* hostlogic_frames.c */
const int *oracle_hostlogic_frame_strides(const hbcu_frame_t *f);

static uint64_t g_launches = 0;

struct hbcu_motion_metric_s
{
    hbcu_motion_metric_config_t cfg;
    unsigned *lut;
    unsigned maxv;
    int bps, w, h;                 /* the compared images' geometry */
    uint16_t **slot;               /* samples widened to 16 bits, w x h */
    int *filled;
    uint64_t *res;
};

static unsigned sample(const uint8_t *base, int stride, int bps, int x, int y)
{
    const uint8_t *row = base + (size_t)y * stride;
    return bps == 2 ? ((const uint16_t *)row)[x] : row[x];
}

static unsigned avg4(unsigned a, unsigned b, unsigned c, unsigned d)
{
    return (((a + b + 1) >> 1) + ((c + d + 1) >> 1) + 1) >> 1;
}

uint64_t oracle_hbcu_motion_metric_waits(void) { return 0; }
uint64_t oracle_hbcu_motion_metric_launches(void) { return g_launches; }

int oracle_hbcu_motion_metric_create(hbcu_motion_metric_t **out, const hbcu_motion_metric_config_t *cfg)
{
    if (cfg->width < 1 || cfg->height < 1 || cfg->depth < 8 || cfg->depth > 16 || cfg->slots < 2 || cfg->results < 1)
    {
        oracle_hostlogic_set_error("motion_metric_create: unsupported geometry");
        return -1;
    }
    struct hbcu_motion_metric_s *m = calloc(1, sizeof(*m));
    m->cfg = *cfg;
    m->maxv = (1u << cfg->depth) - 1;
    m->bps = cfg->depth > 8 ? 2 : 1;
    m->w = cfg->fast ? cfg->width / 4 : cfg->width;
    m->h = cfg->fast ? cfg->height / 4 : cfg->height;
    m->lut = malloc(sizeof(unsigned) * (m->maxv + 1));
    memcpy(m->lut, cfg->gamma_lut, sizeof(unsigned) * (m->maxv + 1));
    m->slot = calloc(cfg->slots, sizeof(*m->slot));
    m->filled = calloc(cfg->slots, sizeof(int));
    for (int s = 0; s < cfg->slots; s++) m->slot[s] = calloc((size_t)m->w * m->h + 1, sizeof(uint16_t));
    m->res = calloc(cfg->results, sizeof(uint64_t));
    *out = m;
    return 0;
}

void oracle_hbcu_motion_metric_destroy(hbcu_motion_metric_t *m)
{
    if (m == NULL) return;
    for (int s = 0; s < m->cfg.slots; s++) free(m->slot[s]);
    free(m->slot);
    free(m->filled);
    free(m->lut);
    free(m->res);
    free(m);
}

int oracle_hbcu_motion_metric_enqueue(hbcu_motion_metric_t *m, int slot, int a_slot, int result,
                                      hbcu_frame_t *frame, const void *luma, int stride)
{
    if (slot < 0 || slot >= m->cfg.slots || a_slot >= m->cfg.slots || a_slot == slot ||
        (a_slot >= 0 && (result < 0 || result >= m->cfg.results || !m->filled[a_slot])))
    {
        oracle_hostlogic_set_error("motion_metric_enqueue: bad argument");
        return -1;
    }
    const uint8_t *src = frame ? oracle_hostlogic_frame_planes(frame)[0] : luma;
    const int ss = frame ? oracle_hostlogic_frame_strides(frame)[0] : stride;
    uint16_t *dst = m->slot[slot];
    for (int y = 0; y < m->h; y++)
        for (int x = 0; x < m->w; x++)
        {
            unsigned v;
            if (m->cfg.fast)
            {
                unsigned s[4][4];
                for (int r = 0; r < 4; r++)
                    for (int c = 0; c < 4; c++) s[r][c] = sample(src, ss, m->bps, 4 * x + c, 4 * y + r);
                /* each quarter pairs its two columns' vertical pairs; the quarters combine left/right, top/bottom */
                v = avg4(avg4(s[0][0], s[1][0], s[0][1], s[1][1]), avg4(s[0][2], s[1][2], s[0][3], s[1][3]),
                         avg4(s[2][0], s[3][0], s[2][1], s[3][1]), avg4(s[2][2], s[3][2], s[2][3], s[3][3]));
            }
            else
            {
                v = sample(src, ss, m->bps, x, y);
            }
            dst[(size_t)y * m->w + x] = (uint16_t)v;
        }
    m->filled[slot] = 1;
    if (a_slot < 0) return 0;
    const uint16_t *a = m->slot[a_slot];
    /* the reduced images are packed; above 8 bits the reference walks them with half the pitch */
    const int pitch = m->cfg.fast && m->bps == 2 ? m->w / 2 : m->w;
    uint64_t sum = 0;
    for (int by = 0; by < m->h / 16; by++)
        for (int bx = 0; bx < m->w / 16; bx++)
        {
            uint32_t block = 0;
            for (int y = by * 16; y < by * 16 + 16; y++)
                for (int x = bx * 16; x < bx * 16 + 16; x++)
                {
                    const unsigned ia = a[(size_t)y * pitch + x], ib = dst[(size_t)y * pitch + x];
                    const int d = (int)m->lut[ia > m->maxv ? m->maxv : ia] - (int)m->lut[ib > m->maxv ? m->maxv : ib];
                    block += (uint32_t)(d * d);
                }
            sum += block;
        }
    if (m->w >= 16 && m->h >= 16) g_launches++;
    m->res[result] = sum;
    return 0;
}

int oracle_hbcu_motion_metric_result(hbcu_motion_metric_t *m, int result, uint64_t *sum)
{
    if (result < 0 || result >= m->cfg.results)
    {
        oracle_hostlogic_set_error("motion_metric_result: bad argument");
        return -1;
    }
    *sum = m->res[result];
    return 0;
}

int oracle_hbcu_motion_metric_sync(hbcu_motion_metric_t *m) { (void)m; return 0; }
int oracle_hbcu_motion_metric_mark(hbcu_motion_metric_t *m, int which) { (void)m; (void)which; return 0; }
int oracle_hbcu_motion_metric_elapsed_ms(hbcu_motion_metric_t *m, float *ms) { (void)m; *ms = 0; return 0; }
