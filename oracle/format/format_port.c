/* format_port.c -- TEST INFRASTRUCTURE: plain-C stand-in for the hbcu_format_* group of include/hbcu.h, for
 * libhostlogic_format.so (format.mk), so that hb_filter_format_cuda (format_cuda.c, compiled untouched) runs
 * its host side -- init, pass-through, refusals, props, EOF, buffer ownership -- on a machine without a GPU.
 *
 * The four conversions restated from FFmpeg's pixel-format descriptors, sample by sample:
 *   semi-planar -> planar   Y[x] = S0[x] >> shift;  Cb[x] = S1[2x] >> shift;  Cr[x] = S1[2x + 1] >> shift
 *   planar -> semi-planar   the reverse, << shift kept to the sample width
 * with shift 0 at 8 bits (NV12) and 6 at 10 bits (P010).  Each call finishes before it returns.  Never linked into the
 * product.
 */
#include "../../include/hbcu.h"

#include <stdlib.h>
#include <string.h>

void oracle_hostlogic_set_error(const char *fmt, ...);

struct hbcu_format_s { hbcu_format_config_t cfg; };

int oracle_hbcu_format_create(hbcu_format_t **out, const hbcu_format_config_t *cfg)
{
    if (cfg->width < 1 || cfg->height < 1 || (cfg->depth != 8 && cfg->depth != 10))
    {
        oracle_hostlogic_set_error("format_create: unsupported geometry or depth");
        return -1;
    }
    *out = calloc(1, sizeof(**out));
    (*out)->cfg = *cfg;
    return 0;
}

void oracle_hbcu_format_destroy(hbcu_format_t *h) { free(h); }

static unsigned get(const uint8_t *row, int i, int bps) { return bps == 1 ? row[i] : ((const uint16_t *)row)[i]; }
static void put(uint8_t *row, int i, int bps, unsigned v)
{
    if (bps == 1) row[i] = (uint8_t)v;
    else ((uint16_t *)row)[i] = (uint16_t)v;
}

int oracle_hbcu_format_convert(hbcu_format_t *h, int64_t ticket,
                               hbcu_frame_t *in_frame, const void *const in_planes[3], const int in_strides[3],
                               hbcu_frame_t *out_frame, void *const out_planes[3], const int out_strides[3])
{
    (void)ticket;
    const uint8_t *src[3];
    uint8_t *dst[3];
    int ss[3], ds[3];
    for (int p = 0; p < 3; p++)
    {
        src[p] = in_frame ? hbcu_frame_plane(in_frame, p) : in_planes[p];
        ss[p]  = in_frame ? hbcu_frame_stride(in_frame, p) : in_strides[p];
        dst[p] = out_frame ? hbcu_frame_plane(out_frame, p) : out_planes[p];
        ds[p]  = out_frame ? hbcu_frame_stride(out_frame, p) : out_strides[p];
    }
    const int w = h->cfg.width, ht = h->cfg.height, cw = (w + 1) / 2, ch = (ht + 1) / 2;
    const int bps = h->cfg.depth > 8 ? 2 : 1, shift = h->cfg.depth > 8 ? 16 - h->cfg.depth : 0;
    const int up = h->cfg.to_semi_planar;
    for (int y = 0; y < ht; y++)
        for (int x = 0; x < w; x++)
        {
            const unsigned v = get(src[0] + (size_t)y * ss[0], x, bps);
            put(dst[0] + (size_t)y * ds[0], x, bps, up ? v << shift : v >> shift);
        }
    for (int y = 0; y < ch; y++)
        for (int x = 0; x < cw; x++)
        {
            if (up)
            {
                put(dst[1] + (size_t)y * ds[1], 2 * x,     bps, get(src[1] + (size_t)y * ss[1], x, bps) << shift);
                put(dst[1] + (size_t)y * ds[1], 2 * x + 1, bps, get(src[2] + (size_t)y * ss[2], x, bps) << shift);
            }
            else
            {
                put(dst[1] + (size_t)y * ds[1], x, bps, get(src[1] + (size_t)y * ss[1], 2 * x,     bps) >> shift);
                put(dst[2] + (size_t)y * ds[2], x, bps, get(src[1] + (size_t)y * ss[1], 2 * x + 1, bps) >> shift);
            }
        }
    return 0;
}

int oracle_hbcu_format_wait(hbcu_format_t *h, int64_t ticket) { (void)h; (void)ticket; return 0; }
int oracle_hbcu_format_poll(hbcu_format_t *h, int64_t ticket) { (void)h; (void)ticket; return 1; }
int oracle_hbcu_format_sync(hbcu_format_t *h) { (void)h; return 0; }
int oracle_hbcu_format_mark(hbcu_format_t *h, int which) { (void)h; (void)which; return 0; }
int oracle_hbcu_format_elapsed_ms(hbcu_format_t *h, float *ms) { (void)h; *ms = 0; return 0; }
