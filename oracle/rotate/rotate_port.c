/* rotate_port.c -- TEST INFRASTRUCTURE: plain-C stand-in for the hbcu_rotate_* group of include/hbcu.h, for
 * libhostlogic_rotate.so (rotate.mk), so that hb_filter_rotate_cuda (rotate_cuda.c, compiled untouched) runs its host
 * side -- init, geometry and PAR, pass-through, refusals, props, EOF, buffer ownership -- on a machine without a GPU.
 *
 * The seven transforms restated element by element, each plane within its own size (an element is a sample, or a
 * Cb/Cr pair of a semi-planar chroma plane, elem_bytes wide).  For an input plane of pw x ph elements, output (x, y):
 *   HFLIP        in[y][pw-1-x]          VFLIP        in[ph-1-y][x]          180          in[ph-1-y][pw-1-x]
 *   CLOCK        in[ph-1-x][y]          CLOCK_FLIP   in[ph-1-x][pw-1-y]
 *   CCLOCK       in[x][pw-1-y]          CCLOCK_FLIP  in[x][y]
 * Each call finishes before it returns.  Never linked into the product.
 */
#include "../../include/hbcu.h"

#include <stdlib.h>
#include <string.h>

void oracle_hostlogic_set_error(const char *fmt, ...);

struct hbcu_rotate_s { hbcu_rotate_config_t cfg; };

int oracle_hbcu_rotate_create(hbcu_rotate_t **out, const hbcu_rotate_config_t *cfg)
{
    if (cfg->transform < HBCU_ROTATE_HFLIP || cfg->transform > HBCU_ROTATE_CCLOCK_FLIP || cfg->planes < 2 || cfg->planes > 3)
    {
        oracle_hostlogic_set_error("rotate_create: unsupported transform or plane count");
        return -1;
    }
    for (int p = 0; p < cfg->planes; p++)
        if (cfg->width[p] < 1 || cfg->height[p] < 1 || cfg->elem_bytes[p] < 1 || cfg->elem_bytes[p] > 4)
        {
            oracle_hostlogic_set_error("rotate_create: unsupported plane geometry");
            return -1;
        }
    *out = calloc(1, sizeof(**out));
    (*out)->cfg = *cfg;
    return 0;
}

void oracle_hbcu_rotate_destroy(hbcu_rotate_t *h) { free(h); }

int oracle_hbcu_rotate_frame(hbcu_rotate_t *h, int64_t ticket,
                             hbcu_frame_t *in_frame, const void *const in_planes[3], const int in_strides[3],
                             hbcu_frame_t *out_frame, void *const out_planes[3], const int out_strides[3])
{
    (void)ticket;
    const int t = h->cfg.transform;
    const int transpose = t >= HBCU_ROTATE_CLOCK;
    for (int p = 0; p < h->cfg.planes; p++)
    {
        const uint8_t *src = in_frame ? hbcu_frame_plane(in_frame, p) : in_planes[p];
        const int ss       = in_frame ? hbcu_frame_stride(in_frame, p) : in_strides[p];
        uint8_t *dst       = out_frame ? hbcu_frame_plane(out_frame, p) : out_planes[p];
        const int ds       = out_frame ? hbcu_frame_stride(out_frame, p) : out_strides[p];
        const int pw = h->cfg.width[p], ph = h->cfg.height[p], e = h->cfg.elem_bytes[p];
        const int ow = transpose ? ph : pw, oh = transpose ? pw : ph;
        for (int y = 0; y < oh; y++)
            for (int x = 0; x < ow; x++)
            {
                int sx, sy;
                switch (t)
                {
                    case HBCU_ROTATE_HFLIP:       sx = pw - 1 - x; sy = y;          break;
                    case HBCU_ROTATE_VFLIP:       sx = x;          sy = ph - 1 - y; break;
                    case HBCU_ROTATE_180:         sx = pw - 1 - x; sy = ph - 1 - y; break;
                    case HBCU_ROTATE_CLOCK:       sx = y;          sy = ph - 1 - x; break;
                    case HBCU_ROTATE_CLOCK_FLIP:  sx = pw - 1 - y; sy = ph - 1 - x; break;
                    case HBCU_ROTATE_CCLOCK:      sx = pw - 1 - y; sy = x;          break;
                    default:                      sx = y;          sy = x;          break;
                }
                memcpy(dst + (size_t)y * ds + (size_t)x * e, src + (size_t)sy * ss + (size_t)sx * e, e);
            }
    }
    return 0;
}

int oracle_hbcu_rotate_wait(hbcu_rotate_t *h, int64_t ticket) { (void)h; (void)ticket; return 0; }
int oracle_hbcu_rotate_poll(hbcu_rotate_t *h, int64_t ticket) { (void)h; (void)ticket; return 1; }
int oracle_hbcu_rotate_sync(hbcu_rotate_t *h) { (void)h; return 0; }
int oracle_hbcu_rotate_mark(hbcu_rotate_t *h, int which) { (void)h; (void)which; return 0; }
int oracle_hbcu_rotate_elapsed_ms(hbcu_rotate_t *h, float *ms) { (void)h; *ms = 0; return 0; }
