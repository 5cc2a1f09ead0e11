/* blend_port.c -- TEST INFRASTRUCTURE: plain-C restatement of libhb/blend.c (the planar paths: blend8on8, blend8on1x,
 * blend_subsample_8on8, blend_subsample_8on1x) and, on top of it, CPU stand-ins for the hbcu_blend_* calls of the
 * product's host object (handbrake_b200/libhb/blend_cuda.c; see hostlogic_nlmeans.c for the idea).
 *
 * The restatement is written per sample, the way the CUDA kernel works: for each sample inside the picture, which
 * overlays of the list does the reference's loop nest visit it with, and with which overlay samples.  Samples the
 * reference writes outside the picture are not written.  oracle_blend_frame() over the recorded inputs must give the
 * reference's recorded outputs (tests/test_blend_gpu.py); that pins the per-sample reading of the loop bounds on a
 * machine without a GPU.  Never linked into the product.
 */
#include "../../include/hbcu.h"

#include <stdlib.h>
#include <string.h>

void oracle_hostlogic_set_error(const char *fmt, ...);
const void *const *oracle_hostlogic_frame_planes(const hbcu_frame_t *f);      /* hostlogic_frames.c */
const int *oracle_hostlogic_frame_strides(const hbcu_frame_t *f);

typedef struct
{
    int width, height, depth, ws, hs, subsample;
    uint32_t c[2][4];
} blend_geom_t;

static inline unsigned get(const uint8_t *plane, int stride, int bps, int x, int y)
{
    const uint8_t *row = plane + (size_t)y * stride;
    return bps == 2 ? ((const uint16_t *)row)[x] : row[x];
}

static inline void put(uint8_t *plane, int stride, int bps, int x, int y, unsigned v)
{
    uint8_t *row = plane + (size_t)y * stride;
    if (bps == 2) ((uint16_t *)row)[x] = (uint16_t)v;
    else          row[x] = (uint8_t)v;
}

/* one overlay onto the frame, in place */
static void blend_one(const blend_geom_t *g, uint8_t *const planes[3], const int strides[3], const hbcu_blend_overlay_t *o)
{
    const int W = g->width, H = g->height, ws = g->ws, hs = g->hs, sw = 1 << ws, sh = 1 << hs;
    const int CW = -((-W) >> ws), CH = -((-H) >> hs);
    const int bps = g->depth > 8 ? 2 : 1, shift = g->depth - 8;
    const unsigned maxv = (256u << shift) - 1, half = maxv >> 1;
    const uint8_t *oY = o->planes[0], *oU = o->planes[1], *oV = o->planes[2], *oA = o->planes[3];
    const int sY = o->strides[0], sU = o->strides[1], sV = o->strides[2], sA = o->strides[3];

    if (g->subsample)
    {
        /* blend.c:73-74 */
        const int width  = o->width < W ? o->width : W;
        const int height = o->height < H ? o->height : H;
        /* luma: every overlay sample (ox, oy) in [0, width) x [0, height) at (x + ox, y + oy) */
        for (int oy = 0; oy < height; oy++)
            for (int ox = 0; ox < width; ox++)
            {
                const int x = o->x + ox, y = o->y + oy;
                if (x < 0 || x >= W || y < 0 || y >= H) continue;
                const unsigned alpha = (unsigned)oA[oy * sA + ox] << shift;
                const unsigned v = get(planes[0], strides[0], bps, x, y);
                put(planes[0], strides[0], bps, x, y, (v * (maxv - alpha) + ((unsigned)oY[oy * sY + ox] << shift) * alpha + half) / maxv);
            }
        /* chroma: the groups whose top-left sample (X, Y) the loop visits, from the aligned, clamped start */
        int x0c = o->x & ~(sw - 1), y0c = o->y & ~(sh - 1);
        if (x0c < 0) x0c = 0;
        if (y0c < 0) y0c = 0;
        for (int cy = y0c >> hs; cy < CH; cy++)
            for (int cx = x0c >> ws; cx < CW; cx++)
            {
                const int ox = (cx << ws) - o->x, oy = (cy << hs) - o->y;
                if (ox >= width || oy >= height) continue;
                const unsigned u0 = get(planes[1], strides[1], bps, cx, cy), v0 = get(planes[2], strides[2], bps, cx, cy);
                unsigned accu_a = 0, accu_b = 0, accu_c = 0;
                for (int yz = 0; yz < sh && oy + yz < height; yz++)
                    for (int xz = 0; xz < sw && ox + xz < width; xz++)
                    {
                        const unsigned coeff = g->c[0][xz] * g->c[1][yz];
                        unsigned ru = u0, rv = v0;
                        if (ox + xz >= 0 && oy + yz >= 0)
                        {
                            const int i = ox + xz, j = oy + yz;
                            const unsigned alpha = (unsigned)oA[j * sA + i] << shift;
                            ru = (ru * (maxv - alpha) + ((unsigned)oU[j * sU + i] << shift) * alpha + half) / maxv;
                            rv = (rv * (maxv - alpha) + ((unsigned)oV[j * sV + i] << shift) * alpha + half) / maxv;
                        }
                        accu_a += coeff * ru;
                        accu_b += coeff * rv;
                        accu_c += coeff;
                    }
                put(planes[1], strides[1], bps, cx, cy, (accu_a + (accu_c >> 1)) / accu_c);
                put(planes[2], strides[2], bps, cx, cy, (accu_b + (accu_c >> 1)) / accu_c);
            }
        return;
    }

    /* plain path, blend.c:434-456 */
    const int left = o->x, top = o->y;
    const int x0 = left < 0 ? -left : 0, y0 = top < 0 ? -top : 0;
    const int ww = (o->width - x0 > W - left) ? W - left + x0 : o->width;
    const int hh = (o->height - y0 > H - top) ? H - top + y0 : o->height;
    for (int yy = y0; yy < hh; yy++)
        for (int xx = x0; xx < ww; xx++)
        {
            const int x = left + xx, y = top + yy;
            if (x < 0 || x >= W || y < 0 || y >= H) continue;
            const unsigned alpha = (unsigned)oA[yy * sA + xx] << shift;
            const unsigned v = get(planes[0], strides[0], bps, x, y);
            put(planes[0], strides[0], bps, x, y, (v * (maxv - alpha) + ((unsigned)oY[yy * sY + xx] << shift) * alpha) / maxv);
        }
    /* chroma rows / columns land at (top >> hs) + yy, (left >> ws) + xx; alpha of the group's top-left luma sample */
    for (int yy = y0 >> hs; yy < hh >> hs; yy++)
        for (int xx = x0 >> ws; xx < ww >> ws; xx++)
        {
            const int cx = (left >> ws) + xx, cy = (top >> hs) + yy;
            if (cx < 0 || cx >= CW || cy < 0 || cy >= CH) continue;
            const unsigned alpha = (unsigned)oA[(yy << hs) * sA + (xx << ws)] << shift;
            for (int p = 1; p < 3; p++)
            {
                const uint8_t *src = p == 1 ? oU : oV;
                const int ss = p == 1 ? sU : sV;
                const unsigned v = get(planes[p], strides[p], bps, cx, cy);
                put(planes[p], strides[p], bps, cx, cy, (v * (maxv - alpha) + ((unsigned)src[yy * ss + xx] << shift) * alpha) / maxv);
            }
        }
}

/* ------------------------------------------------------------------------------------------ hbcu_blend_* stand-ins */
static uint64_t g_uploads = 0;

struct hbcu_blend_s
{
    hbcu_blend_config_t cfg;
    blend_geom_t g;
    /* the staged copy of the current list, as the device holds it */
    hbcu_blend_overlay_t *list;
    uint8_t *blob;
    int count, have;
};

uint64_t oracle_hbcu_blend_uploads(void) { return g_uploads; }

int oracle_hbcu_blend_create(hbcu_blend_t **out, const hbcu_blend_config_t *cfg)
{
    const int ws = cfg->chroma_shift_w, hs = cfg->chroma_shift_h;
    if (!((ws == 1 && hs == 1) || (ws == 1 && hs == 0) || (ws == 0 && hs == 0)) ||
        !((cfg->overlay_shift_w == ws && cfg->overlay_shift_h == hs) || (cfg->overlay_shift_w == 0 && cfg->overlay_shift_h == 0)) ||
        cfg->depth < 8 || cfg->depth > 16 || cfg->width < 1 || cfg->height < 1)
    {
        oracle_hostlogic_set_error("blend_create: unsupported geometry");
        return -1;
    }
    struct hbcu_blend_s *h = calloc(1, sizeof(*h));
    h->cfg = *cfg;
    h->g.width = cfg->width; h->g.height = cfg->height; h->g.depth = cfg->depth;
    h->g.ws = ws; h->g.hs = hs;
    h->g.subsample = cfg->overlay_shift_w != ws || cfg->overlay_shift_h != hs;
    memcpy(h->g.c, cfg->chroma_coeffs, sizeof(h->g.c));
    *out = h;
    return 0;
}

void oracle_hbcu_blend_destroy(hbcu_blend_t *h)
{
    if (h == NULL) return;
    free(h->list);
    free(h->blob);
    free(h);
}

int oracle_hbcu_blend_set_overlays(hbcu_blend_t *h, const hbcu_blend_overlay_t *list, int count, int changed)
{
    if (!changed && h->have && h->count == count)
    {
        int same = 1;
        for (int i = 0; i < count && same; i++)
            same = h->list[i].x == list[i].x && h->list[i].y == list[i].y &&
                   h->list[i].width == list[i].width && h->list[i].height == list[i].height;
        if (same) return 0;
    }
    size_t bytes = 0;
    for (int i = 0; i < count; i++)
        for (int p = 0; p < 4; p++)
        {
            const int sub = p == 1 || p == 2;
            bytes += (size_t)(sub ? -((-list[i].width) >> h->cfg.overlay_shift_w) : list[i].width) *
                     (sub ? -((-list[i].height) >> h->cfg.overlay_shift_h) : list[i].height);
        }
    free(h->list);
    free(h->blob);
    h->list = calloc(count > 0 ? count : 1, sizeof(*h->list));
    h->blob = malloc(bytes > 0 ? bytes : 1);
    uint8_t *dst = h->blob;
    for (int i = 0; i < count; i++)
    {
        h->list[i] = list[i];
        for (int p = 0; p < 4; p++)
        {
            const int sub = p == 1 || p == 2;
            const int pw = sub ? -((-list[i].width) >> h->cfg.overlay_shift_w) : list[i].width;
            const int ph = sub ? -((-list[i].height) >> h->cfg.overlay_shift_h) : list[i].height;
            for (int y = 0; y < ph; y++)
                memcpy(dst + (size_t)y * pw, list[i].planes[p] + (size_t)y * list[i].strides[p], pw);
            h->list[i].planes[p] = dst;
            h->list[i].strides[p] = pw;
            dst += (size_t)pw * ph;
        }
    }
    h->count = count;
    h->have = 1;
    g_uploads++;
    return 0;
}

int oracle_hbcu_blend_frames(hbcu_blend_t *h, hbcu_frame_t *in_frame, const void *const in_planes[3], const int in_strides[3],
                             hbcu_frame_t *out_frame, void *const out_planes[3], const int out_strides[3])
{
    if (!h->have || (in_frame == NULL) != (out_frame == NULL))
    {
        oracle_hostlogic_set_error("blend_frames: bad argument");
        return -1;
    }
    uint8_t *dst[3];
    int ds[3];
    const int bps = h->cfg.depth > 8 ? 2 : 1;
    for (int p = 0; p < 3; p++)
    {
        const uint8_t *src = in_frame ? oracle_hostlogic_frame_planes(in_frame)[p] : in_planes[p];
        const int ss = in_frame ? oracle_hostlogic_frame_strides(in_frame)[p] : in_strides[p];
        dst[p] = out_frame ? (uint8_t *)oracle_hostlogic_frame_planes(out_frame)[p] : out_planes[p];
        ds[p] = out_frame ? oracle_hostlogic_frame_strides(out_frame)[p] : out_strides[p];
        const int w = p ? -((-h->cfg.width) >> h->cfg.chroma_shift_w) : h->cfg.width;
        const int rows = p ? -((-h->cfg.height) >> h->cfg.chroma_shift_h) : h->cfg.height;
        if (src != dst[p])
            for (int y = 0; y < rows; y++)
                memcpy(dst[p] + (size_t)y * ds[p], src + (size_t)y * ss, (size_t)w * bps);
    }
    for (int i = 0; i < h->count; i++)
        blend_one(&h->g, dst, ds, &h->list[i]);
    return 0;
}

int oracle_hbcu_blend_wait(hbcu_blend_t *h) { (void)h; return 0; }
int oracle_hbcu_blend_sync(hbcu_blend_t *h) { (void)h; return 0; }
int oracle_hbcu_blend_mark(hbcu_blend_t *h, int which) { (void)h; (void)which; return 0; }
int oracle_hbcu_blend_elapsed_ms(hbcu_blend_t *h, float *ms) { (void)h; *ms = 0; return 0; }
