/* blend_semiplanar_port.c -- TEST INFRASTRUCTURE: the hbcu_blend_* stand-ins of port/blend_port.c for
 * libhostlogic_semiplanar.so (semiplanar.mk), extended to semi-planar 4:2:0 frames (hbcu_blend_config_t
 * .interleaved_chroma: NV12, P010, P016).
 *
 * port/blend_port.c is compiled here as it is, with its create and frames entry points renamed: the overlay staging,
 * the unchanged-list rule and the planar restatement are its own.  On top of it this file restates, written out on
 * their own and not derived from the planar paths, blend.c's four semi-planar functions (blend8onbi8, blend8onbi1x,
 * blend_subsample_8onbi8, blend_subsample_8onbi1x), per sample the way the CUDA kernel works.  hb_blend_cuda over
 * this restatement must give the reference's recorded outputs (tests/test_blend_semiplanar_gpu.py).  Never linked into
 * the product.
 */
#define oracle_hbcu_blend_create planar_blend_create
#define oracle_hbcu_blend_frames planar_blend_frames
#include "../port/blend_port.c"
#undef oracle_hbcu_blend_create
#undef oracle_hbcu_blend_frames

/* one overlay onto a semi-planar 4:2:0 frame (plane 0 Y, plane 1 Cb/Cr pairs), in place: blend.c's *bi* functions.
 * They differ from the planar ones in more than the chroma address:
 *   - above 8 bits an overlay sample v enters as av_bswap16(v), i.e. v << 8, at every depth (blend.c:193, 214-217, 747,
 *     778-783), while alpha is << (depth - 8) and max = (256 << (depth - 8)) - 1 as in the planar paths;
 *   - blend_subsample_8onbi8's group loops run over the whole 2x2 group (blend.c:388-390): samples of the group past the
 *     overlay's right / bottom edge are weighted in with the frame's unblended chroma. */
static void blend_one_bi(const blend_geom_t *g, uint8_t *const planes[3], const int strides[3], const hbcu_blend_overlay_t *o)
{
    const int W = g->width, H = g->height, CW = -((-W) >> 1), CH = -((-H) >> 1);
    const int bps = g->depth > 8 ? 2 : 1, shift = g->depth - 8, vshift = g->depth > 8 ? 8 : 0;
    const unsigned maxv = (256u << shift) - 1, half = maxv >> 1;
    const uint8_t *oY = o->planes[0], *oU = o->planes[1], *oV = o->planes[2], *oA = o->planes[3];
    const int sY = o->strides[0], sU = o->strides[1], sV = o->strides[2], sA = o->strides[3];
    uint8_t *Y = planes[0], *C = planes[1];
    const int yst = strides[0], cst = strides[1];

    if (g->subsample)
    {
        /* blend.c:167-168 / 356-357: the clip is min(overlay, frame) in size */
        const int width  = o->width < W ? o->width : W;
        const int height = o->height < H ? o->height : H;
        const int whole_group = bps == 1;                 /* blend_subsample_8onbi8 */
        for (int oy = 0; oy < height; oy++)
            for (int ox = 0; ox < width; ox++)
            {
                const int x = o->x + ox, y = o->y + oy;
                if (x < 0 || x >= W || y < 0 || y >= H) continue;
                const unsigned alpha = (unsigned)oA[oy * sA + ox] << shift;
                const unsigned v = get(Y, yst, bps, x, y);
                put(Y, yst, bps, x, y, (v * (maxv - alpha) + ((unsigned)oY[oy * sY + ox] << vshift) * alpha + half) / maxv);
            }
        int x0c = o->x & ~1, y0c = o->y & ~1;
        if (x0c < 0) x0c = 0;
        if (y0c < 0) y0c = 0;
        for (int cy = y0c >> 1; cy < CH; cy++)
            for (int cx = x0c >> 1; cx < CW; cx++)
            {
                const int ox = 2 * cx - o->x, oy = 2 * cy - o->y;
                if (ox >= width || oy >= height) continue;
                const unsigned u0 = get(C, cst, bps, 2 * cx, cy), v0 = get(C, cst, bps, 2 * cx + 1, cy);
                unsigned accu_a = 0, accu_b = 0, accu_c = 0;
                for (int yz = 0; yz < 2 && (whole_group || oy + yz < height); yz++)
                    for (int xz = 0; xz < 2 && (whole_group || ox + xz < width); xz++)
                    {
                        const int i = ox + xz, j = oy + yz;
                        const unsigned coeff = g->c[0][xz] * g->c[1][yz];
                        unsigned ru = u0, rv = v0;
                        if (i >= 0 && j >= 0 && i < width && j < height)
                        {
                            const unsigned alpha = (unsigned)oA[j * sA + i] << shift;
                            ru = (ru * (maxv - alpha) + ((unsigned)oU[j * sU + i] << vshift) * alpha + half) / maxv;
                            rv = (rv * (maxv - alpha) + ((unsigned)oV[j * sV + i] << vshift) * alpha + half) / maxv;
                        }
                        accu_a += coeff * ru;
                        accu_b += coeff * rv;
                        accu_c += coeff;
                    }
                put(C, cst, bps, 2 * cx, cy, (accu_a + (accu_c >> 1)) / accu_c);
                put(C, cst, bps, 2 * cx + 1, cy, (accu_b + (accu_c >> 1)) / accu_c);
            }
        return;
    }

    /* plain path, blend.c:615-637 / 709-731 */
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
            const unsigned v = get(Y, yst, bps, x, y);
            put(Y, yst, bps, x, y, (v * (maxv - alpha) + ((unsigned)oY[yy * sY + xx] << vshift) * alpha) / maxv);
        }
    /* blend.c:668-690 / 763-785: Cb of chroma column (left >> 1) + xx at 2 * that, Cr one sample after it; an odd hh
     * drops the overlay's last chroma row */
    for (int yy = y0 >> 1; yy < hh >> 1; yy++)
        for (int xx = x0 >> 1; xx < ww >> 1; xx++)
        {
            const int cx = (left >> 1) + xx, cy = (top >> 1) + yy;
            if (cx < 0 || cx >= CW || cy < 0 || cy >= CH) continue;
            const unsigned alpha = (unsigned)oA[(yy << 1) * sA + (xx << 1)] << shift;
            const unsigned u = get(C, cst, bps, 2 * cx, cy), v = get(C, cst, bps, 2 * cx + 1, cy);
            put(C, cst, bps, 2 * cx, cy, (u * (maxv - alpha) + ((unsigned)oU[yy * sU + xx] << vshift) * alpha) / maxv);
            put(C, cst, bps, 2 * cx + 1, cy, (v * (maxv - alpha) + ((unsigned)oV[yy * sV + xx] << vshift) * alpha) / maxv);
        }
}

int oracle_hbcu_blend_create(hbcu_blend_t **out, const hbcu_blend_config_t *cfg)
{
    /* the semi-planar formats in use are 4:2:0 only */
    if (!(cfg->interleaved_chroma == 0 || (cfg->interleaved_chroma == 1 && cfg->chroma_shift_w == 1 && cfg->chroma_shift_h == 1)))
    {
        oracle_hostlogic_set_error("blend_create: interleaved chroma needs a 4:2:0 frame");
        return -1;
    }
    return planar_blend_create(out, cfg);
}

int oracle_hbcu_blend_frames(hbcu_blend_t *h, hbcu_frame_t *in_frame, const void *const in_planes[3], const int in_strides[3],
                             hbcu_frame_t *out_frame, void *const out_planes[3], const int out_strides[3])
{
    if (!h->cfg.interleaved_chroma)
        return planar_blend_frames(h, in_frame, in_planes, in_strides, out_frame, out_planes, out_strides);
    if (!h->have || (in_frame == NULL) != (out_frame == NULL))
    {
        oracle_hostlogic_set_error("blend_frames: bad argument");
        return -1;
    }
    /* planes 0 and 1 only; a row of plane 1 is chroma width Cb/Cr pairs */
    uint8_t *dst[3] = {NULL, NULL, NULL};
    int ds[3] = {0, 0, 0};
    const int bps = h->cfg.depth > 8 ? 2 : 1;
    for (int p = 0; p < 2; p++)
    {
        const uint8_t *src = in_frame ? oracle_hostlogic_frame_planes(in_frame)[p] : in_planes[p];
        const int ss = in_frame ? oracle_hostlogic_frame_strides(in_frame)[p] : in_strides[p];
        dst[p] = out_frame ? (uint8_t *)oracle_hostlogic_frame_planes(out_frame)[p] : out_planes[p];
        ds[p] = out_frame ? oracle_hostlogic_frame_strides(out_frame)[p] : out_strides[p];
        const int row_bytes = (p ? 2 * -((-h->cfg.width) >> 1) : h->cfg.width) * bps;
        const int rows = p ? -((-h->cfg.height) >> 1) : h->cfg.height;
        if (src != dst[p])
            for (int y = 0; y < rows; y++)
                memcpy(dst[p] + (size_t)y * ds[p], src + (size_t)y * ss, (size_t)row_bytes);
    }
    for (int i = 0; i < h->count; i++)
        blend_one_bi(&h->g, dst, ds, &h->list[i]);
    return 0;
}
