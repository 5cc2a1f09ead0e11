/* hb_harness.c -- drives hb_filter_object_t instances the way libhb does.
 *
 * Restates the filter part of do_job()/filter_loop() (libhb/work.c:1840-1870,
 * 2527-2600): init each filter with a running hb_filter_init_t, then for every
 * input buffer call work(), close *buf_in if the filter left it set, forward
 * the ->next-linked output list to the next filter, stop a filter after it
 * returned HB_FILTER_DONE, finally close().  Works for any object exposing the
 * libhb filter interface, so the same harness runs the reference objects
 * (oracle/_ref/libhbref.so) and the CUDA objects (libhbcu_filters.so).
 *
 * Frames cross this API as tightly packed planar arrays (plane after plane,
 * row pitch = width*bps) so that Python/numpy callers need no struct mirror.
 */
#include "handbrake/handbrake.h"
#include "hb_harness.h"

typedef struct
{
    int                  n;
    hb_filter_object_t **f;
    int                 *done;
    hb_harness_io_t     *io;
    int                  failed;
    size_t               frame_bytes_out;
    int                  out_pix_fmt, out_w, out_h;
} chain_t;

size_t hb_harness_frame_bytes(int pix_fmt, int w, int h)
{
    const AVPixFmtDescriptor *d = av_pix_fmt_desc_get(pix_fmt);
    if (d == NULL) return 0;
    size_t total = 0;
    const int nplanes = av_pix_fmt_count_planes(pix_fmt);
    for (int p = 0; p < nplanes; p++)
        total += (size_t)av_image_get_linesize(pix_fmt, w, p) * hb_image_height(pix_fmt, h, p);
    return total;
}

hb_buffer_t *hb_harness_frame_from_packed(int pix_fmt, int w, int h, const uint8_t *src)
{
    hb_buffer_t *b = hb_frame_buffer_init(pix_fmt, w, h);
    if (b == NULL) return NULL;
    for (int p = 0; p <= b->f.max_plane; p++)
    {
        const int line = av_image_get_linesize(pix_fmt, w, p);
        for (int y = 0; y < b->plane[p].height; y++)
        {
            memcpy(b->plane[p].data + (size_t)y * b->plane[p].stride, src, line);
            src += line;
        }
    }
    return b;
}

void hb_harness_frame_to_packed(const hb_buffer_t *b, uint8_t *dst)
{
    for (int p = 0; p <= b->f.max_plane; p++)
    {
        const int line = av_image_get_linesize(b->f.fmt, b->f.width, p);
        for (int y = 0; y < b->plane[p].height; y++)
        {
            memcpy(dst, b->plane[p].data + (size_t)y * b->plane[p].stride, line);
            dst += line;
        }
    }
}

static void sink(chain_t *c, hb_buffer_t *list)
{
    hb_harness_io_t *io = c->io;
    while (list != NULL)
    {
        hb_buffer_t *b = list;
        list = b->next;
        b->next = NULL;
        if (b->s.flags & HB_BUF_FLAG_EOF)
        {
            io->saw_eof = 1;
        }
        else if (b->storage_type == HBCU_DEVICE)
        {
            /* a device frame reached the end of the chain: the chain lacks its download adapter */
            hb_error("harness: HBCU_DEVICE buffer at the sink (no hb_filter_hbcu_download at the end of the chain)");
            c->failed = 1;
            io->n_dropped++;
        }
        else if (io->n_out < io->out_capacity)
        {
            const int i = io->n_out;
            if (io->out != NULL)
                hb_harness_frame_to_packed(b, io->out + (size_t)i * c->frame_bytes_out);
            if (io->out_combed) io->out_combed[i] = b->s.combed;
            if (io->out_flags)  io->out_flags[i]  = b->s.flags;
            if (io->out_start)  io->out_start[i]  = b->s.start;
            if (io->out_stop)   io->out_stop[i]   = b->s.stop;
            if (io->out_duration) io->out_duration[i] = b->s.duration;
            if (io->out_new_chap) io->out_new_chap[i] = b->s.new_chap;
            io->n_out++;
        }
        else
        {
            io->n_dropped++;
        }
        hb_buffer_close(&b);
    }
}

/* feed one buffer (or list) into filter k; mirrors one filter_loop iteration per buffer */
static void feed(chain_t *c, int k, hb_buffer_t *list)
{
    if (k >= c->n)
    {
        sink(c, list);
        return;
    }
    while (list != NULL)
    {
        hb_buffer_t *in = list;
        list = in->next;
        in->next = NULL;

        if (c->done[k])
        {
            hb_buffer_close(&in);   /* loop has exited; nothing consumes further input */
            continue;
        }
        hb_buffer_t *out = NULL;
        int status = c->f[k]->work(c->f[k], &in, &out);
        c->f[k]->status = status;
        if (in != NULL)
            hb_buffer_close(&in);                       /* work.c:2566 */
        if (status == HB_FILTER_FAILED)
            c->failed = 1;
        if (out != NULL)
            feed(c, k + 1, out);                        /* work.c:2574-2585 */
        if (status == HB_FILTER_DONE)
            c->done[k] = 1;                             /* work.c:2532 */
    }
}

int hb_harness_run_chain(int n_filters, hb_filter_object_t *const *protos,
                         const char *const *settings, hb_harness_io_t *io)
{
    chain_t c;
    memset(&c, 0, sizeof(c));
    c.io = io;
    c.f = calloc(n_filters, sizeof(*c.f));
    c.done = calloc(n_filters, sizeof(int));
    io->n_out = 0;
    io->n_dropped = 0;
    io->saw_eof = 0;

    hb_filter_init_t init;
    memset(&init, 0, sizeof(init));
    init.pix_fmt         = io->pix_fmt;
    init.geometry.width  = io->width;
    init.geometry.height = io->height;
    init.geometry.par.num = io->par_num > 0 ? io->par_num : 1;
    init.geometry.par.den = io->par_num > 0 ? io->par_den : 1;
    init.vrate.num = io->vrate_num > 0 ? io->vrate_num : 30000;
    init.vrate.den = io->vrate_den > 0 ? io->vrate_den : 1001;
    init.cfr       = io->cfr;
    init.time_base.num = 1;
    init.time_base.den = 90000;
    init.color_prim = init.color_transfer = init.color_matrix = 1;
    init.color_range = 1;
    init.chroma_location = 1;

    int volatile done_flag = 0;
    int rc = 0;
    /* work.c:1857-1870: a filter whose init fails is dropped, the job goes on */
    for (int k = 0; k < n_filters; k++)
    {
        hb_filter_object_t *f = malloc(sizeof(*f));
        memcpy(f, protos[k], sizeof(*f));
        f->settings = settings && settings[k] ? hb_parse_filter_settings(settings[k]) : NULL;
        f->done = &done_flag;
        if (f->sub_filter != NULL)
        {
            /* wrapper filters (mt_frame): the wrapped filter gets its own copy of the settings (hb.c:1697-1700) */
            hb_filter_object_t *sub = malloc(sizeof(*sub));
            memcpy(sub, f->sub_filter, sizeof(*sub));
            sub->settings = settings && settings[k] ? hb_parse_filter_settings(settings[k]) : NULL;
            f->sub_filter = sub;
        }
        if (f->init(f, &init) != 0)
        {
            io->init_failed |= 1 << k;
            if (f->settings) hb_dict_free(&f->settings);
            if (f->sub_filter) { if (f->sub_filter->settings) hb_dict_free(&f->sub_filter->settings); free(f->sub_filter); }
            free(f);
            continue;
        }
        c.f[c.n++] = f;
    }
    io->vrate_num_out = init.vrate.num;
    io->vrate_den_out = init.vrate.den;
    io->cfr_out       = init.cfr;
    io->par_num_out   = init.geometry.par.num;
    io->par_den_out   = init.geometry.par.den;
    io->width_out     = init.geometry.width;
    io->height_out    = init.geometry.height;
    io->info_text[0]  = '\0';
    for (int k = 0; k < c.n && io->collect_info; k++)
    {
        hb_filter_info_t *info = c.f[k]->info ? c.f[k]->info(c.f[k]) : NULL;
        if (info == NULL) continue;
        if (info->human_readable_desc != NULL)
            snprintf(io->info_text, sizeof(io->info_text), "%s", info->human_readable_desc);
        free(info->human_readable_desc);
        free(info);
    }
    c.out_pix_fmt = init.pix_fmt;
    c.out_w = init.geometry.width;
    c.out_h = init.geometry.height;
    c.frame_bytes_out = hb_harness_frame_bytes(c.out_pix_fmt, c.out_w, c.out_h);

    const size_t frame_bytes_in = hb_harness_frame_bytes(io->pix_fmt, io->width, io->height);
    for (int i = 0; i < io->n_in && !c.failed; i++)
    {
        hb_buffer_t *b = hb_harness_frame_from_packed(io->pix_fmt, io->width, io->height,
                                                      io->in + (size_t)i * frame_bytes_in);
        b->s.start    = io->in_start ? io->in_start[i] : (int64_t)i * 3003;
        b->s.stop     = io->in_stop ? io->in_stop[i] : b->s.start + 3003;
        b->s.duration = b->s.stop - b->s.start;
        b->s.flags    = io->in_flags  ? io->in_flags[i]  : PIC_FLAG_PROGRESSIVE_FRAME;
        b->s.combed   = io->in_combed ? io->in_combed[i] : HB_COMB_NONE;
        b->s.new_chap = io->in_new_chap ? io->in_new_chap[i] : i;   /* lets tests check that props travel with the right frame */
        b->f.color_prim = init.color_prim;
        feed(&c, 0, b);
    }
    if (!c.failed)
        feed(&c, 0, hb_buffer_eof_init());
    else
        rc = -1;

    for (int k = 0; k < c.n; k++)
    {
        c.f[k]->close(c.f[k]);
        if (c.f[k]->settings) hb_dict_free(&c.f[k]->settings);
        if (c.f[k]->sub_filter) { if (c.f[k]->sub_filter->settings) hb_dict_free(&c.f[k]->sub_filter->settings); free(c.f[k]->sub_filter); }
        free(c.f[k]);
    }
    free(c.f);
    free(c.done);
    return rc;
}

int hb_harness_run(hb_filter_object_t *proto, const char *settings, hb_harness_io_t *io)
{
    hb_filter_object_t *protos[1] = { proto };
    const char *sets[1] = { settings };
    return hb_harness_run_chain(1, protos, sets, io);
}

/* ------------------------------------------------------------------ */
/* motion metric objects                                                */
/* ------------------------------------------------------------------ */
static hb_buffer_t *luma_frame(int pix_fmt, int w, int h, int pad, const uint8_t *src)
{
    const int line = av_image_get_linesize(pix_fmt, w, 0), stride = line + pad;
    hb_buffer_t *b = hb_buffer_init(stride * h);
    if (b == NULL) return NULL;
    b->s.type = FRAME_BUF;
    b->f.fmt = pix_fmt;
    b->f.width = w;
    b->f.height = h;
    b->plane[0].data = b->data;
    b->plane[0].stride = stride;
    b->plane[0].width = w;
    b->plane[0].height = h;
    b->plane[0].size = stride * h;
    for (int y = 0; y < h; y++)
        memcpy(b->data + (size_t)y * stride, src + (size_t)y * line, line);
    return b;
}

float hb_harness_motion_metric(hb_motion_metric_object_t *proto, int pix_fmt, int w, int h, int pad,
                               const uint8_t *a, const uint8_t *b)
{
    hb_motion_metric_object_t m = *proto;
    m.private_data = NULL;
    hb_filter_init_t init;
    memset(&init, 0, sizeof(init));
    init.pix_fmt = pix_fmt;
    init.geometry.width = w;
    init.geometry.height = h;
    if (m.init(&m, &init) != 0)
        return NAN;
    hb_buffer_t *fa = luma_frame(pix_fmt, w, h, pad, a), *fb = luma_frame(pix_fmt, w, h, pad, b);
    const float v = (fa && fb) ? m.work(&m, fa, fb) : NAN;
    hb_buffer_close(&fa);
    hb_buffer_close(&fb);
    m.close(&m);
    return v;
}

/* ------------------------------------------------------------------ */
/* render_sub stand-in                                                  */
/* ------------------------------------------------------------------ */
#define GUARD_BYTE 0x5a

static hb_harness_blend_t *g_blend_cfg = NULL;

void hb_harness_set_blend(hb_harness_blend_t *cfg) { g_blend_cfg = cfg; }

struct hb_filter_private_s
{
    hb_harness_blend_t *cfg;
    hb_blend_object_t   blend;        /* this instance's copy of the object (its private_data is per instance) */
    int                 frame, next_overlay;
};

static int  render_sub_harness_init(hb_filter_object_t *filter, hb_filter_init_t *init);
static int  render_sub_harness_work(hb_filter_object_t *filter, hb_buffer_t **buf_in, hb_buffer_t **buf_out);
static void render_sub_harness_close(hb_filter_object_t *filter);

hb_filter_object_t hb_filter_render_sub_harness =
{
    .id            = HB_FILTER_RENDER_SUB,
    .enforce_order = 1,
    .name          = "Subtitle burn-in (test stand-in for render_sub)",
    .short_name    = "render_sub_harness",
    .init          = render_sub_harness_init,
    .work          = render_sub_harness_work,
    .close         = render_sub_harness_close,
};

static int render_sub_harness_init(hb_filter_object_t *filter, hb_filter_init_t *init)
{
    hb_harness_blend_t *cfg = g_blend_cfg;
    if (cfg == NULL || cfg->blend == NULL)
    {
        hb_error("render_sub_harness: no blend schedule set");
        return -1;
    }
    hb_filter_private_t *pv = calloc(1, sizeof(*pv));
    if (pv == NULL) return -1;
    pv->cfg = cfg;
    pv->blend = *cfg->blend;
    pv->blend.private_data = NULL;
    cfg->guard_damaged = cfg->same_buffer = cfg->frames = 0;
    /* rendersub.c:1129-1160 (hb_blend_init): the frame's geometry, format and chroma location, the overlay format */
    if (pv->blend.init(&pv->blend, init->geometry.width, init->geometry.height, init->pix_fmt, cfg->chroma_location,
                       init->color_range, cfg->overlay_pix_fmt) != 0)
    {
        if (pv->blend.close) pv->blend.close(&pv->blend);
        free(pv);
        return -1;
    }
    filter->private_data = pv;
    return 0;
}

static void render_sub_harness_close(hb_filter_object_t *filter)
{
    hb_filter_private_t *pv = filter->private_data;
    if (pv == NULL) return;
    pv->blend.close(&pv->blend);
    free(pv);
    filter->private_data = NULL;
}

/* bytes of one row of plane p (FFmpeg's linesize: interleaved Cb/Cr pairs count twice), and per sample position */
static int row_bytes(const hb_buffer_t *b, int p) { return av_image_get_linesize(b->f.fmt, b->f.width, p); }
static int sample_bytes(const hb_buffer_t *b, int p) { return row_bytes(b, p) / b->plane[p].width; }

/* a host frame with guard_x spare samples and guard_y spare rows around every plane, filled with GUARD_BYTE: writes
 * outside the picture land in memory the frame owns and can be found afterwards */
static hb_buffer_t *guarded_copy(const hb_buffer_t *in, int gx, int gy)
{
    int stride[4], size = 0;
    for (int p = 0; p <= in->f.max_plane; p++)
    {
        stride[p] = HB_ALIGN((in->plane[p].width + 2 * gx) * sample_bytes(in, p), 64);
        size += stride[p] * (in->plane[p].height + 2 * gy);
    }
    hb_buffer_t *b = hb_buffer_init(size);
    if (b == NULL) return NULL;
    memset(b->data, GUARD_BYTE, size);
    b->f = in->f;
    hb_buffer_copy_props(b, in);
    uint8_t *base = b->data;
    for (int p = 0; p <= in->f.max_plane; p++)
    {
        const int sb = sample_bytes(in, p);
        b->plane[p] = in->plane[p];
        b->plane[p].stride = stride[p];
        b->plane[p].data = base + (size_t)gy * stride[p] + (size_t)gx * sb;
        b->plane[p].size = stride[p] * in->plane[p].height;
        for (int y = 0; y < in->plane[p].height; y++)
            memcpy(b->plane[p].data + (size_t)y * stride[p], in->plane[p].data + (size_t)y * in->plane[p].stride,
                   (size_t)row_bytes(in, p));
        base += (size_t)stride[p] * (in->plane[p].height + 2 * gy);
    }
    return b;
}

/* every byte of the guarded allocation outside the pictures still GUARD_BYTE? */
static int guard_intact(const hb_buffer_t *b, int gx, int gy)
{
    for (int p = 0; p <= b->f.max_plane; p++)
    {
        const int sb = sample_bytes(b, p);
        const int stride = b->plane[p].stride, w = row_bytes(b, p), h = b->plane[p].height;
        const uint8_t *row0 = b->plane[p].data - (size_t)gy * stride - (size_t)gx * sb;
        for (int y = 0; y < h + 2 * gy; y++)
        {
            const uint8_t *r = row0 + (size_t)y * stride;
            const int inside = y >= gy && y < gy + h;
            for (int x = 0; x < stride; x++)
                if ((!inside || x < gx * sb || x >= gx * sb + w) && r[x] != GUARD_BYTE) return 0;
        }
    }
    return 1;
}

static hb_buffer_t *unguarded_copy(const hb_buffer_t *g)
{
    hb_buffer_t *b = hb_frame_buffer_init(g->f.fmt, g->f.width, g->f.height);
    if (b == NULL) return NULL;
    const hb_buffer_t tmp = *b;
    b->f = g->f;
    b->f.max_plane = tmp.f.max_plane;
    hb_buffer_copy_props(b, g);
    for (int p = 0; p <= b->f.max_plane; p++)
        for (int y = 0; y < b->plane[p].height; y++)
            memcpy(b->plane[p].data + (size_t)y * b->plane[p].stride, g->plane[p].data + (size_t)y * g->plane[p].stride,
                   (size_t)row_bytes(b, p));
    return b;
}

/* this frame's overlays as rendersub hands them over: YUVA buffers at f.x / f.y, linked in list order */
static int build_overlays(hb_filter_private_t *pv, hb_buffer_list_t *list)
{
    const hb_harness_blend_t *cfg = pv->cfg;
    hb_buffer_list_clear(list);
    while (pv->next_overlay < cfg->n_overlays && cfg->overlays[pv->next_overlay].frame < pv->frame) pv->next_overlay++;
    for (; pv->next_overlay < cfg->n_overlays && cfg->overlays[pv->next_overlay].frame == pv->frame; pv->next_overlay++)
    {
        const hb_harness_overlay_t *o = &cfg->overlays[pv->next_overlay];
        hb_buffer_t *b = hb_frame_buffer_init(cfg->overlay_pix_fmt, o->width, o->height);
        if (b == NULL) return -1;
        b->f.x = o->x;
        b->f.y = o->y;
        const uint8_t *src = o->yuva;
        for (int p = 0; p < 4; p++)
            for (int y = 0; y < b->plane[p].height; y++)
            {
                memcpy(b->plane[p].data + (size_t)y * b->plane[p].stride, src, b->plane[p].width);
                src += b->plane[p].width;
            }
        hb_buffer_list_append(list, b);
    }
    return 0;
}

static int render_sub_harness_work(hb_filter_object_t *filter, hb_buffer_t **buf_in, hb_buffer_t **buf_out)
{
    hb_filter_private_t *pv = filter->private_data;
    hb_harness_blend_t *cfg = pv->cfg;
    hb_buffer_t *in = *buf_in;
    *buf_in = NULL;
    if (in->s.flags & HB_BUF_FLAG_EOF)
    {
        *buf_out = in;
        return HB_FILTER_DONE;
    }
    hb_buffer_list_t overlays;
    if (build_overlays(pv, &overlays) != 0)
    {
        hb_buffer_list_close(&overlays);
        hb_buffer_close(&in);
        return HB_FILTER_FAILED;
    }
    const int changed = pv->frame < cfg->n_changed ? cfg->changed[pv->frame] : 1;
    pv->frame++;
    cfg->frames++;

    const int guarded = (cfg->guard_x > 0 || cfg->guard_y > 0) && in->storage_type != HBCU_DEVICE;
    if (guarded)
    {
        hb_buffer_t *g = guarded_copy(in, cfg->guard_x, cfg->guard_y);
        hb_buffer_close(&in);
        if (g == NULL)
        {
            hb_buffer_list_close(&overlays);
            return HB_FILTER_FAILED;
        }
        in = g;
    }
    const hb_buffer_t *given = in;
    hb_buffer_t *out = pv->blend.work(&pv->blend, in, &overlays, changed);
    hb_buffer_list_close(&overlays);            /* rendersub drops its overlays as soon as work() returns */
    if (out == NULL)
        return HB_FILTER_FAILED;
    if (out == given) cfg->same_buffer++;
    if (guarded)
    {
        if (!guard_intact(out, cfg->guard_x, cfg->guard_y)) cfg->guard_damaged++;
        hb_buffer_t *plain = unguarded_copy(out);
        hb_buffer_close(&out);
        if (plain == NULL) return HB_FILTER_FAILED;
        out = plain;
    }
    *buf_out = out;
    return HB_FILTER_OK;
}
