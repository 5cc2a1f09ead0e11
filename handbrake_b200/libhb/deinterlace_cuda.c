/* deinterlace_cuda.c -- hb_filter_yadif_cuda and hb_filter_bwdif_cuda: drop-ins for libhb's Deinterlace filter
 * (reference libhb/deinterlace.c, which builds FFmpeg's yadif / bwdif as an avfilter graph), running the deinterlacing
 * on an H100 through include/hbcu.h (hbcu_deint_*, see handbrake_b200/csrc/deinterlace.cu).
 *
 * Same ids, names, short names and settings template as deinterlace.c; the same init() contract (:70-143):
 *   - mode defaults to 3 and parity to -1; mode & 1 clear is a pass-through: every buffer is handed on untouched, no
 *     handle is created and no kernel runs;
 *   - mode & 4 (bob) gives one picture per field and doubles init->vrate.num, otherwise one picture per frame;
 *   - mode & 2 turns on Yadif's spatial interlacing check (Bwdif always runs its own);
 *   - mode & 32 (set by work.c when comb detection runs) passes a frame whose s.combed is 0 on as a shallow duplicate.
 * init() fails with an hb_error, so that the caller keeps the avfilter alias (INTEGRATION.md 2.4), for a format that is
 * not little-endian planar 3-plane YUV of 8 to 16 bits (semi-planar, gray, YUVA, big-endian, planar RGB), for Yadif on
 * a luma plane under 3 x 3 or a chroma plane under 2 rows, and for Bwdif on any plane under 3 columns or 4 rows.
 * Frame t is filtered from frames t-1, t and t+1 (frame 0 is its own prev, the last frame its own next), so a frame
 * leaves once its successor (or EOF) has arrived.  The field order, the field-end state of Bwdif and the timestamps
 * follow FFmpeg's yadif_common.c and libhb's graph time bases; DESIGN.md 4.9 lists every rule.
 * Host and HBCU_DEVICE buffers are taken per buffer: a device input is read in place; a host input is uploaded once
 * into a device frame (hbcu_xfer_upload) that serves as prev, cur and next.  A device input gives device outputs, a host
 * input host outputs unless init->hw_pix_fmt asks for device frames.  Outputs leave in order from a bounded number in
 * flight.  One device, hbcu_env_device().
 */
#include "handbrake/handbrake.h"
#include "hbcu.h"
#include "hbcu_device_frames.h"

#define DEINT_INFLIGHT     4
#define DEINT_MAX_PENDING  (2 * DEINT_INFLIGHT + 4)
#define DEINT_XFER_DEPTH   32

#define MODE_YADIF_ENABLE     1
#define MODE_YADIF_SPATIAL    2
#define MODE_XXDIF_BOB        4
#define MODE_DECOMB_SELECTIVE 32

/* yadif_common.c's current_field */
enum { FIELD_NORMAL, FIELD_END, FIELD_BACK_END };

typedef struct
{
    hb_buffer_t *out;            /* what leaves the filter */
    hb_buffer_t *dev;            /* the device picture being downloaded into out, NULL when out is ready */
    int64_t      ticket;
} deint_pending_t;

typedef struct
{
    hb_buffer_t *orig;           /* the input as it arrived; NULL once handed on (a host pass-through) */
    hb_buffer_t *dev;            /* its device frame, carrying its props: orig itself for a device input */
    int64_t      up;             /* upload ticket of a host input, -1 for a device input */
} deint_ref_t;

struct hb_filter_private_s
{
    hbcu_deint_t    *gpu;        /* NULL: pass-through */
    int              bwdif, parity, spatial, field, selective;
    int              device, device_out;
    hbcu_xfer_t     *up, *down;
    deint_ref_t      prev, cur;  /* prev.dev == cur.dev while frame 0 is cur */
    int              have_cur, state;
    deint_pending_t  pending[DEINT_MAX_PENDING];
    int              head, count;
    int64_t          next_up, next_down;
    hb_filter_init_t input, output;
};

static int  deint_cuda_init(hb_filter_object_t *filter, hb_filter_init_t *init, int bwdif);
static int  yadif_cuda_init(hb_filter_object_t *filter, hb_filter_init_t *init) { return deint_cuda_init(filter, init, 0); }
static int  bwdif_cuda_init(hb_filter_object_t *filter, hb_filter_init_t *init) { return deint_cuda_init(filter, init, 1); }
static int  deint_cuda_work(hb_filter_object_t *filter, hb_buffer_t **buf_in, hb_buffer_t **buf_out);
static void deint_cuda_close(hb_filter_object_t *filter);

/* deinterlace.c's deint_template, "mode=^"HB_INT_REG"$:parity=^([01])$" with libhb's HB_INT_REG "([0-9]+)", written out */
static const char deint_cuda_template[] = "mode=^([0-9]+)$:parity=^([01])$";

hb_filter_object_t hb_filter_yadif_cuda =
{
    .id                = HB_FILTER_YADIF,
    .enforce_order     = 1,
    .skip              = 0,
    .name              = "Deinterlace",
    .short_name        = "deinterlace",
    .settings          = NULL,
    .init              = yadif_cuda_init,
    .work              = deint_cuda_work,
    .close             = deint_cuda_close,
    .settings_template = deint_cuda_template,
};

hb_filter_object_t hb_filter_bwdif_cuda =
{
    .id                = HB_FILTER_BWDIF,
    .enforce_order     = 1,
    .skip              = 0,
    .name              = "Bwdif",
    .short_name        = "bwdif",
    .settings          = NULL,
    .init              = bwdif_cuda_init,
    .work              = deint_cuda_work,
    .close             = deint_cuda_close,
    .settings_template = deint_cuda_template,
};

static int deint_cuda_init(hb_filter_object_t *filter, hb_filter_init_t *init, int bwdif)
{
    const char *who = bwdif ? "bwdif(cuda)" : "deinterlace(cuda)";
    hb_filter_private_t *pv = calloc(1, sizeof(*pv));
    if (pv == NULL)
    {
        hb_error("%s: calloc failed", who);
        return -1;
    }
    filter->private_data = pv;
    pv->input = *init;

    int mode = 3, parity = -1;
    hb_dict_extract_int(&mode, filter->settings, "mode");
    hb_dict_extract_int(&parity, filter->settings, "parity");
    if (mode & MODE_YADIF_ENABLE)
    {
        const int fmt = init->pix_fmt;
        const AVPixFmtDescriptor *d = av_pix_fmt_desc_get(fmt);
        if (d == NULL)
        {
            hb_error("%s: pixel format %d is not one the filter knows", who, fmt);
            goto fail;
        }
        const int depth = d->comp[0].depth;
        if (av_pix_fmt_count_planes(fmt) != 3 || d->nb_components != 3 || depth < 8 || depth > 16 ||
            (d->flags & (AV_PIX_FMT_FLAG_BE | AV_PIX_FMT_FLAG_RGB)))
        {
            hb_error("%s: %s is not little-endian planar 3-plane YUV of 8 to 16 bits", who, d->name);
            goto fail;
        }
        hbcu_deint_config_t cfg;
        memset(&cfg, 0, sizeof(cfg));
        for (int p = 0; p < 3; p++)
        {
            cfg.width[p]  = hb_image_width(fmt, init->geometry.width, p);
            cfg.height[p] = hb_image_height(fmt, init->geometry.height, p);
            if (bwdif ? (cfg.width[p] < 3 || cfg.height[p] < 4)
                      : (p == 0 ? (cfg.width[p] < 3 || cfg.height[p] < 3) : cfg.height[p] < 2))
            {
                hb_error("%s: plane %d is %dx%d samples (%s)", who, p, cfg.width[p], cfg.height[p],
                         bwdif ? "Bwdif needs 3 columns and 4 rows"
                               : "Yadif needs a luma plane of 3 x 3 and chroma planes of 2 rows");
                goto fail;
            }
        }
        cfg.algorithm    = bwdif ? HBCU_DEINT_BWDIF : HBCU_DEINT_YADIF;
        cfg.sample_bytes = depth > 8 ? 2 : 1;
        cfg.depth        = depth;
        cfg.device       = pv->device = hbcu_env_device();
        if (hbcu_deint_create(&pv->gpu, &cfg) != 0 || hbcu_xfer_create(&pv->up, pv->device, DEINT_XFER_DEPTH) != 0 ||
            hbcu_xfer_create(&pv->down, pv->device, DEINT_XFER_DEPTH) != 0)
        {
            hb_error("%s: %s", who, hbcu_last_error());
            hbcu_deint_destroy(pv->gpu);
            hbcu_xfer_destroy(pv->up);
            goto fail;
        }
        pv->bwdif      = bwdif;
        pv->parity     = parity;
        pv->spatial    = (mode & MODE_YADIF_SPATIAL) != 0;
        pv->field      = (mode & MODE_XXDIF_BOB) != 0;
        pv->selective  = (mode & MODE_DECOMB_SELECTIVE) != 0;
        pv->state      = FIELD_END;
        pv->device_out = hbcu_init_wants_device_output(init);
        if (pv->field)
            init->vrate.num *= 2;
    }
    pv->output = *init;
    return 0;

fail:
    free(pv);
    filter->private_data = NULL;
    return -1;
}

/* a frame leaves the window: its host original once its upload has read it */
static void drop_ref(hb_filter_private_t *pv, deint_ref_t *r)
{
    if (r->up >= 0 && r->orig != NULL)
        hbcu_xfer_wait(pv->up, r->up);
    if (r->dev != r->orig)
        hb_buffer_close(&r->dev);
    hb_buffer_close(&r->orig);
    r->dev = NULL;
    r->up = -1;
}

static void deint_cuda_close(hb_filter_object_t *filter)
{
    hb_filter_private_t *pv = filter->private_data;
    if (pv == NULL) return;
    if (pv->gpu != NULL)
    {
        hbcu_deint_sync(pv->gpu);
        for (int i = 0; i < pv->count; i++)
        {
            deint_pending_t *p = &pv->pending[(pv->head + i) % DEINT_MAX_PENDING];
            if (p->dev != NULL) hbcu_xfer_wait(pv->down, p->ticket);
            hb_buffer_close(&p->dev);
            hb_buffer_close(&p->out);
        }
        if (pv->have_cur)
        {
            if (pv->prev.dev != pv->cur.dev) drop_ref(pv, &pv->prev);
            drop_ref(pv, &pv->cur);
        }
        hbcu_deint_destroy(pv->gpu);
        hbcu_xfer_destroy(pv->up);
        hbcu_xfer_destroy(pv->down);
    }
    free(pv);
    filter->private_data = NULL;
}

/* hands on the finished outputs in order; waits only when more than DEINT_INFLIGHT are pending, or for all of them */
static int harvest(hb_filter_private_t *pv, hb_buffer_list_t *list, int all)
{
    while (pv->count > 0)
    {
        deint_pending_t *p = &pv->pending[pv->head];
        if (p->dev != NULL)
        {
            if (all || pv->count > DEINT_INFLIGHT)
            {
                if (hbcu_xfer_wait(pv->down, p->ticket) != 0) return -1;
            }
            else
            {
                const int done = hbcu_xfer_poll(pv->down, p->ticket);
                if (done < 0) return -1;
                if (done == 0) break;
            }
            hb_buffer_close(&p->dev);
        }
        hb_buffer_list_append(list, p->out);
        p->out = NULL;
        pv->head = (pv->head + 1) % DEINT_MAX_PENDING;
        pv->count--;
    }
    return 0;
}

static void push(hb_filter_private_t *pv, hb_buffer_t *out, hb_buffer_t *dev, int64_t ticket)
{
    deint_pending_t *p = &pv->pending[(pv->head + pv->count) % DEINT_MAX_PENDING];
    p->out = out;
    p->dev = dev;
    p->ticket = ticket;
    pv->count++;
}

/* av_rescale_q(pts, 1/180000, 1/90000): halve, rounding half away from zero */
static int64_t halve(int64_t v)
{
    return v >= 0 ? (v + 1) / 2 : -((-v + 1) / 2);
}

static void set_times(hb_buffer_t *b, int64_t start, int64_t stop)
{
    b->s.start = start;
    b->s.stop = stop;
    b->s.duration = (double)(stop - start);
}

/* the pictures of pv->cur between pv->prev and `next`: s_next is the start of the next frame (extrapolated at EOF),
 * stop the stop of the last picture */
static int render(hb_filter_private_t *pv, hb_buffer_t *next, int64_t s_next, int64_t stop)
{
    hb_buffer_t *cur = pv->cur.dev;
    const int64_t s_cur = cur->s.start;
    if (pv->selective && cur->s.combed == HB_COMB_NONE)
    {
        hb_buffer_t *out;
        if (pv->cur.up < 0)
        {
            out = hb_buffer_shallow_dup(pv->cur.orig);
        }
        else
        {
            /* the host original itself, once its upload has read it; the device copy stays as the next frame's prev */
            if (hbcu_xfer_wait(pv->up, pv->cur.up) != 0) return -1;
            out = pv->cur.orig;
            pv->cur.orig = NULL;
        }
        if (out == NULL) return -1;
        out->s.flags |= PIC_FLAG_PROGRESSIVE_FRAME;
        set_times(out, s_cur, stop);
        push(pv, out, NULL, -1);
        return 0;
    }

    int tff;
    if (pv->parity == 0)      tff = 1;
    else if (pv->parity == 1) tff = 0;
    else                      tff = cur->s.combed ? !!(cur->s.flags & PIC_FLAG_TOP_FIELD_FIRST) : 1;
    const int npics = pv->field ? 2 : 1;
    const int fmt = pv->output.pix_fmt, w = pv->output.geometry.width, h = pv->output.geometry.height;
    hb_buffer_t *dev[2] = {NULL, NULL};
    hbcu_frame_t *outf[2] = {NULL, NULL};
    int parity[2] = {0, 0}, intra[2] = {0, 0};
    for (int k = 0; k < npics; k++)
    {
        dev[k] = hbcu_device_frame_buffer_init(fmt, w, h, pv->device);
        if (dev[k] == NULL)
        {
            hb_error("deinterlace(cuda): out of device memory");
            hb_buffer_close(&dev[0]);
            return -1;
        }
        outf[k] = hbcu_buffer_frame(dev[k]);
        parity[k] = (1 - tff) ^ k;
        if (k == 1 && pv->state == FIELD_BACK_END)
            pv->state = FIELD_END;
        intra[k] = pv->bwdif && pv->state == FIELD_END;
        if (pv->state == FIELD_END)
            pv->state = FIELD_NORMAL;
    }
    if (hbcu_deint_frame(pv->gpu, hbcu_buffer_frame(pv->prev.dev), hbcu_buffer_frame(cur), hbcu_buffer_frame(next), tff,
                         pv->spatial, npics, outf, parity, intra) != 0)
    {
        hb_error("deinterlace(cuda): %s", hbcu_last_error());
        hb_buffer_close(&dev[0]);
        hb_buffer_close(&dev[1]);
        return -1;
    }
    const int64_t mid = halve(s_cur + s_next);
    const int host_out = pv->cur.up >= 0 && !pv->device_out;
    for (int k = 0; k < npics; k++)
    {
        hb_buffer_t *d = dev[k];
        d->f.color_prim      = cur->f.color_prim;
        d->f.color_transfer  = cur->f.color_transfer;
        d->f.color_matrix    = cur->f.color_matrix;
        d->f.color_range     = cur->f.color_range;
        d->f.chroma_location = cur->f.chroma_location;
        hb_buffer_copy_props(d, cur);
        d->s.combed = HB_COMB_NONE;
        d->s.flags |= PIC_FLAG_PROGRESSIVE_FRAME;
        if (k == 1) d->s.new_chap = 0;
        set_times(d, k == 0 ? s_cur : mid, k + 1 < npics ? mid : stop);
        if (!host_out)
        {
            push(pv, d, NULL, -1);
            continue;
        }
        hb_buffer_t *o = hb_frame_buffer_init(fmt, w, h);
        if (o == NULL)
        {
            hb_error("deinterlace(cuda): out of memory");
            hb_buffer_close(&dev[k]);
            if (k == 0) hb_buffer_close(&dev[1]);
            return -1;
        }
        o->f.color_prim      = d->f.color_prim;
        o->f.color_transfer  = d->f.color_transfer;
        o->f.color_matrix    = d->f.color_matrix;
        o->f.color_range     = d->f.color_range;
        o->f.chroma_location = d->f.chroma_location;
        hb_buffer_copy_props(o, d);
        void *planes[3];
        int strides[3];
        for (int c = 0; c < 3; c++)
        {
            planes[c] = o->plane[c].data;
            strides[c] = o->plane[c].stride;
        }
        const int64_t ticket = pv->next_down++;
        if (hbcu_xfer_download(pv->down, ticket, hbcu_buffer_frame(d), planes, strides) != 0)
        {
            hb_error("deinterlace(cuda): %s", hbcu_last_error());
            hb_buffer_close(&o);
            hb_buffer_close(&dev[k]);
            if (k == 0) hb_buffer_close(&dev[1]);
            return -1;
        }
        push(pv, o, d, ticket);
    }
    return 0;
}

/* the input as a window entry: a device input as it is, a host input uploaded into a device frame */
static int take(hb_filter_private_t *pv, hb_buffer_t *in, deint_ref_t *r)
{
    r->orig = in;
    r->up = -1;
    if (hbcu_buffer_frame(in) != NULL)
    {
        r->dev = in;
        return 0;
    }
    r->dev = hbcu_device_frame_buffer_init(in->f.fmt, in->f.width, in->f.height, pv->device);
    if (r->dev == NULL)
    {
        hb_error("deinterlace(cuda): out of device memory");
        return -1;
    }
    hb_buffer_copy_props(r->dev, in);
    r->dev->f.color_prim      = in->f.color_prim;
    r->dev->f.color_transfer  = in->f.color_transfer;
    r->dev->f.color_matrix    = in->f.color_matrix;
    r->dev->f.color_range     = in->f.color_range;
    r->dev->f.chroma_location = in->f.chroma_location;
    const void *planes[3];
    int strides[3];
    for (int c = 0; c < 3; c++)
    {
        planes[c] = in->plane[c].data;
        strides[c] = in->plane[c].stride;
    }
    r->up = pv->next_up++;
    if (hbcu_xfer_upload(pv->up, r->up, hbcu_buffer_frame(r->dev), planes, strides) != 0)
    {
        hb_error("deinterlace(cuda): %s", hbcu_last_error());
        hb_buffer_close(&r->dev);
        r->up = -1;
        return -1;
    }
    return 0;
}

static int deint_cuda_work(hb_filter_object_t *filter, hb_buffer_t **buf_in, hb_buffer_t **buf_out)
{
    hb_filter_private_t *pv = filter->private_data;
    hb_buffer_t *in = *buf_in;
    *buf_in = NULL;
    if (pv->gpu == NULL)
    {
        *buf_out = in;
        return (in->s.flags & HB_BUF_FLAG_EOF) ? HB_FILTER_DONE : HB_FILTER_OK;
    }
    hb_buffer_list_t list;
    hb_buffer_list_clear(&list);
    int failed = 0;
    if (in->s.flags & HB_BUF_FLAG_EOF)
    {
        if (pv->have_cur)
        {
            /* the last frame is its own next; its successor's start is extrapolated (yadif_common.c) */
            pv->state = FIELD_BACK_END;
            hb_buffer_t *cur = pv->cur.dev;
            failed = render(pv, cur, 2 * cur->s.start - pv->prev.dev->s.start, cur->s.stop) != 0;
            if (pv->prev.dev != pv->cur.dev) drop_ref(pv, &pv->prev);
            drop_ref(pv, &pv->cur);
            pv->have_cur = 0;
        }
        failed |= harvest(pv, &list, 1) != 0;
        if (failed) hb_error("deinterlace(cuda): %s", hbcu_last_error());
        hb_buffer_list_append(&list, in);
        *buf_out = hb_buffer_list_clear(&list);
        return failed ? HB_FILTER_FAILED : HB_FILTER_DONE;
    }

    deint_ref_t next;
    if (take(pv, in, &next) != 0)
    {
        hb_buffer_close(&in);
        return HB_FILTER_FAILED;
    }
    if (!pv->have_cur)
    {
        pv->cur = next;
        pv->prev = next;
        pv->have_cur = 1;
        *buf_out = NULL;
        return HB_FILTER_OK;
    }
    failed = render(pv, next.dev, next.dev->s.start, next.dev->s.start) != 0;
    if (pv->prev.dev != pv->cur.dev) drop_ref(pv, &pv->prev);
    pv->prev = pv->cur;
    pv->cur = next;
    if (failed || harvest(pv, &list, 0) != 0)
    {
        hb_error("deinterlace(cuda): %s", hbcu_last_error());
        hb_buffer_list_close(&list);
        return HB_FILTER_FAILED;
    }
    *buf_out = hb_buffer_list_clear(&list);
    return HB_FILTER_OK;
}
