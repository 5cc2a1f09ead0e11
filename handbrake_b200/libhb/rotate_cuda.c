/* rotate_cuda.c -- hb_filter_rotate_cuda: drop-in for hb_filter_rotate (reference libhb/rotate.c), running the
 * rotation or mirror on an H100 through include/hbcu.h (hbcu_rotate_*, see handbrake_b200/csrc/rotate.cu).
 *
 * Same id, short name and settings template as hb_filter_rotate; the same init() contract (rotate.c:146-270):
 *   angle=0:hflip=1     hflip                 angle=180:hflip=0   vflip, hflip      angle=180:hflip=1  vflip
 *   angle=90:hflip=0/1  transpose=clock / clock_flip    angle=270:hflip=0/1  transpose=cclock / cclock_flip
 *   - 90 and 270 swap init->geometry's width and height and its par.num and par.den;
 *   - angle=0:hflip=0, or an angle rotate_init's switch does not know (which ignores hflip), is a pass-through: every
 *     buffer is handed on untouched, no handle is created and no kernel runs;
 *   - `disable` is not read, as rotate_init does not read it.
 * init() fails with an hb_error, so that the caller keeps hb_filter_rotate (INTEGRATION.md 2), for a 4:2:2 format at 90
 * or 270 (the reference converts through swscale there), a format of fewer than two or more than three planes, and a
 * format the pixel-format table does not describe.  4:2:2 flips are accepted.
 * Host and HBCU_DEVICE buffers are taken per buffer: a device input gives a device output, a host input a host output
 * unless init->hw_pix_fmt asks for device frames.  Outputs leave in order from a bounded number in flight and carry the
 * input's props and colour fields; only the geometry and the plane layout change.  A device input is closed as soon as
 * its kernel is queued (hbcu_rotate_frame records the kernel as the frame's reader), so a wrapped decoder surface goes
 * back to the decoder once the kernel has read it.  A host input is closed once its copy to the device is done.  One
 * device, hbcu_env_device().
 */
#include "handbrake/handbrake.h"
#include "hbcu.h"
#include "hbcu_device_frames.h"

#define ROTATE_INFLIGHT    4
#define ROTATE_MAX_PENDING (ROTATE_INFLIGHT + 2)

typedef struct
{
    hb_buffer_t *in, *out;       /* in: a host input, kept until its rotation is done; NULL for a device input */
    int64_t      ticket;
} rotate_pending_t;

struct hb_filter_private_s
{
    hbcu_rotate_t   *gpu;        /* NULL: pass-through */
    int              device, device_out;
    rotate_pending_t pending[ROTATE_MAX_PENDING];
    int              head, count;
    int64_t          next_ticket;
    hb_filter_init_t input, output;
};

static int  rotate_cuda_init(hb_filter_object_t *filter, hb_filter_init_t *init);
static int  rotate_cuda_work(hb_filter_object_t *filter, hb_buffer_t **buf_in, hb_buffer_t **buf_out);
static void rotate_cuda_close(hb_filter_object_t *filter);

/* rotate.c's template, "angle=^(0|90|180|270)$:hflip=^"HB_BOOL_REG"$:disable=^"HB_BOOL_REG"$" with libhb's HB_BOOL_REG
 * "(yes|no|true|false|[01])", written out */
static const char rotate_cuda_template[] =
    "angle=^(0|90|180|270)$:hflip=^(yes|no|true|false|[01])$:disable=^(yes|no|true|false|[01])$";

hb_filter_object_t hb_filter_rotate_cuda =
{
    .id                = HB_FILTER_ROTATE,
    .enforce_order     = 1,
    .skip              = 0,
    .name              = "Rotate (CUDA sm_90a)",
    .short_name        = "rotate",
    .settings          = NULL,
    .init              = rotate_cuda_init,
    .work              = rotate_cuda_work,
    .close             = rotate_cuda_close,
    .settings_template = rotate_cuda_template,
};

/* rotate_init's switch: the transform of angle / hflip, 0 for none */
static int transform_of(int angle, int flip)
{
    switch (angle)
    {
        case 0:   return flip ? HBCU_ROTATE_HFLIP : 0;
        case 90:  return flip ? HBCU_ROTATE_CLOCK_FLIP : HBCU_ROTATE_CLOCK;
        case 180: return flip ? HBCU_ROTATE_VFLIP : HBCU_ROTATE_180;
        case 270: return flip ? HBCU_ROTATE_CCLOCK_FLIP : HBCU_ROTATE_CCLOCK;
        default:  return 0;
    }
}

static int rotate_cuda_init(hb_filter_object_t *filter, hb_filter_init_t *init)
{
    hb_filter_private_t *pv = calloc(1, sizeof(*pv));
    if (pv == NULL)
    {
        hb_error("rotate(cuda): calloc failed");
        return -1;
    }
    filter->private_data = pv;
    pv->input = *init;

    int angle = 0, flip = 0;
    hb_dict_extract_int(&angle, filter->settings, "angle");
    hb_dict_extract_bool(&flip, filter->settings, "hflip");
    const int transform = transform_of(angle, flip);
    const int transpose = angle == 90 || angle == 270;
    if (transform != 0)
    {
        const int fmt = init->pix_fmt;
        const AVPixFmtDescriptor *d = av_pix_fmt_desc_get(fmt);
        const int planes = av_pix_fmt_count_planes(fmt);
        if (d == NULL)
        {
            hb_error("rotate(cuda): pixel format %d is not one the filter knows", fmt);
            goto fail;
        }
        if (planes < 2 || planes > 3)
        {
            hb_error("rotate(cuda): %s has %d planes (2 or 3 are taken)", d->name, planes);
            goto fail;
        }
        if (transpose && d->log2_chroma_w != d->log2_chroma_h)
        {
            hb_error("rotate(cuda): %s cannot be transposed plane by plane (the reference converts it through swscale)",
                     d->name);
            goto fail;
        }
        hbcu_rotate_config_t cfg;
        memset(&cfg, 0, sizeof(cfg));
        cfg.planes = planes;
        for (int p = 0; p < planes; p++)
        {
            cfg.width[p]      = hb_image_width(fmt, init->geometry.width, p);
            cfg.height[p]     = hb_image_height(fmt, init->geometry.height, p);
            cfg.elem_bytes[p] = av_image_get_linesize(fmt, init->geometry.width, p) / cfg.width[p];
        }
        cfg.transform = transform;
        cfg.device    = pv->device = hbcu_env_device();
        cfg.slots     = ROTATE_MAX_PENDING;
        if (hbcu_rotate_create(&pv->gpu, &cfg) != 0)
        {
            hb_error("rotate(cuda): %s", hbcu_last_error());
            goto fail;
        }
        pv->device_out = hbcu_init_wants_device_output(init);
    }
    if (transpose)
    {
        const hb_geometry_t g = init->geometry;
        init->geometry.width   = g.height;
        init->geometry.height  = g.width;
        init->geometry.par.num = g.par.den;
        init->geometry.par.den = g.par.num;
    }
    pv->output = *init;
    return 0;

fail:
    free(pv);
    filter->private_data = NULL;
    return -1;
}

static void rotate_cuda_close(hb_filter_object_t *filter)
{
    hb_filter_private_t *pv = filter->private_data;
    if (pv == NULL) return;
    hbcu_rotate_destroy(pv->gpu);          /* waits for the rotations in flight */
    for (int i = 0; i < pv->count; i++)
    {
        rotate_pending_t *p = &pv->pending[(pv->head + i) % ROTATE_MAX_PENDING];
        hb_buffer_close(&p->in);
        hb_buffer_close(&p->out);
    }
    free(pv);
    filter->private_data = NULL;
}

/* hands on the finished outputs in order: a device output at once (its readers order themselves behind the kernel), a
 * host side once its copies are done; waits only when more than ROTATE_INFLIGHT are pending, or for all of them */
static int harvest(hb_filter_private_t *pv, hb_buffer_list_t *list, int all)
{
    while (pv->count > 0)
    {
        rotate_pending_t *p = &pv->pending[pv->head];
        if (p->in == NULL && hbcu_buffer_frame(p->out) != NULL)
        {
            /* device in, device out: nothing to wait for */
        }
        else if (all || pv->count > ROTATE_INFLIGHT)
        {
            if (hbcu_rotate_wait(pv->gpu, p->ticket) != 0) goto gpu_error;
        }
        else
        {
            const int done = hbcu_rotate_poll(pv->gpu, p->ticket);
            if (done < 0) goto gpu_error;
            if (done == 0) break;
        }
        hb_buffer_list_append(list, p->out);
        p->out = NULL;
        hb_buffer_close(&p->in);
        pv->head = (pv->head + 1) % ROTATE_MAX_PENDING;
        pv->count--;
    }
    return 0;

gpu_error:
    hb_error("rotate(cuda): %s", hbcu_last_error());
    return -1;
}

static int rotate_cuda_work(hb_filter_object_t *filter, hb_buffer_t **buf_in, hb_buffer_t **buf_out)
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
    if (in->s.flags & HB_BUF_FLAG_EOF)
    {
        const int failed = harvest(pv, &list, 1) != 0;
        hb_buffer_list_append(&list, in);
        *buf_out = hb_buffer_list_clear(&list);
        return failed ? HB_FILTER_FAILED : HB_FILTER_DONE;
    }

    hbcu_frame_t *fin = hbcu_buffer_frame(in);
    const int fmt = pv->output.pix_fmt, w = pv->output.geometry.width, h = pv->output.geometry.height;
    hb_buffer_t *out = (fin != NULL || pv->device_out) ? hbcu_device_frame_buffer_init(fmt, w, h, pv->device)
                                                       : hb_frame_buffer_init(fmt, w, h);
    if (out == NULL)
    {
        hb_error("rotate(cuda): out of memory");
        hb_buffer_close(&in);
        return HB_FILTER_FAILED;
    }
    out->f.color_prim      = in->f.color_prim;
    out->f.color_transfer  = in->f.color_transfer;
    out->f.color_matrix    = in->f.color_matrix;
    out->f.color_range     = in->f.color_range;
    out->f.chroma_location = in->f.chroma_location;
    hb_buffer_copy_props(out, in);

    const void *ip[3] = {NULL, NULL, NULL};
    void *op[3] = {NULL, NULL, NULL};
    int is[3] = {0, 0, 0}, os[3] = {0, 0, 0};
    for (int c = 0; c <= in->f.max_plane && c < 3; c++)
    {
        ip[c] = in->plane[c].data;
        is[c] = in->plane[c].stride;
    }
    for (int c = 0; c <= out->f.max_plane && c < 3; c++)
    {
        op[c] = out->plane[c].data;
        os[c] = out->plane[c].stride;
    }
    const int64_t ticket = pv->next_ticket++;
    if (hbcu_rotate_frame(pv->gpu, ticket, fin, ip, is, hbcu_buffer_frame(out), op, os) != 0)
    {
        hb_error("rotate(cuda): %s", hbcu_last_error());
        hb_buffer_close(&in);
        hb_buffer_close(&out);
        return HB_FILTER_FAILED;
    }
    if (fin != NULL)
        hb_buffer_close(&in);              /* the kernel is queued as a reader of the input frame */
    rotate_pending_t *p = &pv->pending[(pv->head + pv->count) % ROTATE_MAX_PENDING];
    p->in = in;
    p->out = out;
    p->ticket = ticket;
    pv->count++;

    if (harvest(pv, &list, 0) != 0)
    {
        hb_buffer_list_close(&list);
        return HB_FILTER_FAILED;
    }
    *buf_out = hb_buffer_list_clear(&list);
    return HB_FILTER_OK;
}
