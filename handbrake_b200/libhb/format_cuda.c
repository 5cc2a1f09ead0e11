/* format_cuda.c -- hb_filter_format_cuda: drop-in for hb_filter_format (reference libhb/format.c) for the conversions a
 * hardware-decoded or hardware-encoded job needs between NVDEC / NVENC's semi-planar frames and the planar pipeline
 * formats, running on an H100 through include/hbcu.h (hbcu_format_*):
 *   nv12 <-> yuv420p, p010le <-> yuv420p10le       (lossless repacks, see handbrake_b200/csrc/format.cu)
 *
 * Same id, short name and settings template as hb_filter_format; the same init() contract (format.c:33-111):
 *   - no `format` key: the filter passes every frame through and init->pix_fmt is left as it is;
 *   - otherwise init->pix_fmt = av_get_pix_fmt(format) for the filters behind it;
 *   - a target equal to the input format passes every frame through untouched, with no device work;
 *   - any other pair (P016, 4:2:2 or 4:4:4, a change of depth, an unknown name) fails init() with an hb_error, so
 *     that the caller keeps hb_filter_format (INTEGRATION.md 2).
 * Host and HBCU_DEVICE buffers are taken per buffer: a device input gives a device output, a host input a host output
 * unless init->hw_pix_fmt asks for device frames.  Outputs leave in order from a bounded number in flight and carry the
 * input's props and colour fields; only f.fmt and the plane layout change.  A device input is closed as soon as its
 * conversion is queued (hbcu_format_convert records the kernel as the frame's reader), so a wrapped decoder surface goes
 * back to the decoder once the kernel has read it, not when a filter downstream has let go of the frame.  A host input
 * is closed once its copy to the device is done.  One device, hbcu_env_device().
 */
#include "handbrake/handbrake.h"
#include "hbcu.h"
#include "hbcu_device_frames.h"

#define FORMAT_INFLIGHT   4
#define FORMAT_MAX_PENDING (FORMAT_INFLIGHT + 2)

typedef struct
{
    hb_buffer_t *in, *out;       /* in: a host input, kept until its conversion is done; NULL for a device input */
    int64_t      ticket;
} format_pending_t;

struct hb_filter_private_s
{
    hbcu_format_t   *gpu;        /* NULL: pass-through */
    int              device, device_out;
    format_pending_t pending[FORMAT_MAX_PENDING];
    int              head, count;
    int64_t          next_ticket;
    hb_filter_init_t input, output;
};

static int  format_cuda_init(hb_filter_object_t *filter, hb_filter_init_t *init);
static int  format_cuda_work(hb_filter_object_t *filter, hb_buffer_t **buf_in, hb_buffer_t **buf_out);
static void format_cuda_close(hb_filter_object_t *filter);

/* format.c's template, "format=^"HB_ALL_REG"$" with libhb's HB_ALL_REG "(.*)", written out */
static const char format_cuda_template[] = "format=^(.*)$";

hb_filter_object_t hb_filter_format_cuda =
{
    .id                = HB_FILTER_FORMAT,
    .enforce_order     = 1,
    .name              = "Format (CUDA sm_90a)",
    .short_name        = "format",
    .settings          = NULL,
    .init              = format_cuda_init,
    .work              = format_cuda_work,
    .close             = format_cuda_close,
    .settings_template = format_cuda_template,
};

/* 4:2:0 with three components: 1 semi-planar, 0 planar, -1 anything else */
static int semi_planar_420(const AVPixFmtDescriptor *d, int planes)
{
    if (d == NULL || d->nb_components != 3 || d->log2_chroma_w != 1 || d->log2_chroma_h != 1) return -1;
    return planes == 2 ? 1 : planes == 3 ? 0 : -1;
}

static int format_cuda_init(hb_filter_object_t *filter, hb_filter_init_t *init)
{
    hb_filter_private_t *pv = calloc(1, sizeof(*pv));
    if (pv == NULL)
    {
        hb_error("format(cuda): calloc failed");
        return -1;
    }
    filter->private_data = pv;
    pv->input = *init;

    char *format = NULL;
    hb_dict_extract_string(&format, filter->settings, "format");
    if (format == NULL)
    {
        pv->output = *init;
        return 0;
    }
    const int target = av_get_pix_fmt(format);
    if (target == AV_PIX_FMT_NONE)
    {
        hb_error("format(cuda): unknown pixel format \"%s\"", format);
        goto fail;
    }
    if (target != init->pix_fmt)
    {
        /* the four repacks: same depth, 4:2:0 on both sides, one side semi-planar, 8 bits (NV12) or 10 bits (P010) */
        const AVPixFmtDescriptor *di = av_pix_fmt_desc_get(init->pix_fmt), *dt = av_pix_fmt_desc_get(target);
        const int si = semi_planar_420(di, av_pix_fmt_count_planes(init->pix_fmt));
        const int st = semi_planar_420(dt, av_pix_fmt_count_planes(target));
        const int depth = di != NULL ? di->comp[0].depth : 0;
        const AVPixFmtDescriptor *semi = si == 1 ? di : dt, *planar = si == 1 ? dt : di;
        if (si < 0 || st < 0 || si == st || dt->comp[0].depth != depth || (depth != 8 && depth != 10) ||
            semi->comp[0].shift != (depth > 8 ? 16 - depth : 0) || planar->comp[0].shift != 0)
        {
            hb_error("format(cuda): %s -> %s is not one of nv12 <-> yuv420p, p010le <-> yuv420p10le",
                     di != NULL ? di->name : "unknown", dt->name);
            goto fail;
        }
        hbcu_format_config_t cfg;
        memset(&cfg, 0, sizeof(cfg));
        cfg.width          = init->geometry.width;
        cfg.height         = init->geometry.height;
        cfg.depth          = depth;
        cfg.to_semi_planar = st == 1;
        cfg.device         = pv->device = hbcu_env_device();
        cfg.slots          = FORMAT_MAX_PENDING;
        if (hbcu_format_create(&pv->gpu, &cfg) != 0)
        {
            hb_error("format(cuda): %s", hbcu_last_error());
            goto fail;
        }
        pv->device_out = hbcu_init_wants_device_output(init);
    }
    free(format);
    init->pix_fmt = target;
    pv->output = *init;
    return 0;

fail:
    free(format);
    free(pv);
    filter->private_data = NULL;
    return -1;
}

static void format_cuda_close(hb_filter_object_t *filter)
{
    hb_filter_private_t *pv = filter->private_data;
    if (pv == NULL) return;
    hbcu_format_destroy(pv->gpu);          /* waits for the conversions in flight */
    for (int i = 0; i < pv->count; i++)
    {
        format_pending_t *p = &pv->pending[(pv->head + i) % FORMAT_MAX_PENDING];
        hb_buffer_close(&p->in);
        hb_buffer_close(&p->out);
    }
    free(pv);
    filter->private_data = NULL;
}

/* hands on the finished outputs in order: a device output at once (its readers order themselves behind the kernel), a
 * host side once its copies are done; waits only when more than FORMAT_INFLIGHT are pending, or for all of them */
static int harvest(hb_filter_private_t *pv, hb_buffer_list_t *list, int all)
{
    while (pv->count > 0)
    {
        format_pending_t *p = &pv->pending[pv->head];
        if (p->in == NULL && hbcu_buffer_frame(p->out) != NULL)
        {
            /* device in, device out: nothing to wait for */
        }
        else if (all || pv->count > FORMAT_INFLIGHT)
        {
            if (hbcu_format_wait(pv->gpu, p->ticket) != 0) goto gpu_error;
        }
        else
        {
            const int done = hbcu_format_poll(pv->gpu, p->ticket);
            if (done < 0) goto gpu_error;
            if (done == 0) break;
        }
        hb_buffer_list_append(list, p->out);
        p->out = NULL;
        hb_buffer_close(&p->in);
        pv->head = (pv->head + 1) % FORMAT_MAX_PENDING;
        pv->count--;
    }
    return 0;

gpu_error:
    hb_error("format(cuda): %s", hbcu_last_error());
    return -1;
}

static int format_cuda_work(hb_filter_object_t *filter, hb_buffer_t **buf_in, hb_buffer_t **buf_out)
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
    const int fmt = pv->output.pix_fmt;
    hb_buffer_t *out = (fin != NULL || pv->device_out) ? hbcu_device_frame_buffer_init(fmt, in->f.width, in->f.height, pv->device)
                                                       : hb_frame_buffer_init(fmt, in->f.width, in->f.height);
    if (out == NULL)
    {
        hb_error("format(cuda): out of memory");
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
    if (hbcu_format_convert(pv->gpu, ticket, fin, ip, is, hbcu_buffer_frame(out), op, os) != 0)
    {
        hb_error("format(cuda): %s", hbcu_last_error());
        hb_buffer_close(&in);
        hb_buffer_close(&out);
        return HB_FILTER_FAILED;
    }
    if (fin != NULL)
        hb_buffer_close(&in);              /* the kernel is queued as a reader of the input frame */
    format_pending_t *p = &pv->pending[(pv->head + pv->count) % FORMAT_MAX_PENDING];
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
