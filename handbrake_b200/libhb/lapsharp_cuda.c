/* lapsharp_cuda.c -- hb_filter_lapsharp_cuda: drop-in for hb_filter_lapsharp wrapped in
 * hb_filter_mt_frame (reference libhb/lapsharp.c:112-123, mt_frame_filter.c:45-237,
 * common.c:5497-5517) running on an H100 through include/hbcu.h.
 *
 * Same settings (y-/cb-/cr-strength, -kernel with the names lap/isolap/log/isolog), same
 * cascade/defaults/sanitising (lapsharp.c:228-297).  mt_frame's "collect cpu_count frames,
 * run them on cpu_count threads, emit them together" becomes: every frame is enqueued at once
 * on the handle's streams, `slots` frames in flight, emitted in order as they complete.
 */
#include "handbrake/handbrake.h"
#include "hbcu.h"
#include "hbcu_device_frames.h"
#include <strings.h>

#define LAPSHARP_STRENGTH_DEFAULT 0.2
#define LAPSHARP_KERNEL_DEFAULT   2
#define LAPSHARP_KERNELS          4
#define LAPSHARP_MAX_PENDING      64

typedef struct
{
    hb_buffer_t *in, *out;
    int64_t      ticket;
    int          dev;
} lapsharp_pending_t;

struct hb_filter_private_s
{
    hbcu_lapsharp_t *gpu[HBCU_MAX_DEVICES];    /* frames are independent: frame t goes to device t % ndev (mt_frame_filter.c:169-237) */
    int ndev, devices[HBCU_MAX_DEVICES];
    lapsharp_pending_t pending[LAPSHARP_MAX_PENDING];
    int head, count, inflight_max;
    int64_t next_ticket;
    int device, device_out;            /* device_out: hand the output on as HBCU_DEVICE buffers (hw_pix_fmt == AV_PIX_FMT_CUDA) */
    hb_filter_init_t input, output;
};

static int  lapsharp_cuda_init(hb_filter_object_t *filter, hb_filter_init_t *init);
static int  lapsharp_cuda_work(hb_filter_object_t *filter, hb_buffer_t **buf_in, hb_buffer_t **buf_out);
static void lapsharp_cuda_close(hb_filter_object_t *filter);

static const char lapsharp_template[] =
    "y-strength=^"HB_FLOAT_REG"$:y-kernel=^"HB_ALL_REG"$:"
    "cb-strength=^"HB_FLOAT_REG"$:cb-kernel=^"HB_ALL_REG"$:"
    "cr-strength=^"HB_FLOAT_REG"$:cr-kernel=^"HB_ALL_REG"$";

hb_filter_object_t hb_filter_lapsharp_cuda =
{
    .id                = HB_FILTER_LAPSHARP,
    .enforce_order     = 1,
    .name              = "Sharpen (lapsharp, CUDA sm_90a)",
    .short_name        = "lapsharp",
    .settings          = NULL,
    .init              = lapsharp_cuda_init,
    .work              = lapsharp_cuda_work,
    .close             = lapsharp_cuda_close,
    .settings_template = lapsharp_template,
};

static int lapsharp_cuda_init(hb_filter_object_t *filter, hb_filter_init_t *init)
{
    static const char *const names[LAPSHARP_KERNELS] = { "lap", "isolap", "log", "isolog" };
    static const char *const keys_s[3] = { "y-strength", "cb-strength", "cr-strength" };
    static const char *const keys_k[3] = { "y-kernel", "cb-kernel", "cr-kernel" };
    hb_filter_private_t *pv = calloc(1, sizeof(*pv));
    if (pv == NULL)
    {
        hb_error("lapsharp(cuda): calloc failed");
        return -1;
    }
    filter->private_data = pv;
    pv->input = *init;

    const AVPixFmtDescriptor *desc = av_pix_fmt_desc_get(init->pix_fmt);
    if (desc == NULL || desc->nb_components < 3)
    {
        hb_error("lapsharp(cuda): unsupported pixel format %d", init->pix_fmt);
        goto fail;
    }
    hbcu_lapsharp_config_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    for (int c = 0; c < 3; c++)
    {
        cfg.strength[c] = -1;
        cfg.kernel[c]   = -1;
        char *name = NULL;
        if (filter->settings != NULL)
        {
            hb_dict_extract_double(&cfg.strength[c], filter->settings, keys_s[c]);
            hb_dict_extract_string(&name, filter->settings, keys_k[c]);
        }
        if (name != NULL)
        {
            for (int k = 0; k < LAPSHARP_KERNELS; k++)
                if (!strcasecmp(name, names[k])) cfg.kernel[c] = k;
            free(name);
        }
    }
    for (int c = 1; c < 3; c++)      /* Cr inherits Cb inherits Y (lapsharp.c:268-276) */
    {
        if (cfg.strength[c] == -1) cfg.strength[c] = cfg.strength[c - 1];
        if (cfg.kernel[c]   == -1) cfg.kernel[c]   = cfg.kernel[c - 1];
    }
    for (int c = 0; c < 3; c++)
    {
        if (cfg.strength[c] == -1) cfg.strength[c] = LAPSHARP_STRENGTH_DEFAULT;
        if (cfg.kernel[c]   == -1) cfg.kernel[c]   = LAPSHARP_KERNEL_DEFAULT;
        if (cfg.strength[c] < 0)   cfg.strength[c] = 0;
        if (cfg.strength[c] > 1.5) cfg.strength[c] = 1.5;
        if (cfg.kernel[c] < 0 || cfg.kernel[c] >= LAPSHARP_KERNELS) cfg.kernel[c] = LAPSHARP_KERNEL_DEFAULT;
    }
    cfg.width          = init->geometry.width;
    cfg.height         = init->geometry.height;
    cfg.depth          = desc->comp[0].depth;
    cfg.chroma_shift_w = desc->log2_chroma_w;
    cfg.chroma_shift_h = desc->log2_chroma_h;
    pv->ndev = hbcu_settings_devices(filter->settings, pv->devices);
    pv->device_out     = hbcu_init_wants_device_output(init);
    if (pv->ndev < 1 || (pv->ndev > 1 && pv->device_out))
    {
        hb_error(pv->ndev < 1 ? "lapsharp(cuda): bad `devices` setting" : "lapsharp(cuda): device-resident output needs a single device");
        goto fail;
    }
    pv->device         = pv->devices[0];
    pv->inflight_max   = 6 * pv->ndev < LAPSHARP_MAX_PENDING - 2 ? 6 * pv->ndev : LAPSHARP_MAX_PENDING - 2;
    cfg.slots          = 6 + 2;
    for (int d = 0; d < pv->ndev; d++)
    {
        cfg.device = pv->devices[d];
        if (hbcu_lapsharp_create(&pv->gpu[d], &cfg) != 0)
        {
            hb_error("lapsharp(cuda): %s", hbcu_last_error());
            goto fail;
        }
    }
    pv->output = *init;
    return 0;

fail:
    for (int d = 0; d < HBCU_MAX_DEVICES; d++)
        if (pv->gpu[d] != NULL) hbcu_lapsharp_destroy(pv->gpu[d]);
    free(pv);
    filter->private_data = NULL;
    return -1;
}

static void lapsharp_cuda_close(hb_filter_object_t *filter)
{
    hb_filter_private_t *pv = filter->private_data;
    if (pv == NULL) return;
    for (int d = 0; d < pv->ndev; d++)
        if (pv->gpu[d] != NULL) hbcu_lapsharp_destroy(pv->gpu[d]);
    for (int i = 0; i < pv->count; i++)
    {
        lapsharp_pending_t *p = &pv->pending[(pv->head + i) % LAPSHARP_MAX_PENDING];
        hb_buffer_close(&p->in);
        hb_buffer_close(&p->out);
    }
    free(pv);
    filter->private_data = NULL;
}

static int harvest(hb_filter_private_t *pv, hb_buffer_list_t *list, int all)
{
    while (pv->count > 0)
    {
        lapsharp_pending_t *p = &pv->pending[pv->head];
        if (hbcu_buffer_frame(p->out) != NULL && hbcu_buffer_frame(p->in) != NULL)
        {
            /* device in, device out: nothing for the host to wait for, the frame's events order the GPU work */
        }
        else if (all || pv->count > pv->inflight_max)
        {
            if (hbcu_lapsharp_wait(pv->gpu[p->dev], p->ticket) != 0) goto gpu_error;
        }
        else
        {
            const int done = hbcu_lapsharp_poll(pv->gpu[p->dev], p->ticket);
            if (done < 0) goto gpu_error;
            if (done == 0) break;
        }
        hb_buffer_list_append(list, p->out);
        p->out = NULL;
        hb_buffer_close(&p->in);
        pv->head = (pv->head + 1) % LAPSHARP_MAX_PENDING;
        pv->count--;
    }
    return 0;

gpu_error:
    hb_error("lapsharp(cuda): %s", hbcu_last_error());
    return -1;
}

static int lapsharp_cuda_work(hb_filter_object_t *filter, hb_buffer_t **buf_in, hb_buffer_t **buf_out)
{
    hb_filter_private_t *pv = filter->private_data;
    hb_buffer_t *in = *buf_in;
    hb_buffer_list_t list;
    hb_buffer_list_clear(&list);

    *buf_in = NULL;
    if (in->s.flags & HB_BUF_FLAG_EOF)
    {
        const int failed = harvest(pv, &list, 1) != 0;
        hb_buffer_list_append(&list, in);
        *buf_out = hb_buffer_list_clear(&list);
        return failed ? HB_FILTER_FAILED : HB_FILTER_DONE;
    }

    /* lapsharp.c:333: the stride region next to the right edge is part of the filter's input
     * (for a device frame hbcu_lapsharp_filter_frames does the same in HBM) */
    hbcu_frame_t *fin = hbcu_buffer_frame(in);
    if (fin == NULL) hb_frame_buffer_mirror_stride(in);
    hb_buffer_t *out = pv->device_out ? hbcu_device_frame_buffer_init(pv->output.pix_fmt, in->f.width, in->f.height, pv->device)
                                      : hb_frame_buffer_init(pv->output.pix_fmt, in->f.width, in->f.height);
    if (out == NULL)
    {
        hb_buffer_close(&in);
        return HB_FILTER_FAILED;
    }
    out->f.color_prim      = pv->output.color_prim;
    out->f.color_transfer  = pv->output.color_transfer;
    out->f.color_matrix    = pv->output.color_matrix;
    out->f.color_range     = pv->output.color_range;
    out->f.chroma_location = pv->output.chroma_location;
    hb_buffer_copy_props(out, in);

    const void *ip[3];
    void *op[3];
    int is[3], os[3];
    for (int c = 0; c < 3; c++)
    {
        ip[c] = in->plane[c].data;  is[c] = in->plane[c].stride;
        op[c] = out->plane[c].data; os[c] = out->plane[c].stride;
    }
    const int64_t ticket = pv->next_ticket++;
    const int dev = (int)(ticket % pv->ndev);
    if (fin != NULL && pv->ndev > 1)
    {
        hb_error("lapsharp(cuda): device-resident input needs a single device");
        hb_buffer_close(&in);
        hb_buffer_close(&out);
        return HB_FILTER_FAILED;
    }
    if (hbcu_lapsharp_filter_frames(pv->gpu[dev], ticket, fin, ip, is, hbcu_buffer_frame(out), op, os) != 0)
    {
        hb_error("lapsharp(cuda): %s", hbcu_last_error());
        hb_buffer_close(&in);
        hb_buffer_close(&out);
        return HB_FILTER_FAILED;
    }
    lapsharp_pending_t *p = &pv->pending[(pv->head + pv->count) % LAPSHARP_MAX_PENDING];
    p->in = in;
    p->out = out;
    p->ticket = ticket;
    p->dev = dev;
    pv->count++;

    if (harvest(pv, &list, 0) != 0)
    {
        hb_buffer_list_close(&list);
        return HB_FILTER_FAILED;
    }
    *buf_out = hb_buffer_list_clear(&list);
    return HB_FILTER_OK;
}
