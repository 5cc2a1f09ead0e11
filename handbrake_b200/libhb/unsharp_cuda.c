/* unsharp_cuda.c -- hb_filter_unsharp_cuda and hb_filter_chroma_smooth_cuda: drop-ins for hb_filter_unsharp /
 * hb_filter_chroma_smooth wrapped in hb_filter_mt_frame (reference libhb/unsharp.c:70-84, chroma_smooth.c:72-86,
 * mt_frame_filter.c:45-237, common.c:5497-5517) running on an H100 through include/hbcu.h (SURVEY.md 8 f2).
 *
 * Same settings keys, cascade, defaults and sanitising (unsharp.c:213-276, chroma_smooth.c:196-270).  mt_frame's
 * "collect cpu_count frames, run them on cpu_count threads, emit them together" becomes frames in flight on the
 * handle's streams, emitted in order as they complete; frames may arrive and leave as HBCU_DEVICE buffers.
 */
#include "handbrake/handbrake.h"
#include "hbcu.h"
#include "hbcu_device_frames.h"

#define UNSHARP_STRENGTH_DEFAULT        0.25
#define UNSHARP_SIZE_DEFAULT            7
#define UNSHARP_SIZE_MIN                3
#define UNSHARP_SIZE_MAX                15
#define UNSHARP_MAX_PENDING             64

typedef struct
{
    hb_buffer_t *in, *out;
    int64_t      ticket;
    int          dev;
} unsharp_pending_t;

struct hb_filter_private_s
{
    hbcu_unsharp_t *gpu[HBCU_MAX_DEVICES];     /* frames are independent: frame t goes to device t % ndev (mt_frame_filter.c:169-237) */
    int ndev, devices[HBCU_MAX_DEVICES];
    unsharp_pending_t pending[UNSHARP_MAX_PENDING];
    int head, count, inflight_max;
    int64_t next_ticket;
    int device, device_out, smooth;
    hb_filter_init_t input, output;
};

static int  unsharp_cuda_init(hb_filter_object_t *filter, hb_filter_init_t *init);
static int  unsharp_cuda_work(hb_filter_object_t *filter, hb_buffer_t **buf_in, hb_buffer_t **buf_out);
static void unsharp_cuda_close(hb_filter_object_t *filter);

static const char unsharp_template[] =
    "y-strength=^"HB_FLOAT_REG"$:y-size=^"HB_INT_REG"$:"
    "cb-strength=^"HB_FLOAT_REG"$:cb-size=^"HB_INT_REG"$:"
    "cr-strength=^"HB_FLOAT_REG"$:cr-size=^"HB_INT_REG"$";

static const char chroma_smooth_template[] =
    "cb-strength=^"HB_FLOAT_REG"$:cb-size=^"HB_INT_REG"$:"
    "cr-strength=^"HB_FLOAT_REG"$:cr-size=^"HB_INT_REG"$";

hb_filter_object_t hb_filter_unsharp_cuda =
{
    .id                = HB_FILTER_UNSHARP,
    .enforce_order     = 1,
    .name              = "Sharpen (unsharp, CUDA sm_90a)",
    .short_name        = "unsharp",
    .settings          = NULL,
    .init              = unsharp_cuda_init,
    .work              = unsharp_cuda_work,
    .close             = unsharp_cuda_close,
    .settings_template = unsharp_template,
};

hb_filter_object_t hb_filter_chroma_smooth_cuda =
{
    .id                = HB_FILTER_CHROMA_SMOOTH,
    .enforce_order     = 1,
    .name              = "Chroma Smooth (CUDA sm_90a)",
    .short_name        = "chromasmooth",
    .settings          = NULL,
    .init              = unsharp_cuda_init,
    .work              = unsharp_cuda_work,
    .close             = unsharp_cuda_close,
    .settings_template = chroma_smooth_template,
};

static int unsharp_cuda_init(hb_filter_object_t *filter, hb_filter_init_t *init)
{
    static const char *const keys_s[3] = { "y-strength", "cb-strength", "cr-strength" };
    static const char *const keys_z[3] = { "y-size", "cb-size", "cr-size" };
    hb_filter_private_t *pv = calloc(1, sizeof(*pv));
    if (pv == NULL)
    {
        hb_error("unsharp(cuda): calloc failed");
        return -1;
    }
    filter->private_data = pv;
    pv->input  = *init;
    pv->smooth = filter->id == HB_FILTER_CHROMA_SMOOTH;

    const AVPixFmtDescriptor *desc = av_pix_fmt_desc_get(init->pix_fmt);
    if (desc == NULL || desc->nb_components < 3)
    {
        hb_error("unsharp(cuda): unsupported pixel format %d", init->pix_fmt);
        goto fail;
    }
    double strength[3] = { -1, -1, -1 };
    int    size[3]     = { -1, -1, -1 };
    /* chroma_smooth reads only the cb-/cr- keys (chroma_smooth.c:205-213) */
    for (int c = pv->smooth ? 1 : 0; c < 3 && filter->settings != NULL; c++)
    {
        hb_dict_extract_double(&strength[c], filter->settings, keys_s[c]);
        hb_dict_extract_int(&size[c], filter->settings, keys_z[c]);
    }
    /* Cr inherits Cb; for unsharp Cb inherits Y (unsharp.c:232-241, chroma_smooth.c:215-224) */
    for (int c = pv->smooth ? 2 : 1; c < 3; c++)
    {
        if (strength[c] == -1) strength[c] = strength[c - 1];
        if (size[c]     == -1) size[c]     = size[c - 1];
    }
    hbcu_unsharp_config_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    const double strength_max = pv->smooth ? 3.0 : 1.5;
    for (int c = 0; c < 3; c++)
    {
        if (strength[c] == -1) strength[c] = UNSHARP_STRENGTH_DEFAULT;
        if (size[c]     == -1) size[c]     = UNSHARP_SIZE_DEFAULT;
        if (strength[c] < 0)            strength[c] = 0;
        if (strength[c] > strength_max) strength[c] = strength_max;
        if (size[c] % 2 == 0) size[c]--;
        if (size[c] < UNSHARP_SIZE_MIN) size[c] = UNSHARP_SIZE_MIN;
        if (size[c] > UNSHARP_SIZE_MAX) size[c] = UNSHARP_SIZE_MAX;
        cfg.amount[c] = strength[c] * 65536.0;                 /* double -> int, unsharp.c:273 */
        cfg.steps[c]  = size[c] / 2;
        if (pv->smooth && c == 0) cfg.amount[c] = 0;           /* luma passes through, chroma_smooth.c:262-268 */
    }
    cfg.width          = init->geometry.width;
    cfg.height         = init->geometry.height;
    cfg.depth          = desc->comp[0].depth;
    cfg.chroma_shift_w = desc->log2_chroma_w;
    cfg.chroma_shift_h = desc->log2_chroma_h;
    cfg.smooth         = pv->smooth;
    pv->ndev           = hbcu_settings_devices(filter->settings, pv->devices);
    pv->device_out     = hbcu_init_wants_device_output(init);
    if (pv->ndev < 1 || (pv->ndev > 1 && pv->device_out))
    {
        hb_error("%s(cuda): %s", filter->short_name, pv->ndev < 1 ? "bad `devices` setting" : "device-resident output needs a single device");
        goto fail;
    }
    pv->device         = pv->devices[0];
    pv->inflight_max   = 6 * pv->ndev < UNSHARP_MAX_PENDING - 2 ? 6 * pv->ndev : UNSHARP_MAX_PENDING - 2;
    cfg.slots          = 6 + 2;
    for (int d = 0; d < pv->ndev; d++)
    {
        cfg.device = pv->devices[d];
        if (hbcu_unsharp_create(&pv->gpu[d], &cfg) != 0)
        {
            hb_error("%s(cuda): %s", filter->short_name, hbcu_last_error());
            goto fail;
        }
    }
    pv->output = *init;
    return 0;

fail:
    for (int d = 0; d < HBCU_MAX_DEVICES; d++)
        if (pv->gpu[d] != NULL) hbcu_unsharp_destroy(pv->gpu[d]);
    free(pv);
    filter->private_data = NULL;
    return -1;
}

static void unsharp_cuda_close(hb_filter_object_t *filter)
{
    hb_filter_private_t *pv = filter->private_data;
    if (pv == NULL) return;
    for (int d = 0; d < pv->ndev; d++)
        if (pv->gpu[d] != NULL) hbcu_unsharp_destroy(pv->gpu[d]);      /* waits for the copies in flight */
    for (int i = 0; i < pv->count; i++)
    {
        unsharp_pending_t *p = &pv->pending[(pv->head + i) % UNSHARP_MAX_PENDING];
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
        unsharp_pending_t *p = &pv->pending[pv->head];
        if (hbcu_buffer_frame(p->out) != NULL && hbcu_buffer_frame(p->in) != NULL)
        {
            /* device in, device out: the frame's events order the GPU work, nothing to wait for here */
        }
        else if (all || pv->count > pv->inflight_max)
        {
            if (hbcu_unsharp_wait(pv->gpu[p->dev], p->ticket) != 0) goto gpu_error;
        }
        else
        {
            const int done = hbcu_unsharp_poll(pv->gpu[p->dev], p->ticket);
            if (done < 0) goto gpu_error;
            if (done == 0) break;
        }
        hb_buffer_list_append(list, p->out);
        p->out = NULL;
        hb_buffer_close(&p->in);
        pv->head = (pv->head + 1) % UNSHARP_MAX_PENDING;
        pv->count--;
    }
    return 0;

gpu_error:
    hb_error("unsharp(cuda): %s", hbcu_last_error());
    return -1;
}

static int unsharp_cuda_work(hb_filter_object_t *filter, hb_buffer_t **buf_in, hb_buffer_t **buf_out)
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
    if (hbcu_buffer_frame(in) != NULL && pv->ndev > 1)
    {
        hb_error("%s(cuda): device-resident input needs a single device", filter->short_name);
        hb_buffer_close(&in);
        hb_buffer_close(&out);
        return HB_FILTER_FAILED;
    }
    if (hbcu_unsharp_filter_frames(pv->gpu[dev], ticket, hbcu_buffer_frame(in), ip, is, hbcu_buffer_frame(out), op, os) != 0)
    {
        hb_error("%s(cuda): %s", filter->short_name, hbcu_last_error());
        hb_buffer_close(&in);
        hb_buffer_close(&out);
        return HB_FILTER_FAILED;
    }
    unsharp_pending_t *p = &pv->pending[(pv->head + pv->count) % UNSHARP_MAX_PENDING];
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
