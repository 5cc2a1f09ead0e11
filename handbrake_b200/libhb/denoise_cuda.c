/* denoise_cuda.c -- hb_filter_denoise_cuda: drop-in for hb_filter_denoise (hqdn3d, reference libhb/denoise.c:64-76,
 * 214-371) running on an H100 through include/hbcu.h (SURVEY.md 8 f4).
 *
 * Same settings keys and default chain (denoise.c:237-266).  The coefficient tables are the numeric contract
 * (hqdn3d_precalc_coef, denoise.c:78-94): they are computed here, on the host, with the expressions of the reference and
 * handed to the device as they are.  Frames are filtered in arrival order (the temporal state chains them), a bounded
 * number in flight; they may arrive and leave as HBCU_DEVICE buffers.
 */
#include "handbrake/handbrake.h"
#include "hbcu.h"
#include "hbcu_device_frames.h"
#include <math.h>

#define HQDN3D_SPATIAL_LUMA_DEFAULT    4.0f
#define HQDN3D_SPATIAL_CHROMA_DEFAULT  3.0f
#define HQDN3D_TEMPORAL_LUMA_DEFAULT   6.0f
#define HQDN3D_MAX_PENDING             16

typedef struct
{
    hb_buffer_t *in, *out;
    int64_t      ticket;
} hqdn3d_pending_t;

struct hb_filter_private_s
{
    hbcu_hqdn3d_t *gpu;
    hqdn3d_pending_t pending[HQDN3D_MAX_PENDING];
    int head, count, inflight_max;
    int64_t next_ticket;
    int device, device_out;
    hb_filter_init_t input, output;
};

static int  denoise_cuda_init(hb_filter_object_t *filter, hb_filter_init_t *init);
static int  denoise_cuda_work(hb_filter_object_t *filter, hb_buffer_t **buf_in, hb_buffer_t **buf_out);
static void denoise_cuda_close(hb_filter_object_t *filter);

static const char denoise_template[] =
    "y-spatial=^"HB_FLOAT_REG"$:cb-spatial=^"HB_FLOAT_REG"$:"
    "cr-spatial=^"HB_FLOAT_REG"$:"
    "y-temporal=^"HB_FLOAT_REG"$:cb-temporal=^"HB_FLOAT_REG"$:"
    "cr-temporal=^"HB_FLOAT_REG"$";

hb_filter_object_t hb_filter_denoise_cuda =
{
    .id                = HB_FILTER_DENOISE,
    .enforce_order     = 1,
    .name              = "Denoise (hqdn3d, CUDA sm_90a)",
    .short_name        = "hqdn3d",
    .settings          = NULL,
    .init              = denoise_cuda_init,
    .work              = denoise_cuda_work,
    .close             = denoise_cuda_close,
    .settings_template = denoise_template,
};

/* denoise.c:78-94, evaluated on the host exactly as written there */
static void precalc_coef(int16_t *ct, int depth, double dist25)
{
    const int lut_bits = depth == 16 ? 8 : 4;
    double gamma, simil, C;

    gamma = log(0.25) / log(1.0 - (dist25 > 252.0 ? 252.0 : dist25) / 255.0 - 0.00001);
    for (int i = -(256 << lut_bits); i < 256 << lut_bits; i++)
    {
        double f = (i * (1 << (9 - lut_bits)) + (1 << (8 - lut_bits)) - 1) / 512.0;   /* midpoint of the bin */
        simil = 1.0 - fabs(f) / 255.0;
        if (simil < 0) simil = 0;
        C = pow(simil, gamma) * 256.0 * f;
        ct[(256 << lut_bits) + i] = lrint(C);
    }
    ct[0] = !!dist25;
}

static int denoise_cuda_init(hb_filter_object_t *filter, hb_filter_init_t *init)
{
    hb_filter_private_t *pv = calloc(1, sizeof(*pv));
    if (pv == NULL)
    {
        hb_error("denoise(cuda): calloc failed");
        return -1;
    }
    filter->private_data = pv;
    pv->input = *init;
    int16_t *tab[6] = { NULL, NULL, NULL, NULL, NULL, NULL };

    const AVPixFmtDescriptor *desc = av_pix_fmt_desc_get(init->pix_fmt);
    if (desc == NULL || desc->nb_components < 3 || av_pix_fmt_count_planes(init->pix_fmt) < 3)    /* planar YUV only */
    {
        hb_error("denoise(cuda): unsupported pixel format %d", init->pix_fmt);
        goto fail;
    }
    const int depth = desc->comp[0].depth;

    /* the default chain of denoise.c:237-266 */
    double spatial_luma, spatial_chroma_b, spatial_chroma_r;
    double temporal_luma, temporal_chroma_b, temporal_chroma_r;
    if (!hb_dict_extract_double(&spatial_luma, filter->settings, "y-spatial"))
        spatial_luma = HQDN3D_SPATIAL_LUMA_DEFAULT;
    if (!hb_dict_extract_double(&spatial_chroma_b, filter->settings, "cb-spatial"))
        spatial_chroma_b = HQDN3D_SPATIAL_CHROMA_DEFAULT * spatial_luma / HQDN3D_SPATIAL_LUMA_DEFAULT;
    if (!hb_dict_extract_double(&spatial_chroma_r, filter->settings, "cr-spatial"))
        spatial_chroma_r = spatial_chroma_b;
    if (!hb_dict_extract_double(&temporal_luma, filter->settings, "y-temporal"))
        temporal_luma = HQDN3D_TEMPORAL_LUMA_DEFAULT * spatial_luma / HQDN3D_SPATIAL_LUMA_DEFAULT;
    if (!hb_dict_extract_double(&temporal_chroma_b, filter->settings, "cb-temporal"))
        temporal_chroma_b = temporal_luma * spatial_chroma_b / spatial_luma;
    if (!hb_dict_extract_double(&temporal_chroma_r, filter->settings, "cr-temporal"))
        temporal_chroma_r = temporal_chroma_b;
    const double dist[6] = { spatial_luma, temporal_luma, spatial_chroma_b, temporal_chroma_b, spatial_chroma_r, temporal_chroma_r };

    hbcu_hqdn3d_config_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    const int entries = 512 << (depth == 16 ? 8 : 4);
    for (int i = 0; i < 6; i++)
    {
        tab[i] = malloc((size_t)entries * sizeof(int16_t));
        if (tab[i] == NULL) goto fail;
        precalc_coef(tab[i], depth, dist[i]);
        cfg.coef[i] = tab[i];
    }
    cfg.width          = init->geometry.width;
    cfg.height         = init->geometry.height;
    cfg.depth          = depth;
    cfg.chroma_shift_w = desc->log2_chroma_w;
    cfg.chroma_shift_h = desc->log2_chroma_h;
    cfg.device         = hbcu_env_device();
    pv->device         = cfg.device;
    pv->device_out     = hbcu_init_wants_device_output(init);
    pv->inflight_max   = 6;
    cfg.slots          = pv->inflight_max + 2;
    if (hbcu_hqdn3d_create(&pv->gpu, &cfg) != 0)
    {
        hb_error("denoise(cuda): %s", hbcu_last_error());
        goto fail;
    }
    for (int i = 0; i < 6; i++) free(tab[i]);
    pv->output = *init;
    return 0;

fail:
    for (int i = 0; i < 6; i++) free(tab[i]);
    free(pv);
    filter->private_data = NULL;
    return -1;
}

static void denoise_cuda_close(hb_filter_object_t *filter)
{
    hb_filter_private_t *pv = filter->private_data;
    if (pv == NULL) return;
    if (pv->gpu != NULL) hbcu_hqdn3d_destroy(pv->gpu);
    for (int i = 0; i < pv->count; i++)
    {
        hqdn3d_pending_t *p = &pv->pending[(pv->head + i) % HQDN3D_MAX_PENDING];
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
        hqdn3d_pending_t *p = &pv->pending[pv->head];
        if (hbcu_buffer_frame(p->out) != NULL && hbcu_buffer_frame(p->in) != NULL)
        {
            /* device in, device out: the frame's events order the GPU work */
        }
        else if (all || pv->count > pv->inflight_max)
        {
            if (hbcu_hqdn3d_wait(pv->gpu, p->ticket) != 0) goto gpu_error;
        }
        else
        {
            const int done = hbcu_hqdn3d_poll(pv->gpu, p->ticket);
            if (done < 0) goto gpu_error;
            if (done == 0) break;
        }
        hb_buffer_list_append(list, p->out);
        p->out = NULL;
        hb_buffer_close(&p->in);
        pv->head = (pv->head + 1) % HQDN3D_MAX_PENDING;
        pv->count--;
    }
    return 0;

gpu_error:
    hb_error("denoise(cuda): %s", hbcu_last_error());
    return -1;
}

static int denoise_cuda_work(hb_filter_object_t *filter, hb_buffer_t **buf_in, hb_buffer_t **buf_out)
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
    if (hbcu_hqdn3d_filter_frames(pv->gpu, ticket, hbcu_buffer_frame(in), ip, is, hbcu_buffer_frame(out), op, os) != 0)
    {
        hb_error("denoise(cuda): %s", hbcu_last_error());
        hb_buffer_close(&in);
        hb_buffer_close(&out);
        return HB_FILTER_FAILED;
    }
    hqdn3d_pending_t *p = &pv->pending[(pv->head + pv->count) % HQDN3D_MAX_PENDING];
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
