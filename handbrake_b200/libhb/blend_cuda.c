/* blend_cuda.c -- hb_blend_cuda: drop-in for hb_blend (reference libhb/blend.c:788-885), the object libhb's subtitle
 * renderer (rendersub.c) composites its YUVA overlays with, running on an H100 through include/hbcu.h.
 *
 * Same init / work / close contract:
 *   - init takes the frame's geometry, format, chroma location and the overlay format; it fails (non-zero) for a
 *     combination blend.c's CUDA twin does not support (a semi-planar frame other than 4:2:0, a subsampled overlay on
 *     a frame with other subsampling) and when there is no usable device, so that the caller can take hb_blend
 *     instead.  Semi-planar 4:2:0 frames (NV12, P010, P016, what NVDEC decodes into) take blend.c's *bi* paths;
 *   - work composites the overlays in list order.  No overlays: the input buffer comes back as it is, nothing runs on
 *     the GPU (blend.c:856-859).  A host frame is blended in place (duplicated first if it is not writable,
 *     blend.c:861-865) and is finished when work returns.  A device frame is never written (frames are written once):
 *     the result is a new device frame, queued behind the input's producer, and work returns without waiting.
 *   - the overlays are copied before work returns: the caller frees or reuses them right after.  A list the caller
 *     marks unchanged, with the same count and geometry, is not uploaded again.
 * One device, hbcu_env_device().
 */
#include "handbrake/handbrake.h"
#include "hbcu.h"
#include "hbcu_device_frames.h"

struct hb_blend_private_s
{
    hbcu_blend_t         *gpu;
    int                   device;
    hbcu_blend_overlay_t *list;
    int                   list_cap;
};

static int          blend_cuda_init(hb_blend_object_t *object, int in_width, int in_height, int in_pix_fmt,
                                    int in_chroma_location, int in_color_range, int overlay_pix_fmt);
static hb_buffer_t *blend_cuda_work(hb_blend_object_t *object, hb_buffer_t *in, hb_buffer_list_t *overlays, int changed);
static void         blend_cuda_close(hb_blend_object_t *object);

hb_blend_object_t hb_blend_cuda =
{
    .name  = "Blend (CUDA sm_90a)",
    .init  = blend_cuda_init,
    .work  = blend_cuda_work,
    .close = blend_cuda_close,
};

static int blend_cuda_init(hb_blend_object_t *object, int in_width, int in_height, int in_pix_fmt,
                           int in_chroma_location, int in_color_range, int overlay_pix_fmt)
{
    (void)in_color_range;
    object->private_data = NULL;
    const AVPixFmtDescriptor *in_desc = av_pix_fmt_desc_get(in_pix_fmt);
    const AVPixFmtDescriptor *ov_desc = av_pix_fmt_desc_get(overlay_pix_fmt);
    const int in_planes = av_pix_fmt_count_planes(in_pix_fmt);
    /* blend.c:817-842 picks the *bi* functions by plane count; the semi-planar formats in use for them are 4:2:0 */
    const int semi_planar = in_desc != NULL && in_planes == 2 && in_desc->log2_chroma_w == 1 && in_desc->log2_chroma_h == 1;
    if (in_desc == NULL || ov_desc == NULL || (in_planes != 3 && !semi_planar) || in_desc->nb_components != 3 ||
        av_pix_fmt_count_planes(overlay_pix_fmt) != 4 || ov_desc->comp[0].depth != 8 ||
        in_desc->comp[0].depth < 8 || in_desc->comp[0].depth > 16)
    {
        hb_error("blend(cuda): unsupported frame format %d or overlay format %d", in_pix_fmt, overlay_pix_fmt);
        return -1;
    }
    const int subsample = in_desc->log2_chroma_w != ov_desc->log2_chroma_w || in_desc->log2_chroma_h != ov_desc->log2_chroma_h;
    if (subsample && (ov_desc->log2_chroma_w != 0 || ov_desc->log2_chroma_h != 0))
    {
        hb_error("blend(cuda): a %s overlay needs a frame with the same chroma subsampling", ov_desc->name);
        return -1;
    }
    hb_blend_private_t *pv = calloc(1, sizeof(*pv));
    if (pv == NULL)
    {
        hb_error("blend(cuda): calloc failed");
        return -1;
    }
    hbcu_blend_config_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.width           = in_width;
    cfg.height          = in_height;
    cfg.depth           = in_desc->comp[0].depth;
    cfg.chroma_shift_w  = in_desc->log2_chroma_w;
    cfg.chroma_shift_h  = in_desc->log2_chroma_h;
    cfg.overlay_shift_w = ov_desc->log2_chroma_w;
    cfg.overlay_shift_h = ov_desc->log2_chroma_h;
    cfg.device          = pv->device = hbcu_env_device();
    cfg.interleaved_chroma = semi_planar;
    hb_compute_chroma_smoothing_coefficient(cfg.chroma_coeffs, in_pix_fmt, in_chroma_location);
    if (hbcu_blend_create(&pv->gpu, &cfg) != 0)
    {
        hb_error("blend(cuda): %s", hbcu_last_error());
        free(pv);
        return -1;
    }
    object->private_data = pv;
    return 0;
}

static void blend_cuda_close(hb_blend_object_t *object)
{
    hb_blend_private_t *pv = object->private_data;
    if (pv == NULL) return;
    hbcu_blend_destroy(pv->gpu);          /* waits for the work in flight */
    free(pv->list);
    free(pv);
    object->private_data = NULL;
}

static hb_buffer_t *blend_cuda_work(hb_blend_object_t *object, hb_buffer_t *in, hb_buffer_list_t *overlays, int changed)
{
    hb_blend_private_t *pv = object->private_data;
    const int count = hb_buffer_list_count(overlays);
    if (count == 0)
        return in;

    if (count > pv->list_cap)
    {
        hbcu_blend_overlay_t *l = realloc(pv->list, sizeof(*l) * count);
        if (l == NULL)
        {
            hb_error("blend(cuda): out of memory");
            hb_buffer_close(&in);
            return NULL;
        }
        pv->list = l;
        pv->list_cap = count;
    }
    int i = 0;
    for (hb_buffer_t *o = hb_buffer_list_head(overlays); o != NULL; o = o->next, i++)
    {
        hbcu_blend_overlay_t *d = &pv->list[i];
        d->x = o->f.x;
        d->y = o->f.y;
        d->width = o->f.width;
        d->height = o->f.height;
        for (int p = 0; p < 4; p++)
        {
            d->planes[p]  = o->plane[p].data;
            d->strides[p] = o->plane[p].stride;
        }
    }
    if (hbcu_blend_set_overlays(pv->gpu, pv->list, count, changed) != 0)
        goto fail;

    hbcu_frame_t *fin = hbcu_buffer_frame(in);
    if (fin != NULL)
    {
        hb_buffer_t *out = hbcu_device_frame_buffer_init(in->f.fmt, in->f.width, in->f.height, pv->device);
        if (out == NULL)
            goto fail;
        out->f.color_prim      = in->f.color_prim;
        out->f.color_transfer  = in->f.color_transfer;
        out->f.color_matrix    = in->f.color_matrix;
        out->f.color_range     = in->f.color_range;
        out->f.chroma_location = in->f.chroma_location;
        hb_buffer_copy_props(out, in);
        if (hbcu_blend_frames(pv->gpu, fin, NULL, NULL, hbcu_buffer_frame(out), NULL, NULL) != 0)
        {
            hb_buffer_close(&out);
            goto fail;
        }
        hb_buffer_close(&in);              /* the copy is queued as a reader of the input frame */
        return out;
    }

    hb_buffer_t *out = in;
    if (hb_buffer_is_writable(in) == 0)
    {
        out = hb_buffer_dup(in);
        hb_buffer_close(&in);
        if (out == NULL)
        {
            hb_error("blend(cuda): out of memory");
            return NULL;
        }
        in = out;
    }
    void *planes[3] = {NULL, NULL, NULL};      /* a semi-planar frame has no plane 2 */
    int strides[3] = {0, 0, 0};
    for (int c = 0; c <= out->f.max_plane; c++)
    {
        planes[c]  = out->plane[c].data;
        strides[c] = out->plane[c].stride;
    }
    if (hbcu_blend_frames(pv->gpu, NULL, (const void *const *)planes, strides, NULL, planes, strides) != 0 ||
        hbcu_blend_wait(pv->gpu) != 0)
        goto fail;
    return out;

fail:
    hb_error("blend(cuda): %s", hbcu_last_error());
    hb_buffer_close(&in);
    return NULL;
}
