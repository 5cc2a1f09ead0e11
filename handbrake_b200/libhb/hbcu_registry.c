/* hbcu_registry.c -- how the CUDA filter objects are substituted for the CPU
 * ones: hb_filter_get() (libhb/common.c:5331-5495) returns the *_cuda object
 * for the ids this library implements, i.e. exactly the pointer swap a libhb
 * maintainer would make (cf. replace_filter, platform/macosx/vt_common.c:486-535).
 */
#include "handbrake/handbrake.h"

extern hb_filter_object_t hb_filter_nlmeans_cuda;
extern hb_filter_object_t hb_filter_comb_detect_cuda;
extern hb_filter_object_t hb_filter_decomb_cuda;
extern hb_filter_object_t hb_filter_lapsharp_cuda;
extern hb_filter_object_t hb_filter_unsharp_cuda;
extern hb_filter_object_t hb_filter_denoise_cuda;
extern hb_filter_object_t hb_filter_chroma_smooth_cuda;
extern hb_filter_object_t hb_filter_detelecine_cuda;
extern hb_filter_object_t hb_filter_vfr_cuda;
extern hb_filter_object_t hb_filter_format_cuda;
extern hb_filter_object_t hb_filter_rotate_cuda;
extern hb_filter_object_t hb_filter_yadif_cuda;
extern hb_filter_object_t hb_filter_bwdif_cuda;

hb_filter_object_t *hb_filter_get(int filter_id)
{
    switch (filter_id)
    {
        case HB_FILTER_NLMEANS:     return &hb_filter_nlmeans_cuda;
        case HB_FILTER_COMB_DETECT: return &hb_filter_comb_detect_cuda;
        case HB_FILTER_DECOMB:      return &hb_filter_decomb_cuda;
        case HB_FILTER_LAPSHARP:    return &hb_filter_lapsharp_cuda;   /* no mt_frame wrapper needed: streams */
        case HB_FILTER_UNSHARP:     return &hb_filter_unsharp_cuda;
        case HB_FILTER_DENOISE:     return &hb_filter_denoise_cuda;    /* hqdn3d */
        case HB_FILTER_CHROMA_SMOOTH: return &hb_filter_chroma_smooth_cuda;
        case HB_FILTER_DETELECINE:  return &hb_filter_detelecine_cuda;    /* pullup: metrics on the device, decisions on the host */
        case HB_FILTER_VFR:         return &hb_filter_vfr_cuda;           /* motion metric on the device, read only when a drop is due */
        case HB_FILTER_FORMAT:      return &hb_filter_format_cuda;        /* nv12 / p010le <-> planar; init fails for other pairs */
        case HB_FILTER_ROTATE:      return &hb_filter_rotate_cuda;        /* flips and transposes; init fails for 4:2:2 transposes */
        case HB_FILTER_YADIF:       return &hb_filter_yadif_cuda;         /* init fails for semi-planar, gray and YUVA input */
        case HB_FILTER_BWDIF:       return &hb_filter_bwdif_cuda;
        default:                return NULL;
    }
}

/* common.c:5497-5517 */
hb_filter_object_t *hb_filter_init(int filter_id)
{
    hb_filter_object_t *src = hb_filter_get(filter_id);
    if (src == NULL) return NULL;
    hb_filter_object_t *f = malloc(sizeof(*f));
    if (f == NULL) return NULL;
    memcpy(f, src, sizeof(*f));
    return f;
}

void hb_filter_close(hb_filter_object_t **pf)
{
    if (pf == NULL || *pf == NULL) return;
    hb_filter_object_t *f = *pf;
    if (f->sub_filter != NULL) hb_filter_close(&f->sub_filter);
    if (f->settings != NULL) hb_dict_free(&f->settings);
    free(f);
    *pf = NULL;
}
