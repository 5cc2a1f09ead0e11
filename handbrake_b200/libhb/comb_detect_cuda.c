/* comb_detect_cuda.c -- hb_filter_comb_detect_cuda: drop-in for hb_filter_comb_detect
 * (reference libhb/comb_detect.c:129-140) running on an H100 through include/hbcu.h.
 *
 * Same plugin surface as the reference: same settings keys and defaults
 * (comb_detect.c:1118-1140), thresholds scaled by depth (:1152-1153), gamma table
 * built on the host with the reference's expression (:1074-1081) and uploaded,
 * three-frame window with the first frame duplicated as its own predecessor and
 * the last as its own successor, exhaustive check on those two passes
 * (:1111,1534,1552), frames passed through untouched with s.combed set, a frame
 * leaves only once more than three are queued (:1579-1582), close-time log line.
 *
 * What changes: the verdict of a frame is computed asynchronously (luma upload
 * and three kernels on the filter's streams) and collected when the frame is
 * about to leave the queue, three calls later, so work() never waits for the GPU
 * in steady state.  The debug modes that paint the mask into the picture
 * (MODE_MASK 4, MODE_COMPOSITE 8; comb_detect.c:23-26) are not implemented:
 * init() fails for them and libhb drops the filter.
 */
#include "handbrake/handbrake.h"
#include "hbcu.h"
#include "hbcu_device_frames.h"

#define MODE_GAMMA        1
#define MODE_FILTER       2
#define MODE_MASK         4
#define MODE_COMPOSITE    8

#define FILTER_CLASSIC      1
#define FILTER_ERODE_DILATE 2

struct hb_filter_private_s
{
    hbcu_comb_detect_t *gpu;

    /* reference window: ref[0] prev, ref[1] cur, ref[2] next, with their frame indices */
    hb_buffer_t *ref[3];
    int64_t      ref_index[3];
    int          ref_used[3];        /* 1: the buffer also sits in out_list (must not be closed here) */

    hb_buffer_list_t out_list;
    int64_t          out_index[8];   /* frame index of each queued buffer, oldest first */
    int              out_pending[8]; /* verdict not collected yet */
    int              out_count;

    int64_t next_index;
    int     ready;
    int     force_exhaustive;
    int     mode;

    int comb_heavy, comb_light, comb_none, frames;
};

static int  comb_detect_cuda_init(hb_filter_object_t *filter, hb_filter_init_t *init);
static int  comb_detect_cuda_work(hb_filter_object_t *filter, hb_buffer_t **buf_in, hb_buffer_t **buf_out);
static void comb_detect_cuda_close(hb_filter_object_t *filter);

static const char comb_detect_template[] =
    "mode=^"HB_INT_REG"$:spatial-metric=^([012])$:"
    "motion-thresh=^"HB_INT_REG"$:spatial-thresh=^"HB_INT_REG"$:"
    "filter-mode=^([012])$:block-thresh=^"HB_INT_REG"$:"
    "block-width=^"HB_INT_REG"$:block-height=^"HB_INT_REG"$:"
    "disable=^"HB_BOOL_REG"$";

hb_filter_object_t hb_filter_comb_detect_cuda =
{
    .id                = HB_FILTER_COMB_DETECT,
    .enforce_order     = 1,
    .name              = "Comb Detect (CUDA sm_90a)",
    .short_name        = "comb-detect",
    .settings          = NULL,
    .init              = comb_detect_cuda_init,
    .work              = comb_detect_cuda_work,
    .close             = comb_detect_cuda_close,
    .settings_template = comb_detect_template,
};

static int comb_detect_cuda_init(hb_filter_object_t *filter, hb_filter_init_t *init)
{
    hb_filter_private_t *pv = calloc(1, sizeof(*pv));
    if (pv == NULL)
    {
        hb_error("comb_detect(cuda): calloc failed");
        return -1;
    }
    filter->private_data = pv;
    hb_buffer_list_clear(&pv->out_list);

    const AVPixFmtDescriptor *desc = av_pix_fmt_desc_get(init->pix_fmt);
    if (desc == NULL)
    {
        hb_error("comb_detect(cuda): unsupported pixel format %d", init->pix_fmt);
        goto fail;
    }
    const int depth     = desc->comp[0].depth;
    const int max_value = (1 << depth) - 1;

    hbcu_comb_detect_config_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    /* defaults, comb_detect.c:1118-1125 */
    int mode = MODE_GAMMA | MODE_FILTER, filter_mode = FILTER_ERODE_DILATE, spatial_metric = 2;
    int motion_threshold = 3, spatial_threshold = 3;
    int block_threshold = 40, block_width = 16, block_height = 16;
    if (filter->settings)
    {
        hb_dict_t *dict = filter->settings;
        hb_dict_extract_int(&mode, dict, "mode");
        hb_dict_extract_int(&spatial_metric, dict, "spatial-metric");
        hb_dict_extract_int(&motion_threshold, dict, "motion-thresh");
        hb_dict_extract_int(&spatial_threshold, dict, "spatial-thresh");
        hb_dict_extract_int(&filter_mode, dict, "filter-mode");
        hb_dict_extract_int(&block_threshold, dict, "block-thresh");
        hb_dict_extract_int(&block_width, dict, "block-width");
        hb_dict_extract_int(&block_height, dict, "block-height");
    }
    if (mode & (MODE_MASK | MODE_COMPOSITE))
    {
        hb_error("comb_detect(cuda): debug modes 4/8 (mask painting) are not implemented on the GPU path");
        goto fail;
    }
    if (block_width > init->geometry.width)   block_width  = init->geometry.width;
    if (block_height > init->geometry.height) block_height = init->geometry.height;

    /* thresholds scale with depth (comb_detect.c:1152-1162) */
    motion_threshold  <<= (depth - 8);
    spatial_threshold <<= (depth - 8);
    cfg.gamma_motion_threshold   = (float)motion_threshold / (float)max_value;
    cfg.gamma_spatial_threshold  = (float)spatial_threshold / (float)max_value;
    cfg.gamma_spatial_threshold6 = 6 * cfg.gamma_spatial_threshold;
    cfg.comb32detect_min = depth >= 8 ? 10 << (depth - 8) : 10;
    cfg.comb32detect_max = depth >= 8 ? 15 << (depth - 8) : 15;

    /* gamma table: the numeric contract of the gamma path (comb_detect.c:1074-1081) */
    float *gamma_lut = malloc(sizeof(float) * (max_value + 1));
    if (gamma_lut == NULL)
    {
        hb_error("comb_detect(cuda): malloc failed");
        goto fail;
    }
    for (int i = 0; i < max_value + 1; i++)
    {
        gamma_lut[i] = pow(((float)i / (float)max_value), 2.2f);
    }

    cfg.width  = init->geometry.width;
    cfg.height = hb_image_height(init->pix_fmt, init->geometry.height, 0);
    cfg.depth  = depth;
    cfg.device = 0;
    const char *dev_env = getenv("HBCU_DEVICE");
    if (dev_env != NULL) cfg.device = atoi(dev_env);
    cfg.slots             = 6;
    cfg.mode              = mode;
    cfg.spatial_metric    = spatial_metric;
    cfg.filter_mode       = filter_mode;
    cfg.motion_threshold  = motion_threshold;
    cfg.spatial_threshold = spatial_threshold;
    cfg.block_threshold   = block_threshold;
    cfg.block_width       = block_width;
    cfg.block_height      = block_height;
    cfg.gamma_lut         = gamma_lut;
    const int rc = hbcu_comb_detect_create(&pv->gpu, &cfg);
    free(gamma_lut);
    if (rc != 0)
    {
        hb_error("comb_detect(cuda): %s", hbcu_last_error());
        goto fail;
    }
    pv->mode = mode;
    pv->force_exhaustive = 1;         /* comb_detect.c:1111 */
    pv->ref_index[0] = pv->ref_index[1] = pv->ref_index[2] = -1;
    return 0;

fail:
    free(pv);
    filter->private_data = NULL;
    return -1;
}

static void comb_detect_cuda_close(hb_filter_object_t *filter)
{
    hb_filter_private_t *pv = filter->private_data;
    if (pv == NULL) return;

    hb_log("comb detect: heavy %i | light %i | uncombed %i | total %i",
           pv->comb_heavy, pv->comb_light, pv->comb_none, pv->frames);

    if (pv->gpu != NULL) hbcu_comb_detect_destroy(pv->gpu);   /* waits for in-flight uploads */
    hb_buffer_list_close(&pv->out_list);
    for (int ii = 0; ii < 3; ii++)
    {
        if (!pv->ref_used[ii]) hb_buffer_close(&pv->ref[ii]);
    }
    free(pv);
    filter->private_data = NULL;
}

/* slide the window: drop prev (unless it travels in out_list), append b as next */
static void store_ref(hb_filter_private_t *pv, hb_buffer_t *b, int64_t index)
{
    if (!pv->ref_used[0]) hb_buffer_close(&pv->ref[0]);
    for (int k = 0; k < 2; k++)
    {
        pv->ref[k]       = pv->ref[k + 1];
        pv->ref_index[k] = pv->ref_index[k + 1];
        pv->ref_used[k]  = pv->ref_used[k + 1];
    }
    pv->ref[2]       = b;
    pv->ref_index[2] = index;
    pv->ref_used[2]  = 0;
}

static int upload_luma(hb_filter_private_t *pv, hb_buffer_t *b, int64_t index)
{
    /* the frame itself passes through untouched, host or device; only its luma is looked at */
    hbcu_frame_t *fin = hbcu_buffer_frame(b);
    if ((fin != NULL ? hbcu_comb_detect_upload_frame(pv->gpu, index, fin)
                     : hbcu_comb_detect_upload(pv->gpu, index, b->plane[0].data, b->plane[0].stride)) != 0)
    {
        hb_error("comb_detect(cuda): %s", hbcu_last_error());
        return -1;
    }
    return 0;
}

/* comb_segmenter + the bookkeeping of process_frame (comb_detect.c:1499-1535), asynchronous */
static int process_frame(hb_filter_private_t *pv)
{
    if (hbcu_comb_detect_run(pv->gpu, pv->ref_index[0], pv->ref_index[1], pv->ref_index[2], pv->force_exhaustive) != 0)
    {
        hb_error("comb_detect(cuda): %s", hbcu_last_error());
        return -1;
    }
    pv->ref_used[1] = 1;
    hb_buffer_list_append(&pv->out_list, pv->ref[1]);
    pv->out_index[pv->out_count]   = pv->ref_index[1];
    pv->out_pending[pv->out_count] = 1;
    pv->out_count++;
    pv->force_exhaustive = 0;
    return 0;
}

/* collect the verdict of the i-th queued frame and tag its buffer */
static int resolve(hb_filter_private_t *pv, int i, hb_buffer_t *buf)
{
    if (!pv->out_pending[i]) return 0;
    int combed = HB_COMB_NONE;
    if (hbcu_comb_detect_result(pv->gpu, pv->out_index[i], &combed) != 0)
    {
        hb_error("comb_detect(cuda): %s", hbcu_last_error());
        return -1;
    }
    buf->s.combed = combed;
    pv->out_pending[i] = 0;
    switch (combed)
    {
        case HB_COMB_HEAVY: pv->comb_heavy++; break;
        case HB_COMB_LIGHT: pv->comb_light++; break;
        default:            pv->comb_none++;  break;
    }
    pv->frames++;
    return 0;
}

static void pop_out_slot(hb_filter_private_t *pv)
{
    for (int i = 1; i < pv->out_count; i++)
    {
        pv->out_index[i - 1]   = pv->out_index[i];
        pv->out_pending[i - 1] = pv->out_pending[i];
    }
    pv->out_count--;
}

static int comb_detect_cuda_work(hb_filter_object_t *filter, hb_buffer_t **buf_in, hb_buffer_t **buf_out)
{
    hb_filter_private_t *pv = filter->private_data;
    hb_buffer_t *in = *buf_in;

    *buf_in = NULL;                               /* input is always consumed (comb_detect.c:1545) */
    if (in->s.flags & HB_BUF_FLAG_EOF)
    {
        int failed = 0;
        /* the last frame is its own successor; same pixels, so no second upload */
        store_ref(pv, hb_buffer_shallow_dup(pv->ref[2]), pv->ref_index[2]);
        if (pv->ref[0] != NULL)
        {
            pv->force_exhaustive = 1;
            if (process_frame(pv) != 0) failed = 1;
        }
        int i = 0;
        for (hb_buffer_t *b = hb_buffer_list_head(&pv->out_list); b != NULL && !failed; b = b->next, i++)
        {
            if (resolve(pv, i, b) != 0) failed = 1;
        }
        pv->out_count = 0;
        hb_buffer_list_append(&pv->out_list, in);
        *buf_out = hb_buffer_list_clear(&pv->out_list);
        return failed ? HB_FILTER_FAILED : HB_FILTER_DONE;
    }

    const int64_t index = pv->next_index++;
    if (upload_luma(pv, in, index) != 0)
    {
        hb_buffer_close(&in);
        return HB_FILTER_FAILED;
    }
    if (!pv->ready)
    {
        /* first frame: it is also its own predecessor (comb_detect.c:1562-1571) */
        store_ref(pv, hb_buffer_shallow_dup(in), index);
        store_ref(pv, in, index);
        pv->ready = 1;
        return HB_FILTER_DELAY;
    }

    store_ref(pv, in, index);
    if (process_frame(pv) != 0) return HB_FILTER_FAILED;

    /* a buffer may still be in the window; it leaves once more than three are queued */
    if (hb_buffer_list_count(&pv->out_list) > 3)
    {
        hb_buffer_t *head = hb_buffer_list_head(&pv->out_list);
        if (resolve(pv, 0, head) != 0) return HB_FILTER_FAILED;
        *buf_out = hb_buffer_list_rem_head(&pv->out_list);
        pop_out_slot(pv);
    }
    return HB_FILTER_OK;
}
