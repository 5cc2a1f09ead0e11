/* vfr_cuda.c -- hb_filter_vfr_cuda: drop-in for hb_filter_vfr (reference libhb/vfr.c), the framerate shaper, with the
 * motion metric it drops frames by (libhb/motion_metric.c) running on an H100 through include/hbcu.h.
 *
 * Same id, short name, settings template, defaults and init() changes as vfr.c, and the same timestamps, drops,
 * duplicates and output order for every input.  The filter never writes or copies a picture: every output is an input
 * buffer or an hb_buffer_shallow_dup of one (for a device frame, one more reference on the same frame).
 *
 * The control flow is vfr.c's, restated on fixed arrays (the delay queue holds at most 4 frames, the analysis list at
 * most MAX_FRAME_ANALYSIS_DEPTH), quirks included:
 *   - three frames wait in the delay queue; their times are renumbered through last_start / last_stop, input gaps are
 *     spread over four frames through lost_time (the remainder in slot 3), and an input whose stop is not past
 *     last_stop[0] is dropped and counted;
 *   - frame_metric[] is shifted by delete_metric(): after a pass, frame_metric[0] holds the stale metric of the new
 *     head, and that value takes part in the next minimum, exactly as in vfr.c;
 *   - find_drop_frame() has the shortcut exit, the analysis-duration cut-off and a strict < (the lowest index wins).
 *
 * Lazy metric read: each pair's metric is queued on the GPU when vfr.c computes it, but its value is read only when
 * find_drop_frame() gets past both of its early exits and compares metrics.  In the common peak-rate case (a source
 * below the peak) that never happens, so the filter adds no host wait to a device-resident chain; a constant-rate drop
 * decision waits once, for results already queued (newest first: its wait covers the older ones).
 *
 * Frames may be host or device buffers, per buffer.  Modes 1 and 2 need a device (hbcu_env_device()); without one
 * init() fails and libhb keeps hb_filter_vfr.  Mode 0 computes no metric and touches no device.
 */
#include <limits.h>
#include "libavutil/avutil.h"
#include "handbrake/handbrake.h"
#include "hbcu.h"
#include "hbcu_device_frames.h"

#define MAX_FRAME_ANALYSIS_DEPTH 10
#define DELAY_FRAMES             4
#define METRIC_SLOTS             (MAX_FRAME_ANALYSIS_DEPTH + 1)   /* the list's frames and the newest one */
#define METRIC_RESULTS           (MAX_FRAME_ANALYSIS_DEPTH + 2)

struct hb_filter_private_s
{
    hb_job_t      * job;
    int             cfr;
    hb_rational_t   input_vrate;
    hb_rational_t   vrate;
    hb_buffer_t   * delay[DELAY_FRAMES];      /* delay queue, oldest first */
    int             delay_count;
    int             dropped_frames;
    int             extended_frames;
    int64_t         last_start[4];
    int64_t         last_stop[4];
    int64_t         lost_time[4];
    int64_t         total_lost_time;
    int64_t         total_gained_time;
    int             count_frames;
    double          frame_duration;
    double          out_last_stop;
    int             drops;
    int             dups;

    int             frame_analysis_depth;
    int64_t         frame_analysis_duration;
    hb_buffer_t   * list[MAX_FRAME_ANALYSIS_DEPTH];      /* frame-rate list */
    int             list_slot[MAX_FRAME_ANALYSIS_DEPTH]; /* the metric slot holding each listed frame */
    int             count;
    double          frame_metric[MAX_FRAME_ANALYSIS_DEPTH];
    int             metric_result[MAX_FRAME_ANALYSIS_DEPTH];   /* result slot frame_metric[i] is still to be read from, or -1 */

    hbcu_motion_metric_t * gpu;
    int             width, height;            /* the init geometry every frame must have */
    int             metric_w, metric_h;       /* what the sum is divided by (reduced on the fast path) */
    int             failed;
};

static int                vfr_cuda_init(hb_filter_object_t *filter, hb_filter_init_t *init);
static int                vfr_cuda_work(hb_filter_object_t *filter, hb_buffer_t **buf_in, hb_buffer_t **buf_out);
static void               vfr_cuda_close(hb_filter_object_t *filter);
static hb_filter_info_t * vfr_cuda_info(hb_filter_object_t *filter);

static const char vfr_cuda_template[] = "mode=^([012])$:rate=^" HB_RATIONAL_REG "$";

hb_filter_object_t hb_filter_vfr_cuda =
{
    .id                = HB_FILTER_VFR,
    .enforce_order     = 1,
    .name              = "Framerate Shaper (CUDA sm_90a)",
    .short_name        = "vfr",
    .settings          = NULL,
    .init              = vfr_cuda_init,
    .work              = vfr_cuda_work,
    .close             = vfr_cuda_close,
    .info              = vfr_cuda_info,
    .settings_template = vfr_cuda_template,
};

/* motion_metric.c's init: the gamma table (with its max - 1 denominator), the fast path from the init geometry */
static int metric_init(hb_filter_private_t *pv, hb_filter_init_t *init)
{
    const AVPixFmtDescriptor *desc = av_pix_fmt_desc_get(init->pix_fmt);
    if (desc == NULL || desc->comp[0].depth < 8 || desc->comp[0].depth > 16)
    {
        hb_error("vfr(cuda): unsupported pixel format %d", init->pix_fmt);
        return -1;
    }
    /* P010 / P016 keep their samples in the high bits: the reference indexes its (1 << depth)-entry table with them
     * (motion_metric.c:240-251, 285-291), past its end for P010.  Above 8 bits a semi-planar frame is for mode 0 only;
     * NV12 is fine, the metric reads plane 0 */
    if (av_pix_fmt_count_planes(init->pix_fmt) == 2 && desc->comp[0].depth > 8)
    {
        hb_error("vfr(cuda): the motion metric does not take %s frames; only mode 0 (variable frame rate) does", desc->name);
        return -1;
    }
    const int depth = desc->comp[0].depth, max_value = (1 << depth) - 1;
    unsigned *lut = malloc(sizeof(unsigned) * (max_value + 1));
    if (lut == NULL)
    {
        hb_error("vfr(cuda): malloc failed");
        return -1;
    }
    for (int i = 0; i <= max_value; i++)
        lut[i] = 4095 * pow(((float)i / (float)(max_value - 1)), 2.2f);

    const int fast = init->geometry.width >= 1920 || init->geometry.height >= 1080;
    pv->width    = init->geometry.width;
    pv->height   = init->geometry.height;
    pv->metric_w = fast ? pv->width / 4 : pv->width;
    pv->metric_h = fast ? pv->height / 4 : pv->height;

    hbcu_motion_metric_config_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.width     = pv->width;
    cfg.height    = pv->height;
    cfg.depth     = depth;
    cfg.fast      = fast;
    cfg.device    = hbcu_env_device();
    cfg.slots     = METRIC_SLOTS;
    cfg.results   = METRIC_RESULTS;
    cfg.gamma_lut = lut;
    const int rc = hbcu_motion_metric_create(&pv->gpu, &cfg);
    free(lut);
    if (rc != 0)
    {
        hb_error("vfr(cuda): %s", hbcu_last_error());
        return -1;
    }
    return 0;
}

/* the newest listed frame, in metric slot `slot`; with a_slot >= 0 its metric against that slot goes to `result` */
static int metric_enqueue(hb_filter_private_t *pv, hb_buffer_t *b, int slot, int a_slot, int result)
{
    if (b->f.width != pv->width || b->f.height != pv->height)
    {
        hb_error("vfr(cuda): a %dx%d frame in a %dx%d job", b->f.width, b->f.height, pv->width, pv->height);
        return -1;
    }
    hbcu_frame_t *f = hbcu_buffer_frame(b);
    if (hbcu_motion_metric_enqueue(pv->gpu, slot, a_slot, result, f, f ? NULL : b->plane[0].data, b->plane[0].stride) != 0)
    {
        hb_error("vfr(cuda): %s", hbcu_last_error());
        return -1;
    }
    return 0;
}

/* frame_metric[i] as motion_metric.c returns it: (float)sum / (width * height) */
static int metric_read(hb_filter_private_t *pv, int i)
{
    const int r = pv->metric_result[i];
    if (r < 0)
        return 0;
    uint64_t sum;
    if (hbcu_motion_metric_result(pv->gpu, r, &sum) != 0)
    {
        hb_error("vfr(cuda): %s", hbcu_last_error());
        return -1;
    }
    const float metric = (float)sum / (pv->metric_w * pv->metric_h);
    /* delete_metric() may have left a copy of the entry past the list's end */
    for (int k = 0; k < MAX_FRAME_ANALYSIS_DEPTH; k++)
        if (pv->metric_result[k] == r)
        {
            pv->frame_metric[k]  = metric;
            pv->metric_result[k] = -1;
        }
    return 0;
}

static void delete_metric(hb_filter_private_t *pv, int pos, int size)
{
    memmove(&pv->frame_metric[pos], &pv->frame_metric[pos + 1], (size - (pos + 1)) * sizeof(double));
    memmove(&pv->metric_result[pos], &pv->metric_result[pos + 1], (size - (pos + 1)) * sizeof(int));
}

static hb_buffer_t *list_remove(hb_filter_private_t *pv, int i)
{
    hb_buffer_t *b = pv->list[i];
    memmove(&pv->list[i], &pv->list[i + 1], (pv->count - i - 1) * sizeof(pv->list[0]));
    memmove(&pv->list_slot[i], &pv->list_slot[i + 1], (pv->count - i - 1) * sizeof(int));
    pv->count--;
    return b;
}

/* appends `in` to the frame-rate list and queues the metric of the last two listed frames */
static int list_add(hb_filter_private_t *pv, hb_buffer_t *in)
{
    int slot = 0, result = -1;
    for (int used = 1; used; )
    {
        used = 0;
        for (int k = 0; k < pv->count; k++) used |= pv->list_slot[k] == slot;
        if (used) slot++;
    }
    pv->list[pv->count] = in;
    pv->list_slot[pv->count] = slot;
    pv->count++;
    if (pv->count >= 2)
    {
        for (int used = 1; used; )
        {
            result++;
            used = 0;
            for (int k = 0; k < MAX_FRAME_ANALYSIS_DEPTH; k++) used |= pv->metric_result[k] == result;
        }
        pv->metric_result[pv->count - 1] = result;
    }
    return metric_enqueue(pv, in, slot, pv->count >= 2 ? pv->list_slot[pv->count - 2] : -1, result);
}

/* vfr.c find_drop_frame(), with the metrics read only once they decide: -1 no drop, -2 failure */
static int find_drop_frame(hb_filter_private_t *pv, int count)
{
    int ii, min;
    double cfr_stop;

    cfr_stop = pv->out_last_stop + pv->frame_duration * (count - 1);
    if (pv->list[count - 1]->s.stop >= (int64_t)cfr_stop)
        return -1;

    const hb_buffer_t *first = pv->list[0];
    for (ii = 1; ii < count; ii++)
        if (pv->list[ii]->s.stop - first->s.start > pv->frame_analysis_duration)
            break;

    cfr_stop = pv->out_last_stop + pv->frame_duration * (ii - 1);
    if (pv->list[ii - 1]->s.stop >= (int64_t)cfr_stop)
        return -1;

    for (int k = ii - 1; k >= 0; k--)
        if (metric_read(pv, k) != 0)
            return -2;
    min = 0;
    for (int k = 1; k < ii; k++)
        if (pv->frame_metric[k] < pv->frame_metric[min])
            min = k;
    return min;
}

/* vfr.c adjust_frame_rate(): modes 0 (pass through), 1 (CFR) and 2 (PFR); in == NULL flushes the list */
static hb_buffer_t *adjust_frame_rate(hb_filter_private_t *pv, hb_buffer_t *in)
{
    if (pv->cfr == 0)
    {
        if (in)
        {
            ++pv->count_frames;
            pv->out_last_stop = in->s.stop;
        }
        return in;
    }

    int count;
    if (in != NULL)
    {
        if (pv->out_last_stop == (int64_t)AV_NOPTS_VALUE)
            pv->out_last_stop = in->s.start;
        if (list_add(pv, in) != 0)
        {
            pv->failed = 1;
            return NULL;
        }
        count = pv->count;
        if (count < 2 || count < pv->frame_analysis_depth)
            return NULL;
    }
    else
    {
        count = pv->count;
    }

    hb_buffer_list_t list;
    hb_buffer_t     *out;
    double           cfr_stop;

    hb_buffer_list_clear(&list);

    const int drop_frame = find_drop_frame(pv, count);
    if (drop_frame == -2)
    {
        pv->failed = 1;
        return NULL;
    }
    if (drop_frame >= 0)
    {
        /* the frame that appears to have the least motion */
        out = list_remove(pv, drop_frame);
        hb_buffer_close(&out);
        delete_metric(pv, drop_frame, count);
        ++pv->drops;
        return NULL;
    }

    out = list_remove(pv, 0);
    hb_buffer_list_append(&list, out);
    delete_metric(pv, 0, count);

    out->s.start = pv->out_last_stop;
    cfr_stop = pv->out_last_stop + pv->frame_duration;

    ++pv->count_frames;
    if (pv->cfr > 1)
    {
        /* PFR: keep the frame, extend it to the average-rate bound */
        if (out->s.stop < cfr_stop)
        {
            out->s.stop = pv->out_last_stop = cfr_stop;
        }
        else
        {
            pv->out_last_stop = out->s.stop;
        }
    }
    else
    {
        /* CFR: one frame duration each, the excess as shallow duplicates */
        double excess = (double)out->s.stop - cfr_stop;
        out->s.stop = pv->out_last_stop = cfr_stop;
        for (; excess >= pv->frame_duration; excess -= pv->frame_duration)
        {
            hb_buffer_t *dup = hb_buffer_shallow_dup(out);
            if (dup == NULL)
            {
                hb_error("vfr(cuda): out of memory");
                pv->failed = 1;
                break;
            }
            dup->s.new_chap = 0;
            dup->s.start = cfr_stop;
            cfr_stop += pv->frame_duration;
            dup->s.stop = pv->out_last_stop = cfr_stop;
            hb_buffer_list_append(&list, dup);
            ++pv->dups;
            ++pv->count_frames;
        }
    }

    return hb_buffer_list_clear(&list);
}

static hb_buffer_t *flush_frames(hb_filter_private_t *pv)
{
    hb_buffer_list_t list;

    hb_buffer_list_clear(&list);
    while (pv->count > 0 && !pv->failed)
        hb_buffer_list_append(&list, adjust_frame_rate(pv, NULL));
    return hb_buffer_list_clear(&list);
}

static hb_buffer_t *delay_get(hb_filter_private_t *pv)
{
    if (pv->delay_count == 0)
        return NULL;
    hb_buffer_t *b = pv->delay[0];
    memmove(&pv->delay[0], &pv->delay[1], (pv->delay_count - 1) * sizeof(pv->delay[0]));
    pv->delay_count--;
    return b;
}

static int vfr_cuda_init(hb_filter_object_t *filter, hb_filter_init_t *init)
{
    hb_filter_private_t *pv = calloc(1, sizeof(struct hb_filter_private_s));
    filter->private_data = pv;
    if (pv == NULL)
    {
        hb_error("vfr(cuda): calloc failed");
        return -1;
    }

    pv->cfr         = init->cfr;
    pv->input_vrate = pv->vrate = init->vrate;
    hb_dict_extract_int(&pv->cfr, filter->settings, "mode");
    hb_dict_extract_rational(&pv->vrate, filter->settings, "rate");

    if (pv->cfr && metric_init(pv, init) != 0)
    {
        free(pv);
        filter->private_data = NULL;
        return -1;
    }

    /* frame-drop analysis always looks at least 2 buffers */
    pv->frame_analysis_depth = 2;
    double in_vrate  = (double)pv->input_vrate.num / pv->input_vrate.den;
    double out_vrate = (double)pv->vrate.num / pv->vrate.den;
    if (in_vrate > out_vrate)
    {
        /* repeats to expect per kept frame (or kept frames per repeat below a factor of 2), plus one */
        double factor = in_vrate / out_vrate;
        if (factor > 1.0 && factor < 2.0)
        {
            factor = 1 / (factor - 1);
        }
        pv->frame_analysis_depth = ceil(factor) + 1;
        if (pv->frame_analysis_depth > MAX_FRAME_ANALYSIS_DEPTH)
        {
            pv->frame_analysis_depth = MAX_FRAME_ANALYSIS_DEPTH;
        }
    }
    pv->frame_analysis_duration = pv->frame_analysis_depth * 90000 / in_vrate;
    pv->frame_metric[0] = INT_MAX;
    for (int i = 0; i < MAX_FRAME_ANALYSIS_DEPTH; i++)
        pv->metric_result[i] = -1;

    pv->job = init->job;

    if (pv->cfr == 2)
    {
        /* PFR: the source's rate unless it is above the peak */
        double source_fps = (double)init->vrate.num / init->vrate.den;
        double peak_fps = (double)pv->vrate.num / pv->vrate.den;
        if (source_fps > peak_fps)
        {
            init->vrate = pv->vrate;
        }
    }
    else
    {
        init->vrate = pv->vrate;
    }
    pv->frame_duration = (double)pv->vrate.den * 90000. / pv->vrate.num;
    pv->out_last_stop  = (int64_t)AV_NOPTS_VALUE;
    init->cfr          = pv->cfr;

    return 0;
}

static hb_filter_info_t *vfr_cuda_info(hb_filter_object_t *filter)
{
    hb_filter_private_t *pv = filter->private_data;
    hb_filter_info_t    *info;

    if (!pv)
        return NULL;

    info = calloc(1, sizeof(hb_filter_info_t));
    if (info == NULL)
        return NULL;
    info->human_readable_desc = malloc(128);
    if (info->human_readable_desc == NULL)
    {
        free(info);
        return NULL;
    }
    info->human_readable_desc[0] = 0;

    double source_fps = (double)pv->input_vrate.num / pv->input_vrate.den;
    double rate_fps   = (double)pv->vrate.num / pv->vrate.den;
    info->output.vrate = pv->input_vrate;
    if (pv->cfr == 2)
    {
        if (source_fps > rate_fps)
        {
            info->output.vrate = pv->vrate;
        }
    }
    else
    {
        info->output.vrate = pv->vrate;
    }
    info->output.cfr = pv->cfr;
    if (pv->cfr == 0)
    {
        snprintf(info->human_readable_desc, 128, "frame rate: same as source (around %.3f fps)",
                 (float)pv->vrate.num / pv->vrate.den);
    }
    else if (pv->cfr == 2)
    {
        snprintf(info->human_readable_desc, 128, "frame rate: %.3f fps -> peak rate limited to %.3f fps",
                 source_fps, rate_fps);
    }
    else
    {
        snprintf(info->human_readable_desc, 128, "frame rate: %.3f fps -> constant %.3f fps",
                 source_fps, rate_fps);
    }
    return info;
}

static void vfr_cuda_close(hb_filter_object_t *filter)
{
    hb_filter_private_t *pv = filter->private_data;

    if (!pv)
        return;

    if (pv->cfr)
    {
        hb_log("vfr: %d frames output, %d dropped and %d duped for CFR/PFR",
               pv->count_frames, pv->drops, pv->dups);
    }
    else
    {
        hb_log("vfr: %d frames output, %d dropped",
               pv->count_frames, pv->drops);
    }

    if (pv->job)
    {
        hb_interjob_t *interjob = hb_interjob_get(pv->job->h);

        /* the dropped-frame count makes a second pass's frame rate more accurate */
        interjob->out_frame_count = pv->count_frames;
        interjob->total_time = pv->out_last_stop;
    }

    hb_log("vfr: lost time: %"PRId64" (%i frames)",
           pv->total_lost_time, pv->dropped_frames);
    hb_log("vfr: gained time: %"PRId64" (%i frames) (%"PRId64" not accounted for)",
           pv->total_gained_time, pv->extended_frames,
           pv->total_lost_time - pv->total_gained_time);

    if (pv->dropped_frames)
    {
        hb_log("vfr: average dropped frame duration: %"PRId64,
               (pv->total_lost_time / pv->dropped_frames));
    }

    hb_buffer_t *b;
    while ((b = delay_get(pv)) != NULL)
        hb_buffer_close(&b);
    while (pv->count > 0)
    {
        b = list_remove(pv, 0);
        hb_buffer_close(&b);
    }
    hbcu_motion_metric_destroy(pv->gpu);      /* waits for the work in flight, drops its frame references */

    free(pv);
    filter->private_data = NULL;
}

static int vfr_cuda_work(hb_filter_object_t *filter, hb_buffer_t **buf_in, hb_buffer_t **buf_out)
{
    hb_filter_private_t *pv  = filter->private_data;
    hb_buffer_t         *in  = *buf_in;
    hb_buffer_t         *out = NULL;

    *buf_in = NULL;
    *buf_out = NULL;

    if (in->s.flags & HB_BUF_FLAG_EOF)
    {
        hb_buffer_list_t list;
        hb_buffer_t     *next;
        int              counter = 2;

        /* the queued frames take their renumbered times from the arrays */
        hb_buffer_list_clear(&list);
        while ((next = delay_get(pv)) != NULL)
        {
            next->s.start = pv->last_start[counter];
            next->s.stop  = pv->last_stop[counter--];
            hb_buffer_list_append(&list, adjust_frame_rate(pv, next));
        }
        hb_buffer_list_append(&list, flush_frames(pv));
        hb_buffer_list_append(&list, in);
        *buf_out = hb_buffer_list_clear(&list);
        return pv->failed ? HB_FILTER_FAILED : HB_FILTER_DONE;
    }

    /* a gap between the last stop and this start: frames were dropped upstream; spread the lost time in quarters */
    if (pv->delay_count > 0 && in->s.start > pv->last_stop[0])
    {
        int64_t temp_duration = in->s.start - pv->last_stop[0];
        pv->lost_time[0] += (temp_duration / 4);
        pv->lost_time[1] += (temp_duration / 4);
        pv->lost_time[2] += (temp_duration / 4);
        pv->lost_time[3] += (temp_duration - 3 * (temp_duration / 4));

        pv->total_lost_time += temp_duration;
    }
    else if (in->s.stop <= pv->last_stop[0])
    {
        /* a frame that does not end after the previous one (bad source): dropped */
        ++pv->drops;
        hb_buffer_close(&in);
        return HB_FILTER_OK;
    }

    int i;
    for (i = 3; i >= 1; i--)
    {
        pv->last_start[i] = pv->last_start[i - 1];
        pv->last_stop[i]  = pv->last_stop[i - 1];
    }

    /* continuous time stamps: this frame starts where the previous one stopped */
    if (pv->delay_count == 0)
    {
        pv->last_start[0] = in->s.start;
        pv->last_stop[0]  = in->s.stop;
    }
    else
    {
        pv->last_start[0] = pv->last_stop[1];
        pv->last_stop[0]  = pv->last_start[0] + (in->s.stop - in->s.start);
    }

    pv->delay[pv->delay_count++] = in;

    /* three frames stay queued, so the durations of the last two can still be rewritten */
    if (pv->delay_count < DELAY_FRAMES)
        return HB_FILTER_OK;

    out = delay_get(pv);
    if (pv->lost_time[3] > 0)
    {
        int time_shift = 0;

        /* make up lost time: extend the four cached durations, keeping them contiguous */
        for (i = 3; i >= 0; i--)
        {
            pv->last_start[i] += time_shift;
            pv->last_stop[i] += pv->lost_time[i] + time_shift;

            pv->total_gained_time += pv->lost_time[i];
            time_shift += pv->lost_time[i];

            pv->lost_time[i] = 0;

            pv->extended_frames++;
        }
    }

    out->s.start = pv->last_start[3];
    out->s.stop  = pv->last_stop[3];

    *buf_out = adjust_frame_rate(pv, out);

    return pv->failed ? HB_FILTER_FAILED : HB_FILTER_OK;
}
