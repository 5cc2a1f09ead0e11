/* nlmeans_cuda.c -- hb_filter_nlmeans_cuda: drop-in for hb_filter_nlmeans
 * (reference libhb/nlmeans.c:202-213) whose per-pixel work runs on an H100
 * through the C-ABI in include/hbcu.h.  Host side stays C, as in libhb.
 *
 * Same plugin surface as the reference: same settings_template and keys, same
 * cascade / defaults / sanitising of the 19 settings (nlmeans.c:279-343), the
 * same exp table (nlmeans.c:346-358, computed here on the host with the very
 * same C expressions and uploaded, never recomputed on the device), same
 * look-AHEAD temporal window (output t uses inputs t .. t+nframes-1), same
 * shrinking window at EOF (nlmeans.c:636-640), same output order and props.
 *
 * What changes: the taskset of `threads` CPU workers (nlmeans.c:546-597)
 * becomes CUDA stream dispatch -- frame t is enqueued as soon as frame
 * t+max_frames-1 has been uploaded, up to `depth` outputs are in flight, and
 * finished frames are handed downstream in order.  Burst sizes therefore
 * differ from the reference (which emits `threads` frames at a time); output
 * order and content do not.  The `threads` setting is accepted and sizes the
 * number of frames kept in flight.  The prefilter modes (nlmeans.c:72-83) run on
 * the GPU too, with the reference's single-worker behaviour (SURVEY.md 8a a5).
 *
 * Several GPUs (setting `devices=0,1,..` or HBCU_DEVICES): the same one ordered
 * input stream is dealt block-cyclically -- `block` consecutive frames per device
 * in turn -- the way mt_frame_filter.c:169-237 deals frames to CPU threads, and
 * harvested in stream order.  A block's look-ahead window reaches nframes-1
 * frames into the next block: those frames cross PCIe once (to their owner) and
 * reach the previous block's device by an NVLink peer copy
 * (hbcu_nlmeans_upload_peer).  Every device keeps its own contiguous index space,
 * and -- like the reference's taskset, one thread per worker (nlmeans.c:546-597) --
 * its own submission thread: work() only queues commands (upload, halo copy,
 * filter) and the device's thread turns them into CUDA calls, so the stream
 * submission of G GPUs does not serialise on the filter's one thread.
 */
#include "handbrake/handbrake.h"
#include "hbcu.h"
#include "hbcu_device_frames.h"

#define NLMEANS_STRENGTH_DEFAULT    6
#define NLMEANS_ORIGIN_TUNE_DEFAULT 1
#define NLMEANS_PATCH_SIZE_DEFAULT  7
#define NLMEANS_RANGE_DEFAULT       3
#define NLMEANS_FRAMES_DEFAULT      2
#define NLMEANS_PREFILTER_DEFAULT   0
#define NLMEANS_FRAMES_MAX          32
#define NLMEANS_EXPSIZE             HBCU_NLMEANS_EXPSIZE

#define NLM_MAX_INFLIGHT 16
#define NLM_MAX_DEVICES  HBCU_MAX_DEVICES
#define NLM_BLOCK_DEFAULT 8

typedef struct
{
    int64_t      index;   /* position in the stream */
    int          dev;     /* which of pv->gpu[] owns the frame */
    int64_t      li;      /* its index in that device's own index space */
    hb_buffer_t *in;      /* input buffer we took ownership of (source of the async upload) */
    hb_buffer_t *out;     /* output buffer, NULL until the frame has been enqueued */
    volatile int uploaded;   /* multi-device: the owner's thread has issued the upload (a halo copy may read it) */
    volatile int submitted;  /* multi-device: the owner's thread has issued kernels + download (wait / poll are valid) */
} nlm_pending_t;

/* commands of a device's submission thread (multi-device only) */
enum { NLM_CMD_UPLOAD, NLM_CMD_PEER, NLM_CMD_FILTER, NLM_CMD_STOP };
typedef struct
{
    int            kind;
    int64_t        li;              /* index in this device's index space */
    nlm_pending_t *p;               /* UPLOAD / FILTER: the frame */
    int            navail;          /* FILTER */
    int            src_dev;         /* PEER: halo source */
    int64_t        src_li;
    nlm_pending_t *src_p;           /* PEER: wait until its upload has been issued */
} nlm_cmd_t;

typedef struct
{
    struct hb_filter_private_s *pv;
    int          dev;
    hb_thread_t *thread;
    hb_lock_t   *lock;
    hb_cond_t   *cv;                /* queue not empty */
    nlm_cmd_t   *q;
    int          cap, head, count;
} nlm_worker_t;


struct hb_filter_private_s
{
    int device, device_out;        /* device_out: outputs leave as HBCU_DEVICE buffers (hw_pix_fmt == AV_PIX_FMT_CUDA) */
    int depth;
    int bps;

    int    prefilter[3];
    int    threads;
    int    max_frames;

    int             ndev;                          /* devices the stream is dealt to (1: everything on `device`) */
    int             devices[NLM_MAX_DEVICES];      /* CUDA ordinals; an ordinal may repeat (two handles on one GPU) */
    hbcu_nlmeans_t *gpu[NLM_MAX_DEVICES];
    int64_t         local_next[NLM_MAX_DEVICES];   /* frames handed to each device so far = its next local index */
    int             dev_inflight[NLM_MAX_DEVICES]; /* outputs enqueued on the device and not yet emitted */
    int             block;                         /* frames per block of the block-cyclic dealing */
    nlm_worker_t    worker[NLM_MAX_DEVICES];       /* multi-device: one submission thread per device */
    hb_lock_t      *done_lock;                     /* guards `submitted` transitions seen by harvest() and `errmsg` */
    hb_cond_t      *done_cv;
    volatile int    failed;                        /* a submission thread hit a GPU error */
    char            errmsg[256];
    int             inflight_max;   /* outputs in flight per device */
    int             ring;

    /* frames received but not yet emitted, oldest first: [head, head+count) modulo cap */
    nlm_pending_t  *pending;
    int             cap, head, count;
    int64_t         next_in;        /* index of the next input frame  */
    int64_t         next_enqueue;   /* next frame to hand to the GPU */

    hb_filter_init_t input;
    hb_filter_init_t output;
};

static int  nlmeans_cuda_init(hb_filter_object_t *filter, hb_filter_init_t *init);
static int  nlmeans_cuda_work(hb_filter_object_t *filter, hb_buffer_t **buf_in, hb_buffer_t **buf_out);
static void nlmeans_cuda_close(hb_filter_object_t *filter);

static const char nlmeans_template[] =
    "y-strength=^"HB_FLOAT_REG"$:y-origin-tune=^"HB_FLOAT_REG"$:"
    "y-patch-size=^"HB_INT_REG"$:y-range=^"HB_INT_REG"$:"
    "y-frame-count=^"HB_INT_REG"$:y-prefilter=^"HB_INT_REG"$:"
    "cb-strength=^"HB_FLOAT_REG"$:cb-origin-tune=^"HB_FLOAT_REG"$:"
    "cb-patch-size=^"HB_INT_REG"$:cb-range=^"HB_INT_REG"$:"
    "cb-frame-count=^"HB_INT_REG"$:cb-prefilter=^"HB_INT_REG"$:"
    "cr-strength=^"HB_FLOAT_REG"$:cr-origin-tune=^"HB_FLOAT_REG"$:"
    "cr-patch-size=^"HB_INT_REG"$:cr-range=^"HB_INT_REG"$:"
    "cr-frame-count=^"HB_INT_REG"$:cr-prefilter=^"HB_INT_REG"$:"
    "threads=^"HB_INT_REG"$";

hb_filter_object_t hb_filter_nlmeans_cuda =
{
    .id                = HB_FILTER_NLMEANS,
    .enforce_order     = 1,
    .name              = "Denoise (nlmeans, CUDA sm_90a)",
    .short_name        = "nlmeans",
    .settings          = NULL,
    .init              = nlmeans_cuda_init,
    .work              = nlmeans_cuda_work,
    .close             = nlmeans_cuda_close,
    .settings_template = nlmeans_template,
};

static nlm_pending_t *pending_at(hb_filter_private_t *pv, int i)
{
    return &pv->pending[(pv->head + i) % pv->cap];
}

/* settings dict -> device configuration (nlmeans.c:279-358).  Exported so that bench.py
 * builds its kernel-only handle from exactly the code path init() uses. */
int hb_nlmeans_cuda_build_config(const hb_dict_t *dict, int pix_fmt, int width, int height,
                                 hbcu_nlmeans_config_t *cfg, int *max_frames_out, int *threads_out,
                                 int prefilter_out[3])
{
    static const char *const prefix[3] = { "y", "cb", "cr" };
    double strength[3], origin_tune[3];
    int patch_size[3], range[3], nframes[3], prefilter[3];
    int threads = -1, max_frames = 0;

    const AVPixFmtDescriptor *desc = av_pix_fmt_desc_get(pix_fmt);
    if (desc == NULL || desc->nb_components < 3)
    {
        hb_error("nlmeans(cuda): unsupported pixel format %d", pix_fmt);
        return -1;
    }
    const int depth = desc->comp[0].depth;

    for (int c = 0; c < 3; c++)
    {
        strength[c] = origin_tune[c] = -1;
        patch_size[c] = range[c] = nframes[c] = prefilter[c] = -1;
    }
    if (dict != NULL)
    {
        char key[32];
        for (int c = 0; c < 3; c++)
        {
            snprintf(key, sizeof(key), "%s-strength", prefix[c]);    hb_dict_extract_double(&strength[c], dict, key);
            snprintf(key, sizeof(key), "%s-origin-tune", prefix[c]); hb_dict_extract_double(&origin_tune[c], dict, key);
            snprintf(key, sizeof(key), "%s-patch-size", prefix[c]);  hb_dict_extract_int(&patch_size[c], dict, key);
            snprintf(key, sizeof(key), "%s-range", prefix[c]);       hb_dict_extract_int(&range[c], dict, key);
            snprintf(key, sizeof(key), "%s-frame-count", prefix[c]); hb_dict_extract_int(&nframes[c], dict, key);
            snprintf(key, sizeof(key), "%s-prefilter", prefix[c]);   hb_dict_extract_int(&prefilter[c], dict, key);
        }
        hb_dict_extract_int(&threads, dict, "threads");
    }

    /* Cr inherits Cb, Cb inherits Y, Y takes the defaults (nlmeans.c:306-326) */
    for (int c = 1; c < 3; c++)
    {
        if (strength[c]    == -1) strength[c]    = strength[c-1];
        if (origin_tune[c] == -1) origin_tune[c] = origin_tune[c-1];
        if (patch_size[c]  == -1) patch_size[c]  = patch_size[c-1];
        if (range[c]       == -1) range[c]       = range[c-1];
        if (nframes[c]     == -1) nframes[c]     = nframes[c-1];
        if (prefilter[c]   == -1) prefilter[c]   = prefilter[c-1];
    }

    memset(cfg, 0, sizeof(*cfg));
    for (int c = 0; c < 3; c++)
    {
        if (strength[c]    == -1) strength[c]    = NLMEANS_STRENGTH_DEFAULT;
        if (origin_tune[c] == -1) origin_tune[c] = NLMEANS_ORIGIN_TUNE_DEFAULT;
        if (patch_size[c]  == -1) patch_size[c]  = NLMEANS_PATCH_SIZE_DEFAULT;
        if (range[c]       == -1) range[c]       = NLMEANS_RANGE_DEFAULT;
        if (nframes[c]     == -1) nframes[c]     = NLMEANS_FRAMES_DEFAULT;
        if (prefilter[c]   == -1) prefilter[c]   = NLMEANS_PREFILTER_DEFAULT;

        /* sanitise (nlmeans.c:328-338) */
        if (strength[c] < 0)        strength[c] = 0;
        if (origin_tune[c] < 0.01)  origin_tune[c] = 0.01;
        if (origin_tune[c] > 1)     origin_tune[c] = 1;
        if (patch_size[c] % 2 == 0) patch_size[c]--;
        if (patch_size[c] < 1)      patch_size[c] = 1;
        if (range[c] % 2 == 0)      range[c]--;
        if (range[c] < 1)           range[c] = 1;
        if (nframes[c] < 1)         nframes[c] = 1;
        if (nframes[c] > NLMEANS_FRAMES_MAX) nframes[c] = NLMEANS_FRAMES_MAX;
        if (prefilter[c] < 0)       prefilter[c] = 0;

        if (max_frames < nframes[c]) max_frames = nframes[c];

        /* strength scales with bit depth (nlmeans.c:343) */
        strength[c] *= depth > 8 ? (depth - 8) * (depth - 8) : 1;

        /* exp table: these expressions are the numeric contract (nlmeans.c:346-358);
         * evaluated on the host exactly as written there */
        hbcu_nlmeans_plane_t *pp = &cfg->plane[c];
        const float weight_factor        = 1.0/patch_size[c]/patch_size[c] / (strength[c] * strength[c]);
        const float min_weight_in_table  = 0.0005;
        const float stretch              = NLMEANS_EXPSIZE / (-log(min_weight_in_table));
        pp->weight_fact                  = weight_factor * stretch;
        pp->diff_max                     = NLMEANS_EXPSIZE / pp->weight_fact;
        for (int i = 0; i < NLMEANS_EXPSIZE; i++)
        {
            pp->exptable[i] = exp(-i/stretch);
        }
        pp->exptable[NLMEANS_EXPSIZE-1] = 0;

        pp->patch_size  = patch_size[c];
        pp->range       = range[c];
        pp->nframes     = nframes[c];
        pp->origin_tune = origin_tune[c];
        pp->bypass      = strength[c] == 0;   /* nlmeans.c:493-499 */
        pp->prefilter   = prefilter[c];
        if (prefilter_out) prefilter_out[c] = prefilter[c];
    }
    cfg->width          = width;
    cfg->height         = height;
    cfg->depth          = depth;
    cfg->chroma_shift_w = desc->log2_chroma_w;
    cfg->chroma_shift_h = desc->log2_chroma_h;
    cfg->device         = 0;
    const char *dev_env = getenv("HBCU_DEVICE");
    if (dev_env != NULL) cfg->device = atoi(dev_env);
    if (max_frames_out) *max_frames_out = max_frames;
    if (threads_out) *threads_out = threads;
    return 0;
}

/* ------------------------------------------------------------------ */
/* per-device submission threads (multi-device only)                      */
/* ------------------------------------------------------------------ */
static void worker_fail(hb_filter_private_t *pv, const char *what)
{
    hb_lock(pv->done_lock);
    if (!pv->failed) snprintf(pv->errmsg, sizeof(pv->errmsg), "%s: %s", what, hbcu_last_error());    /* the error string is per thread */
    pv->failed = 1;
    hb_cond_broadcast(pv->done_cv);
    hb_unlock(pv->done_lock);
}

static void worker_push(nlm_worker_t *w, const nlm_cmd_t *cmd)
{
    hb_lock(w->lock);
    /* cannot overflow: the queue holds three commands per pending frame and is sized for it */
    w->q[(w->head + w->count) % w->cap] = *cmd;
    w->count++;
    hb_cond_signal(w->cv);
    hb_unlock(w->lock);
}

static void worker_main(void *arg)
{
    nlm_worker_t *w = arg;
    hb_filter_private_t *pv = w->pv;
    hbcu_nlmeans_t *gpu = pv->gpu[w->dev];
    for (;;)
    {
        hb_lock(w->lock);
        while (w->count == 0) hb_cond_wait(w->cv, w->lock);
        const nlm_cmd_t c = w->q[w->head];
        w->head = (w->head + 1) % w->cap;
        w->count--;
        hb_unlock(w->lock);
        if (c.kind == NLM_CMD_STOP) return;
        switch (c.kind)
        {
            case NLM_CMD_UPLOAD:
            {
                const void *planes[3];
                int strides[3];
                for (int k = 0; k < 3; k++)
                {
                    planes[k]  = c.p->in->plane[k].data;
                    strides[k] = c.p->in->plane[k].stride;
                }
                if (!pv->failed && hbcu_nlmeans_upload(gpu, c.li, planes, strides) != 0) worker_fail(pv, "upload");
                __atomic_store_n(&c.p->uploaded, 1, __ATOMIC_RELEASE);
                break;
            }
            case NLM_CMD_PEER:
                /* the halo's owner must have ISSUED its upload (its event is what the copy orders itself behind) */
                while (!__atomic_load_n(&c.src_p->uploaded, __ATOMIC_ACQUIRE) && !pv->failed) hb_yield();
                if (!pv->failed && hbcu_nlmeans_upload_peer(gpu, c.li, pv->gpu[c.src_dev], c.src_li) != 0) worker_fail(pv, "halo copy");
                break;
            case NLM_CMD_FILTER:
            {
                void *planes[3];
                int   strides[3];
                for (int k = 0; k < 3; k++)
                {
                    planes[k]  = c.p->out->plane[k].data;
                    strides[k] = c.p->out->plane[k].stride;
                }
                if (!pv->failed && hbcu_nlmeans_filter(gpu, c.li, c.navail, planes, strides) != 0) worker_fail(pv, "filter");
                hb_lock(pv->done_lock);
                c.p->submitted = 1;
                hb_cond_broadcast(pv->done_cv);
                hb_unlock(pv->done_lock);
                break;
            }
        }
    }
}

static int workers_start(hb_filter_private_t *pv)
{
    pv->done_lock = hb_lock_init();
    pv->done_cv   = hb_cond_init();
    if (pv->done_lock == NULL || pv->done_cv == NULL) return -1;
    for (int d = 0; d < pv->ndev; d++)
    {
        nlm_worker_t *w = &pv->worker[d];
        w->pv   = pv;
        w->dev  = d;
        w->cap  = 3 * pv->cap + 4;
        w->q    = calloc(w->cap, sizeof(*w->q));
        w->lock = hb_lock_init();
        w->cv   = hb_cond_init();
        if (w->q == NULL || w->lock == NULL || w->cv == NULL) return -1;
        w->thread = hb_thread_init("nlmeans-cuda-device", worker_main, w, HB_NORMAL_PRIORITY);
        if (w->thread == NULL) return -1;
    }
    return 0;
}

static void workers_stop(hb_filter_private_t *pv)
{
    for (int d = 0; d < pv->ndev; d++)
    {
        nlm_worker_t *w = &pv->worker[d];
        if (w->thread != NULL)
        {
            nlm_cmd_t stop;
            memset(&stop, 0, sizeof(stop));
            stop.kind = NLM_CMD_STOP;
            worker_push(w, &stop);
            hb_thread_close(&w->thread);         /* joins */
        }
        if (w->lock != NULL) hb_lock_close(&w->lock);
        if (w->cv != NULL) hb_cond_close(&w->cv);
        free(w->q);
        w->q = NULL;
    }
    if (pv->done_lock != NULL) hb_lock_close(&pv->done_lock);
    if (pv->done_cv != NULL) hb_cond_close(&pv->done_cv);
}

static int nlmeans_cuda_init(hb_filter_object_t *filter, hb_filter_init_t *init)
{
    hb_filter_private_t *pv = calloc(1, sizeof(*pv));
    if (pv == NULL)
    {
        hb_error("nlmeans(cuda): calloc failed");
        return -1;
    }
    filter->private_data = pv;
    pv->input = *init;

    hbcu_nlmeans_config_t cfg;
    if (hb_nlmeans_cuda_build_config(filter->settings, init->pix_fmt, init->geometry.width, init->geometry.height,
                                     &cfg, &pv->max_frames, &pv->threads, pv->prefilter) != 0)
    {
        goto fail;
    }
    pv->depth = cfg.depth;
    pv->bps   = pv->depth > 8 ? 2 : 1;

    /* the devices the stream is dealt to: setting `devices` (not part of the reference's template: a front end that
     * validates settings exposes it by appending the key, INTEGRATION.md), else HBCU_DEVICES, else the one device */
    pv->block = NLM_BLOCK_DEFAULT;
    if (filter->settings != NULL) hb_dict_extract_int(&pv->block, filter->settings, "block");
    pv->ndev = hbcu_settings_devices(filter->settings, pv->devices);       /* `devices` setting, HBCU_DEVICES, or the one device */
    if (pv->ndev < 1)
    {
        hb_error("nlmeans(cuda): bad `devices` setting");
        goto fail;
    }
    if (getenv("HBCU_BLOCK") != NULL && pv->block == NLM_BLOCK_DEFAULT) pv->block = atoi(getenv("HBCU_BLOCK"));
    /* a block's look-ahead window must end inside the NEXT block */
    if (pv->block < pv->max_frames - 1) pv->block = pv->max_frames - 1;
    if (pv->block < 1) pv->block = 1;

    pv->device_out = hbcu_init_wants_device_output(init);
    if (pv->ndev > 1 && pv->device_out)
    {
        hb_error("nlmeans(cuda): device-resident output needs a single device (devices=%d given)", pv->ndev);
        goto fail;
    }

    /* `threads` CPU workers -> that many output frames in flight on the streams (per device) */
    pv->inflight_max = pv->threads < 1 ? 4 : pv->threads;
    if (pv->ndev > 1 && pv->inflight_max < pv->block + 2) pv->inflight_max = pv->block + 2;    /* a whole block and the start of the next */
    if (pv->inflight_max > NLM_MAX_INFLIGHT) pv->inflight_max = NLM_MAX_INFLIGHT;
    /* Local indices of the outputs in flight on one device are consecutive except for the halo frames between two of
     * its blocks (they produce no output there): the span of `inflight_max` outputs, in local indices */
    const int halo  = pv->ndev > 1 ? pv->max_frames - 1 : 0;
    const int span  = pv->inflight_max + halo * ((pv->inflight_max + pv->block - 1) / pv->block + 1);
    pv->ring = pv->max_frames + span + 1;
    pv->cap  = pv->ndev * (pv->inflight_max + halo) + pv->max_frames + 2;
    pv->pending = calloc(pv->cap, sizeof(*pv->pending));
    if (pv->pending == NULL)
    {
        hb_error("nlmeans(cuda): calloc failed");
        goto fail;
    }

    cfg.ring_frames = pv->ring;
    cfg.out_slots   = span;
    for (int d = 0; d < pv->ndev; d++)
    {
        cfg.device = pv->devices[d];
        if (hbcu_nlmeans_create(&pv->gpu[d], &cfg) != 0 ||
            (d > 0 && hbcu_nlmeans_set_stream_slice(pv->gpu[d], 1) != 0))    /* only gpu[0] ever sees the stream's first frame */
        {
            /* no CPU fallback: the job continues without the filter (work.c:1861-1868) */
            hb_error("nlmeans(cuda): %s", hbcu_last_error());
            goto fail;
        }
    }
    if (pv->ndev == 1)
        hb_log("NLMeans (CUDA) on device %d, %d frames in flight", pv->devices[0], pv->inflight_max);
    else
        hb_log("NLMeans (CUDA) dealt over %d devices in blocks of %d frames, %d frames in flight each", pv->ndev, pv->block, pv->inflight_max);

    pv->device = pv->devices[0];
    pv->output = *init;
    if (pv->ndev > 1 && workers_start(pv) != 0)
    {
        hb_error("nlmeans(cuda): could not start the per-device submission threads");
        goto fail;
    }
    return 0;

fail:
    workers_stop(pv);
    for (int d = 0; d < NLM_MAX_DEVICES; d++)
        if (pv->gpu[d] != NULL) hbcu_nlmeans_destroy(pv->gpu[d]);
    free(pv->pending);
    free(pv);
    filter->private_data = NULL;
    return -1;
}

static void nlmeans_cuda_close(hb_filter_object_t *filter)
{
    hb_filter_private_t *pv = filter->private_data;
    if (pv == NULL) return;
    workers_stop(pv);                                    /* queued commands are executed, then the threads end */
    /* every handle first drains its device; peers only read each other's rings from queued copies, so destroy them
     * after ALL devices are idle */
    for (int d = 0; d < pv->ndev; d++)
        if (pv->gpu[d] != NULL) hbcu_nlmeans_sync(pv->gpu[d]);
    for (int d = 0; d < pv->ndev; d++)
        if (pv->gpu[d] != NULL) hbcu_nlmeans_destroy(pv->gpu[d]);
    for (int i = 0; i < pv->count; i++)
    {
        nlm_pending_t *p = pending_at(pv, i);
        hb_buffer_close(&p->in);
        hb_buffer_close(&p->out);
    }
    free(pv->pending);
    free(pv);
    filter->private_data = NULL;
}

/* block-cyclic owner of stream frame t */
static int owner_of(const hb_filter_private_t *pv, int64_t t)
{
    return pv->ndev == 1 ? 0 : (int)((t / pv->block) % pv->ndev);
}

/* hand frame `index` to its GPU: kernels + download into a fresh output buffer */
static int enqueue_frame(hb_filter_private_t *pv, nlm_pending_t *p, int navail)
{
    hb_buffer_t *out = pv->device_out
        ? hbcu_device_frame_buffer_init(pv->output.pix_fmt, pv->output.geometry.width, pv->output.geometry.height, pv->device)
        : hb_frame_buffer_init(pv->output.pix_fmt, pv->output.geometry.width, pv->output.geometry.height);
    if (out == NULL) return -1;
    out->f.color_prim      = pv->output.color_prim;
    out->f.color_transfer  = pv->output.color_transfer;
    out->f.color_matrix    = pv->output.color_matrix;
    out->f.color_range     = pv->output.color_range;
    out->f.chroma_location = pv->output.chroma_location;
    hb_buffer_copy_props(out, p->in);                      /* nlmeans.c:519 */

    void *planes[3];
    int   strides[3];
    for (int c = 0; c < 3; c++)
    {
        planes[c]  = out->plane[c].data;
        strides[c] = out->plane[c].stride;
    }
    if (navail > pv->max_frames) navail = pv->max_frames;  /* what the device holds behind p->li: the block's rest + its halo */
    if (pv->ndev > 1)
    {
        nlm_cmd_t c;
        memset(&c, 0, sizeof(c));
        c.kind = NLM_CMD_FILTER;
        c.li = p->li;
        c.p = p;
        c.navail = navail;
        p->out = out;
        p->submitted = 0;
        pv->dev_inflight[p->dev]++;
        worker_push(&pv->worker[p->dev], &c);
        return 0;
    }
    hbcu_nlmeans_t *gpu = pv->gpu[p->dev];
    const int rc = pv->device_out ? hbcu_nlmeans_filter_frame(gpu, p->li, navail, hbcu_buffer_frame(out))
                                  : hbcu_nlmeans_filter(gpu, p->li, navail, planes, strides);
    if (rc != 0)
    {
        hb_error("nlmeans(cuda): %s", hbcu_last_error());
        hb_buffer_close(&out);
        return -1;
    }
    p->out = out;
    pv->dev_inflight[p->dev]++;
    return 0;
}

/* enqueue, in stream order, every frame whose look-ahead window is complete (or, at EOF, whatever is left).
 * Returns 1 when it stopped because the next frame's device has `inflight_max` outputs pending, 0 otherwise, -1 on error */
static int enqueue_ready(hb_filter_private_t *pv, int flushing)
{
    while (pv->next_enqueue < pv->next_in)
    {
        const int64_t t = pv->next_enqueue;
        const int avail = (int)(pv->next_in - t);
        if (!flushing && avail < pv->max_frames) break;
        nlm_pending_t *oldest = pending_at(pv, 0);
        nlm_pending_t *p = pending_at(pv, (int)(t - oldest->index));
        if (pv->dev_inflight[p->dev] >= pv->inflight_max) return 1;
        if (enqueue_frame(pv, p, avail) != 0) return -1;
        pv->next_enqueue++;
    }
    return 0;
}

/* move finished frames (oldest first) to the list; block == wait for the oldest in flight */
static int harvest(hb_filter_private_t *pv, hb_buffer_list_t *list, int block_one, int block_all)
{
    while (pv->count > 0)
    {
        nlm_pending_t *p = pending_at(pv, 0);
        if (p->out == NULL) break;                           /* not enqueued yet */
        if (pv->ndev > 1)
        {
            /* the device's thread has to have issued the frame before wait / poll mean anything */
            int ready;
            hb_lock(pv->done_lock);
            while (!(ready = p->submitted) && !pv->failed && (block_one || block_all)) hb_cond_wait(pv->done_cv, pv->done_lock);
            hb_unlock(pv->done_lock);
            if (pv->failed)
            {
                hb_error("nlmeans(cuda): %s", pv->errmsg);
                return -1;
            }
            if (!ready) break;
        }
        hbcu_nlmeans_t *gpu = pv->gpu[p->dev];
        if (hbcu_buffer_frame(p->out) != NULL)
        {
            /* device output: its consumer orders itself behind the kernel through the frame's events.  A host input
             * buffer may be released once its (asynchronous) upload has left it */
            if (hbcu_buffer_frame(p->in) == NULL && hbcu_nlmeans_wait_upload(gpu, p->li) != 0) goto gpu_error;
        }
        else if (block_all || block_one)
        {
            if (hbcu_nlmeans_wait(gpu, p->li) != 0) goto gpu_error;
            block_one = 0;
        }
        else
        {
            int done = hbcu_nlmeans_poll(gpu, p->li);
            if (done < 0) goto gpu_error;
            if (done == 0) break;
        }
        hb_buffer_list_append(list, p->out);
        p->out = NULL;
        hb_buffer_close(&p->in);
        pv->dev_inflight[p->dev]--;
        pv->head = (pv->head + 1) % pv->cap;
        pv->count--;
    }
    return 0;

gpu_error:
    hb_error("nlmeans(cuda): %s", hbcu_last_error());
    return -1;
}

/* enqueue what can be enqueued; while a device's queue is full, wait for the oldest frame in flight and go on */
static int pump(hb_filter_private_t *pv, hb_buffer_list_t *list, int flushing)
{
    for (;;)
    {
        const int full = enqueue_ready(pv, flushing);
        if (full < 0) return -1;
        if (harvest(pv, list, full, 0) != 0) return -1;
        if (!full) return 0;
    }
}

static int nlmeans_cuda_work(hb_filter_object_t *filter, hb_buffer_t **buf_in, hb_buffer_t **buf_out)
{
    hb_filter_private_t *pv = filter->private_data;
    hb_buffer_t *in = *buf_in;
    hb_buffer_list_t list;
    hb_buffer_list_clear(&list);

    if (in->s.flags & HB_BUF_FLAG_EOF)
    {
        /* flush with the shrinking window (nlmeans.c:599-664), then forward EOF */
        while (pv->count > 0)
        {
            if (pump(pv, &list, 1) != 0 || harvest(pv, &list, 1, 0) != 0)
            {
                hb_buffer_list_close(&list);
                return HB_FILTER_FAILED;
            }
        }
        hb_buffer_list_append(&list, in);
        *buf_out = hb_buffer_list_clear(&list);
        *buf_in  = NULL;
        return HB_FILTER_DONE;
    }

    /* nlmeans_add_frame: the frame goes to its device; we keep the buffer until its
     * output is emitted because the upload reads it asynchronously */
    const void *planes[3];
    int strides[3];
    for (int c = 0; c < 3; c++)
    {
        planes[c]  = in->plane[c].data;
        strides[c] = in->plane[c].stride;
    }
    if (pv->count == pv->cap)
    {
        hb_error("nlmeans(cuda): internal queue overflow");
        return HB_FILTER_FAILED;
    }
    hbcu_frame_t *fin = hbcu_buffer_frame(in);
    if (fin != NULL && pv->ndev > 1)
    {
        hb_error("nlmeans(cuda): device-resident input needs a single device (devices=%d given)", pv->ndev);
        return HB_FILTER_FAILED;
    }
    const int64_t t  = pv->next_in;
    const int     d  = owner_of(pv, t);
    const int64_t li = pv->local_next[d];
    nlm_pending_t *p = pending_at(pv, pv->count);
    if (pv->failed)
    {
        hb_error("nlmeans(cuda): %s", pv->errmsg);
        return HB_FILTER_FAILED;
    }
    /* the entry is complete before any thread can see it */
    p->index = t;
    p->dev   = d;
    p->li    = li;
    p->in    = in;
    p->out   = NULL;
    p->uploaded = p->submitted = 0;
    if (pv->ndev > 1)
    {
        /* the owner's thread issues the upload; a frame among the first nframes-1 of its block is also the look-ahead of
         * the previous block, on another device: that device's thread copies it over NVLink once the upload is issued */
        nlm_cmd_t c;
        memset(&c, 0, sizeof(c));
        c.kind = NLM_CMD_UPLOAD;
        c.li = li;
        c.p = p;
        worker_push(&pv->worker[d], &c);
        pv->local_next[d]++;
        if (t >= pv->block && (t % pv->block) < pv->max_frames - 1)
        {
            const int q = owner_of(pv, t - pv->block);
            memset(&c, 0, sizeof(c));
            c.kind = NLM_CMD_PEER;
            c.li = pv->local_next[q];
            c.src_dev = d;
            c.src_li = li;
            c.src_p = p;
            worker_push(&pv->worker[q], &c);
            pv->local_next[q]++;
        }
    }
    else
    {
        if ((fin != NULL ? hbcu_nlmeans_upload_frame(pv->gpu[d], li, fin)
                         : hbcu_nlmeans_upload(pv->gpu[d], li, planes, strides)) != 0)
        {
            hb_error("nlmeans(cuda): %s", hbcu_last_error());
            return HB_FILTER_FAILED;
        }
        pv->local_next[d]++;
    }
    pv->count++;
    pv->next_in++;
    *buf_in = NULL;

    /* keep the device queues bounded: while a device has `inflight_max` outputs pending, wait for the oldest */
    if (pump(pv, &list, 0) != 0)
    {
        hb_buffer_list_close(&list);
        return HB_FILTER_FAILED;
    }
    *buf_out = hb_buffer_list_clear(&list);
    return HB_FILTER_OK;
}
