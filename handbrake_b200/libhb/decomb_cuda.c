/* decomb_cuda.c -- hb_filter_decomb_cuda: drop-in for hb_filter_decomb
 * (reference libhb/decomb.c:182-193) running on an H100 through include/hbcu.h.
 *
 * Same plugin surface as the reference: settings keys and defaults (decomb.c:234-273),
 * prev/cur/next window with the first frame as its own predecessor and the last as its
 * own successor (:573-612), per-frame mode from s.combed (decomb template :816-831:
 * BLEND for lightly combed frames, pass-through dup for uncombed frames when
 * SELECTIVE), field order from the picture flags or the parity setting (:513-523),
 * two output fields with halved durations when bob is on (:527-569), bob doubling
 * init->vrate.num (:427-430), close-time log line (:446-450).
 *
 * What changes: the cpu_count row segments (yadif taskset) and the three EEDI2 plane
 * threads become kernels on the filter's streams; output pictures are produced
 * asynchronously and handed downstream in order (bounded number in flight), so the
 * burst pattern differs from the reference (which returns its pictures in the same
 * work() call) while order and content do not.
 */
#include "handbrake/handbrake.h"
#include "hbcu.h"
#include "hbcu_device_frames.h"

#define PARITY_DEFAULT -1
#define DECOMB_MAX_PENDING 64
#define DECOMB_BLOCK_DEFAULT 8

typedef struct
{
    hb_buffer_t *buf;       /* output picture */
    int64_t      ticket;    /* >= 0: the GPU is still writing it; -1: ready (pass-through) */
    int          dev;       /* which of pv->gpu[] wrote it */
} decomb_pending_t;

struct hb_filter_private_s
{
    int device, device_out;        /* device_out: pictures leave as HBCU_DEVICE buffers (hw_pix_fmt == AV_PIX_FMT_CUDA) */
    /* several GPUs (setting `devices=` / HBCU_DEVICES; not with EEDI2, whose edge mask carries state from field to field):
     * the ordered stream is dealt block-cyclically -- `block` frames per device in turn (mt_frame_filter.c:169-237 deals
     * frames to threads the same way); a picture reads prev / cur / next, so the first and the last frame of a block are
     * uploaded to the neighbouring block's device as well */
    int ndev, devices[HBCU_MAX_DEVICES], block;
    hbcu_decomb_t *gpu[HBCU_MAX_DEVICES];
    unsigned ref_devs[3];          /* devices (bit mask) ref[k] was uploaded to */
    int mode;
    int parity;

    hb_buffer_t *ref[3];
    int64_t      ref_index[3];
    int          ready;
    int64_t      next_index;
    int64_t      next_ticket;

    decomb_pending_t pending[DECOMB_MAX_PENDING];
    int              head, count;
    int              inflight_max;

    int deinterlaced, blended, unfiltered, frames;

    hb_filter_init_t input;
    hb_filter_init_t output;
};

static int  decomb_cuda_init(hb_filter_object_t *filter, hb_filter_init_t *init);
static int  decomb_cuda_work(hb_filter_object_t *filter, hb_buffer_t **buf_in, hb_buffer_t **buf_out);
static void decomb_cuda_close(hb_filter_object_t *filter);

static const char decomb_template[] =
    "mode=^"HB_INT_REG"$:magnitude-thresh=^"HB_INT_REG"$:variance-thresh=^"HB_INT_REG"$:"
    "laplacian-thresh=^"HB_INT_REG"$:dilation-thresh=^"HB_INT_REG"$:"
    "erosion-thresh=^"HB_INT_REG"$:noise-thresh=^"HB_INT_REG"$:"
    "search-distance=^"HB_INT_REG"$:postproc=^([0-3])$:parity=^([01])$";

hb_filter_object_t hb_filter_decomb_cuda =
{
    .id                = HB_FILTER_DECOMB,
    .enforce_order     = 1,
    .name              = "Decomb (CUDA sm_90a)",
    .short_name        = "decomb",
    .settings          = NULL,
    .init              = decomb_cuda_init,
    .work              = decomb_cuda_work,
    .close             = decomb_cuda_close,
    .settings_template = decomb_template,
};

static int decomb_cuda_init(hb_filter_object_t *filter, hb_filter_init_t *init)
{
    hb_filter_private_t *pv = calloc(1, sizeof(*pv));
    if (pv == NULL)
    {
        hb_error("decomb(cuda): calloc failed");
        return -1;
    }
    filter->private_data = pv;
    pv->input = *init;

    const AVPixFmtDescriptor *desc = av_pix_fmt_desc_get(init->pix_fmt);
    if (desc == NULL || desc->nb_components < 3 || av_pix_fmt_count_planes(init->pix_fmt) < 3)    /* planar YUV only */
    {
        hb_error("decomb(cuda): unsupported pixel format %d", init->pix_fmt);
        goto fail;
    }

    hbcu_decomb_config_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    /* defaults, decomb.c:234-243 */
    pv->mode                    = HBCU_DECOMB_YADIF | HBCU_DECOMB_BLEND | HBCU_DECOMB_CUBIC;
    cfg.magnitude_threshold     = 10;
    cfg.variance_threshold      = 20;
    cfg.laplacian_threshold     = 20;
    cfg.dilation_threshold      = 4;
    cfg.erosion_threshold       = 2;
    cfg.noise_threshold         = 50;
    cfg.maximum_search_distance = 24;
    cfg.post_processing         = 1;
    pv->parity                  = PARITY_DEFAULT;
    if (filter->settings)
    {
        hb_dict_t *dict = filter->settings;
        hb_dict_extract_int(&pv->mode, dict, "mode");
        hb_dict_extract_int(&pv->parity, dict, "parity");
        if (pv->mode & HBCU_DECOMB_EEDI2)
        {
            hb_dict_extract_int(&cfg.magnitude_threshold, dict, "magnitude-thresh");
            hb_dict_extract_int(&cfg.variance_threshold, dict, "variance-thresh");
            hb_dict_extract_int(&cfg.laplacian_threshold, dict, "laplacian-thresh");
            hb_dict_extract_int(&cfg.dilation_threshold, dict, "dilation-thresh");
            hb_dict_extract_int(&cfg.erosion_threshold, dict, "erosion-thresh");
            hb_dict_extract_int(&cfg.noise_threshold, dict, "noise-thresh");
            hb_dict_extract_int(&cfg.maximum_search_distance, dict, "search-distance");
            hb_dict_extract_int(&cfg.post_processing, dict, "postproc");
        }
    }
    cfg.width          = init->geometry.width;
    cfg.height         = init->geometry.height;
    cfg.depth          = desc->comp[0].depth;
    cfg.chroma_shift_w = desc->log2_chroma_w;
    cfg.chroma_shift_h = desc->log2_chroma_h;
    pv->ndev           = hbcu_settings_devices(filter->settings, pv->devices);
    pv->block          = DECOMB_BLOCK_DEFAULT;
    if (filter->settings) hb_dict_extract_int(&pv->block, filter->settings, "block");
    if (pv->block < 1) pv->block = 1;
    pv->device_out     = hbcu_init_wants_device_output(init);
    if (pv->ndev < 1 || (pv->ndev > 1 && (pv->device_out || (pv->mode & HBCU_DECOMB_EEDI2))))
    {
        hb_error("decomb(cuda): %s", pv->ndev < 1 ? "bad `devices` setting"
                 : "several devices need host output and a mode without EEDI2 (its edge mask carries state between fields)");
        goto fail;
    }
    pv->device         = pv->devices[0];
    pv->inflight_max   = 6 * pv->ndev < DECOMB_MAX_PENDING - 4 ? 6 * pv->ndev : DECOMB_MAX_PENDING - 4;
    cfg.slots          = pv->ndev > 1 ? pv->block + 6 : 6;
    cfg.out_slots      = 6 + 2 + 2;
    cfg.mode           = pv->mode;
    for (int d = 0; d < pv->ndev; d++)
    {
        cfg.device = pv->devices[d];
        if (hbcu_decomb_create(&pv->gpu[d], &cfg) != 0)
        {
            hb_error("decomb(cuda): %s", hbcu_last_error());
            goto fail;
        }
    }
    pv->ref_index[0] = pv->ref_index[1] = pv->ref_index[2] = -1;

    if (pv->mode & HBCU_DECOMB_BOB)
    {
        init->vrate.num *= 2;                    /* decomb.c:427-430 */
    }
    pv->output = *init;
    return 0;

fail:
    for (int d = 0; d < HBCU_MAX_DEVICES; d++)
        if (pv->gpu[d] != NULL) hbcu_decomb_destroy(pv->gpu[d]);
    free(pv);
    filter->private_data = NULL;
    return -1;
}

/* block-cyclic owner of stream frame t */
static int owner_of(const hb_filter_private_t *pv, int64_t t)
{
    return pv->ndev == 1 || t < 0 ? 0 : (int)((t / pv->block) % pv->ndev);
}

static void decomb_cuda_close(hb_filter_object_t *filter)
{
    hb_filter_private_t *pv = filter->private_data;
    if (pv == NULL) return;
    if (pv->frames > 1)
    {
        hb_log("decomb: deinterlaced %i | blended %i | unfiltered %i | total %i",
               pv->deinterlaced, pv->blended, pv->unfiltered, pv->frames);
    }
    for (int d = 0; d < pv->ndev; d++)
        if (pv->gpu[d] != NULL) hbcu_decomb_destroy(pv->gpu[d]);      /* waits for in-flight copies */
    for (int i = 0; i < pv->count; i++)
        hb_buffer_close(&pv->pending[(pv->head + i) % DECOMB_MAX_PENDING].buf);
    for (int ii = 0; ii < 3; ii++)
        hb_buffer_close(&pv->ref[ii]);
    free(pv);
    filter->private_data = NULL;
}

static void store_ref(hb_filter_private_t *pv, hb_buffer_t *b, int64_t index, unsigned devs)
{
    /* the upload of a frame reads its buffer asynchronously: make sure it is over (on every device it went to) before
     * the buffer goes back to the pool (normally long done -- the frame entered three calls ago) */
    if (pv->ref[0] != NULL && pv->ref_index[0] >= 0 && hbcu_buffer_frame(pv->ref[0]) == NULL)
        for (int d = 0; d < pv->ndev; d++)
            if (pv->ref_devs[0] & (1u << d)) hbcu_decomb_wait_upload(pv->gpu[d], pv->ref_index[0]);
    hb_buffer_close(&pv->ref[0]);
    for (int k = 0; k < 2; k++)
    {
        pv->ref[k]       = pv->ref[k + 1];
        pv->ref_index[k] = pv->ref_index[k + 1];
        pv->ref_devs[k]  = pv->ref_devs[k + 1];
    }
    pv->ref[2]       = b;
    pv->ref_index[2] = index;
    pv->ref_devs[2]  = devs;
}

/* move finished pictures (oldest first) to the list */
static int harvest(hb_filter_private_t *pv, hb_buffer_list_t *list, int min_free, int all)
{
    while (pv->count > 0)
    {
        decomb_pending_t *p = &pv->pending[pv->head];
        if (p->ticket >= 0)
        {
            const int must_wait = all || (DECOMB_MAX_PENDING - pv->count) < min_free || pv->count > pv->inflight_max;
            if (must_wait)
            {
                if (hbcu_decomb_wait(pv->gpu[p->dev], p->ticket) != 0) goto gpu_error;
            }
            else
            {
                const int done = hbcu_decomb_poll(pv->gpu[p->dev], p->ticket);
                if (done < 0) goto gpu_error;
                if (done == 0) break;
            }
        }
        hb_buffer_list_append(list, p->buf);
        p->buf = NULL;
        pv->head = (pv->head + 1) % DECOMB_MAX_PENDING;
        pv->count--;
    }
    return 0;

gpu_error:
    hb_error("decomb(cuda): %s", hbcu_last_error());
    return -1;
}

static void push_pending(hb_filter_private_t *pv, hb_buffer_t *buf, int64_t ticket, int dev)
{
    decomb_pending_t *p = &pv->pending[(pv->head + pv->count) % DECOMB_MAX_PENDING];
    p->buf    = buf;
    p->ticket = ticket;
    p->dev    = dev;
    pv->count++;
}

/* process_frame (decomb.c:500-571) */
static int process_frame(hb_filter_private_t *pv)
{
    hb_buffer_t *cur = pv->ref[1];
    if ((pv->mode & HBCU_DECOMB_SELECTIVE) && cur->s.combed == HB_COMB_NONE)
    {
        push_pending(pv, hb_buffer_shallow_dup(cur), -1, 0);
        pv->frames++;
        pv->unfiltered++;
        return 0;
    }

    int tff;
    if (pv->parity < 0)
    {
        const uint16_t flags = cur->s.flags;
        tff = ((flags & PIC_FLAG_PROGRESSIVE_FRAME) == 0) ? !!(flags & PIC_FLAG_TOP_FIELD_FIRST) : 1;
    }
    else
    {
        tff = (pv->parity & 1) ^ 1;
    }
    const int num_frames = (pv->mode & HBCU_DECOMB_BOB) ? 2 : 1;
    const int dev = owner_of(pv, pv->ref_index[1]);        /* prev and next were uploaded there too */
    hb_buffer_t *made[2] = { NULL, NULL };
    for (int frame = 0; frame < num_frames; frame++)
    {
        const int parity = frame ^ tff ^ 1;

        /* mode for this frame (decomb template :816-841) */
        int is_combed = HB_COMB_HEAVY, mode = 0;
        if (pv->mode & HBCU_DECOMB_SELECTIVE) is_combed = cur->s.combed;
        if ((pv->mode & HBCU_DECOMB_BLEND) && is_combed == HB_COMB_LIGHT) mode = HBCU_DECOMB_BLEND;
        else if (is_combed != HB_COMB_NONE) mode = pv->mode & ~HBCU_DECOMB_SELECTIVE;
        if (mode == HBCU_DECOMB_BLEND) pv->blended++;
        else if (mode != 0)            pv->deinterlaced++;
        else                           pv->unfiltered++;
        pv->frames++;

        hb_buffer_t *buf = pv->device_out ? hbcu_device_frame_buffer_init(cur->f.fmt, cur->f.width, cur->f.height, pv->device)
                                          : hb_frame_buffer_init(cur->f.fmt, cur->f.width, cur->f.height);
        if (buf == NULL) return -1;
        buf->f.color_prim      = pv->output.color_prim;
        buf->f.color_transfer  = pv->output.color_transfer;
        buf->f.color_matrix    = pv->output.color_matrix;
        buf->f.color_range     = pv->output.color_range;
        buf->f.chroma_location = pv->output.chroma_location;

        void *planes[3];
        int strides[3];
        for (int c = 0; c < 3; c++)
        {
            planes[c]  = buf->plane[c].data;
            strides[c] = buf->plane[c].stride;
        }
        const int64_t ticket = pv->next_ticket++;
        /* `mode` keeps the bob bit: the reference tests `mode == BLEND` / `mode == CUBIC` on it
         * (decomb template :756,:776), so e.g. cubic+bob runs no line filter at all */
        const int rc = pv->device_out
            ? hbcu_decomb_filter_frame(pv->gpu[dev], ticket, pv->ref_index[0], pv->ref_index[1], pv->ref_index[2], mode, parity, tff,
                                       hbcu_buffer_frame(buf))
            : hbcu_decomb_filter(pv->gpu[dev], ticket, pv->ref_index[0], pv->ref_index[1], pv->ref_index[2], mode, parity, tff,
                                 planes, strides);
        if (rc != 0)
        {
            hb_error("decomb(cuda): %s", hbcu_last_error());
            hb_buffer_close(&buf);
            return -1;
        }
        hb_buffer_copy_props(buf, cur);
        made[frame] = buf;
        /* a device picture needs no wait: its consumer orders itself behind the kernel through the frame's events */
        push_pending(pv, buf, pv->device_out ? -1 : ticket, dev);
    }
    if (pv->mode & HBCU_DECOMB_BOB)
    {
        /* halve the durations (decomb.c:560-569) */
        hb_buffer_t *first = made[0], *second = made[1];
        first->s.stop -= (first->s.stop - first->s.start) / 2LL;
        second->s.start = first->s.stop;
        second->s.new_chap = 0;
    }
    return 0;
}

static int decomb_cuda_work(hb_filter_object_t *filter, hb_buffer_t **buf_in, hb_buffer_t **buf_out)
{
    hb_filter_private_t *pv = filter->private_data;
    hb_buffer_t *in = *buf_in;
    hb_buffer_list_t list;
    hb_buffer_list_clear(&list);

    *buf_in = NULL;                                /* input is always consumed (decomb.c:581) */
    if (in->s.flags & HB_BUF_FLAG_EOF)
    {
        int failed = 0;
        if (pv->ref[2] != NULL)
        {
            /* the last frame is its own successor: same pixels, no second upload */
            store_ref(pv, hb_buffer_shallow_dup(pv->ref[2]), pv->ref_index[2], pv->ref_devs[2]);
            if (harvest(pv, &list, 2, 0) != 0 || process_frame(pv) != 0) failed = 1;
        }
        if (!failed && harvest(pv, &list, 0, 1) != 0) failed = 1;
        hb_buffer_list_append(&list, in);
        *buf_out = hb_buffer_list_clear(&list);
        return failed ? HB_FILTER_FAILED : HB_FILTER_DONE;
    }

    const int64_t index = pv->next_index++;
    const void *planes[3];
    int strides[3];
    for (int c = 0; c < 3; c++)
    {
        planes[c]  = in->plane[c].data;
        strides[c] = in->plane[c].stride;
    }
    hbcu_frame_t *fin = hbcu_buffer_frame(in);
    if (fin != NULL && pv->ndev > 1)
    {
        hb_error("decomb(cuda): device-resident input needs a single device");
        hb_buffer_close(&in);
        return HB_FILTER_FAILED;
    }
    /* the frame goes to its owner and, as the `next` of the previous block's last frame / the `prev` of the next block's
     * first frame, to that block's device as well */
    unsigned devs = 1u << owner_of(pv, index);
    if (pv->ndev > 1)
    {
        if (index % pv->block == 0 && index > 0) devs |= 1u << owner_of(pv, index - 1);
        if (index % pv->block == pv->block - 1)  devs |= 1u << owner_of(pv, index + 1);
    }
    for (int d = 0; d < pv->ndev; d++)
    {
        if (!(devs & (1u << d))) continue;
        if ((fin != NULL ? hbcu_decomb_upload_frame(pv->gpu[d], index, fin) : hbcu_decomb_upload(pv->gpu[d], index, planes, strides)) != 0)
        {
            hb_error("decomb(cuda): %s", hbcu_last_error());
            hb_buffer_close(&in);
            return HB_FILTER_FAILED;
        }
    }
    if (!pv->ready)
    {
        store_ref(pv, hb_buffer_shallow_dup(in), index, devs);
        store_ref(pv, in, index, devs);
        pv->ready = 1;
        return HB_FILTER_DELAY;
    }
    store_ref(pv, in, index, devs);
    if (harvest(pv, &list, 2, 0) != 0 || process_frame(pv) != 0 || harvest(pv, &list, 0, 0) != 0)
    {
        hb_buffer_list_close(&list);
        return HB_FILTER_FAILED;
    }
    *buf_out = hb_buffer_list_clear(&list);
    return HB_FILTER_OK;
}
