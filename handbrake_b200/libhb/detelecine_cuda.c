/* detelecine_cuda.c -- hb_filter_detelecine_cuda: drop-in for hb_filter_detelecine (pullup inverse telecine, reference
 * libhb/detelecine.c:113-133, 1006-1277) running on an H100 through include/hbcu.h (SURVEY.md 8 f4).
 *
 * Division of labour.  pullup is a small state machine over a queue of fields -- which field is compared with which,
 * where the cadence breaks, how many fields make the next frame and which of them -- fed by three per-block metrics of
 * every field and two max-reductions over them.  Everything that touches samples (the metrics, the reductions, weaving
 * two fields into a frame) runs on the device; pictures and metric arrays never leave it.  The state machine below works on
 * a few integers per field and asks the device for a pair of maxima per decision: one wait per input frame.
 *
 * Same settings keys, defaults and clamping as hb_detelecine_init (:1006-1095), same frame dropping / pass-through
 * protocol as hb_detelecine_work (:1116-1277): the first frame is passed through while the queue fills
 * (pullup_fakecount), frames of length < 2 are dropped, output carries the CURRENT input's timestamps.
 */
#include "handbrake/handbrake.h"
#include "hbcu.h"
#include "hbcu_device_frames.h"

#define DT_PICTURES    10      /* pullup_init_context: nbuffers < 10 -> 10 (:604-607); nothing ever raises it */
#define DT_MAX_FIELDS  64      /* nodes of the field ring: 9 to start with (:623), one more whenever it is full (:285-296) */
#define DT_NONE        (-1)

enum { HAVE_BREAKS = 1, HAVE_AFFINITY = 2 };      /* field flags  (:20-21) */
enum { BREAK_LEFT = 1, BREAK_RIGHT = 2 };         /* field breaks (:22-23) */

typedef struct
{
    int parity, picture;        /* picture DT_NONE: the field has been consumed (or never filled) */
    int flags, breaks, affinity;
    int prev, next;             /* ring links; a node is also the index of its metric slot on the device */
} dt_field_t;

typedef struct
{
    int lock, length, parity;
    int ifields[3], ofields[2];
    int picture;                /* the picture that holds the woven frame, DT_NONE until known */
} dt_frame_t;

struct hb_filter_private_s
{
    hbcu_detelecine_t *gpu;
    int strict_breaks, parity_setting;
    int half_value, quarter_value;
    int lock[DT_PICTURES][2];
    dt_field_t fld[DT_MAX_FIELDS];
    int nfld, first, last, head;
    dt_frame_t frame;
    int fakecount;
    int slot_breaks[DT_MAX_FIELDS], slot_affinity[DT_MAX_FIELDS];
    int results[4 * DT_MAX_FIELDS];
    int unsynced;               /* an upload from a host buffer may still be in flight */
    hb_buffer_t *pending_out;   /* a woven frame whose copy to the host is still running: it leaves with the NEXT call's output
                                 * (or ahead of EOF), so its PCIe copy overlaps the next picture's upload and metrics */
    int failed;
    int device, device_out;     /* device_out: woven frames leave as HBCU_DEVICE buffers (hw_pix_fmt == AV_PIX_FMT_CUDA) */
    hb_filter_init_t input, output;
};

static int  detelecine_cuda_init(hb_filter_object_t *filter, hb_filter_init_t *init);
static int  detelecine_cuda_work(hb_filter_object_t *filter, hb_buffer_t **buf_in, hb_buffer_t **buf_out);
static void detelecine_cuda_close(hb_filter_object_t *filter);

static const char detelecine_template[] =
    "skip-left=^"HB_INT_REG"$:skip-right=^"HB_INT_REG"$:"
    "skip-top=^"HB_INT_REG"$:skip-bottom=^"HB_INT_REG"$:"
    "strict-breaks=^"HB_BOOL_REG"$:plane=^([012])$:parity=^([01])$:"
    "disable=^"HB_BOOL_REG"$";

hb_filter_object_t hb_filter_detelecine_cuda =
{
    .id                = HB_FILTER_DETELECINE,
    .enforce_order     = 1,
    .name              = "Detelecine (pullup, CUDA sm_90a)",
    .short_name        = "detelecine",
    .settings          = NULL,
    .init              = detelecine_cuda_init,
    .work              = detelecine_cuda_work,
    .close             = detelecine_cuda_close,
    .settings_template = detelecine_template,
};

#define GPU(call)                                                         \
    do {                                                                  \
        if (!pv->failed && (call) != 0) {                                 \
            hb_error("detelecine(cuda): %s", hbcu_last_error());          \
            pv->failed = 1;                                               \
        }                                                                 \
    } while (0)

/* ---------------------------------------------------------------- picture locks (:773-789)
 * A lock request names field 0, field 1 or (2) both. */
static void lock_picture(hb_filter_private_t *pv, int picture, int which)
{
    if (picture == DT_NONE) return;
    if ((which + 1) & 1) pv->lock[picture][0]++;
    if ((which + 1) & 2) pv->lock[picture][1]++;
}

static void release_picture(hb_filter_private_t *pv, int picture, int which)
{
    if (picture == DT_NONE) return;
    if ((which + 1) & 1) pv->lock[picture][0]--;
    if ((which + 1) & 2) pv->lock[picture][1]--;
}

/* pullup_get_buffer (:791-842) is only ever called for a whole picture (parity 2: :1134 and :927), which leaves one
 * rule: the first picture neither of whose fields is in use */
static int get_whole_picture(hb_filter_private_t *pv)
{
    for (int i = 0; i < DT_PICTURES; i++)
    {
        if (pv->lock[i][0] == 0 && pv->lock[i][1] == 0)
        {
            lock_picture(pv, i, 2);
            return i;
        }
    }
    return DT_NONE;
}

/* ---------------------------------------------------------------- the field ring */
static void ring_init(hb_filter_private_t *pv)
{
    pv->nfld = 9;                                   /* head + 8 (:267-283, :623) */
    for (int i = 0; i < pv->nfld; i++)
    {
        memset(&pv->fld[i], 0, sizeof(pv->fld[i]));
        pv->fld[i].picture = DT_NONE;
        pv->fld[i].next = (i + 1) % pv->nfld;
        pv->fld[i].prev = (i + pv->nfld - 1) % pv->nfld;
    }
    pv->head = 0;
    pv->first = pv->last = DT_NONE;
}

/* pullup_check_field_queue (:285-296): a full ring gets a fresh node between head and first */
static int ring_grow_if_full(hb_filter_private_t *pv)
{
    if (pv->first == DT_NONE || pv->fld[pv->head].next != pv->first) return 0;
    if (pv->nfld == DT_MAX_FIELDS)
    {
        hb_error("detelecine(cuda): more than %d fields queued", DT_MAX_FIELDS);
        pv->failed = 1;
        return -1;
    }
    const int n = pv->nfld++;
    memset(&pv->fld[n], 0, sizeof(pv->fld[n]));
    pv->fld[n].picture = DT_NONE;
    pv->fld[n].prev = pv->head;
    pv->fld[n].next = pv->first;
    pv->fld[pv->head].next = n;
    pv->fld[pv->first].prev = n;
    return 0;
}

static int queue_length(const hb_filter_private_t *pv)       /* :319-328 */
{
    if (pv->first == DT_NONE || pv->last == DT_NONE) return 0;
    int count = 1;
    for (int f = pv->first; f != pv->last; f = pv->fld[f].next) count++;
    return count;
}

/* pullup_submit_field (:956-986): the field takes the node at `head`; its three metric arrays are computed against the
 * nodes behind it -- as far as those still own a picture (:242) */
static void submit_field(hb_filter_private_t *pv, int picture, int parity)
{
    if (ring_grow_if_full(pv) != 0) return;
    if (pv->last != DT_NONE && pv->fld[pv->last].parity == parity) return;     /* two fields of one parity in a row: drop */

    const int f = pv->head;
    dt_field_t *F = &pv->fld[f];
    F->parity = parity;
    F->picture = picture;
    lock_picture(pv, picture, parity);
    F->flags = F->breaks = F->affinity = 0;

    const int before = F->prev, before2 = pv->fld[before].prev;
    const int neighbour = pv->fld[before].picture;
    const int comb_top = neighbour == DT_NONE ? DT_NONE : parity ? neighbour : picture;
    const int comb_bottom = neighbour == DT_NONE ? DT_NONE : parity ? picture : neighbour;
    GPU(hbcu_detelecine_metrics(pv->gpu, f, picture, parity, pv->fld[before2].picture, comb_top, comb_bottom));

    if (pv->first == DT_NONE) pv->first = f;
    pv->last = f;
    pv->head = F->next;
}

/* ---------------------------------------------------------------- decisions */
/* Every reduction the coming evaluation can ask for is queued first and fetched with one wait.  Which fields lack
 * breaks / affinity depends only on flags and picture identities, never on metric values, so the set is known up front
 * (a superset: the affinity shortcut below may settle two more fields on the way). */
static void fetch_reductions(hb_filter_private_t *pv, int n)
{
    int slots = 0, f = pv->first;
    for (int i = 0; i < n - 1; i++, f = pv->fld[f].next)
    {
        const dt_field_t *F = &pv->fld[f];
        if (i < n - 3 && !(F->flags & HAVE_BREAKS))
        {
            const int f2 = pv->fld[F->next].next, f3 = pv->fld[f2].next;
            GPU(hbcu_detelecine_breaks(pv->gpu, f2, f3, slots));
            pv->slot_breaks[f] = slots++;
        }
        if (!(F->flags & HAVE_AFFINITY))
        {
            GPU(hbcu_detelecine_affinity(pv->gpu, F->prev, f, F->next, slots));
            pv->slot_affinity[f] = slots++;
        }
    }
    if (slots > 0)
    {
        GPU(hbcu_detelecine_fetch(pv->gpu, pv->results, slots));
        pv->unsynced = 0;
    }
}

/* pullup_compute_breaks (:345-380): does the cadence break between f1 and f2?  Decided from how field f2 and field f3
 * differ from their same-parity predecessors (f0, f1). */
static void settle_breaks(hb_filter_private_t *pv, int f0)
{
    dt_field_t *F0 = &pv->fld[f0], *F1 = &pv->fld[F0->next], *F2 = &pv->fld[F1->next], *F3 = &pv->fld[F2->next];
    if (F0->flags & HAVE_BREAKS) return;
    F0->flags |= HAVE_BREAKS;

    /* repeated fields are a certain sign */
    if (F0->picture == F2->picture && F1->picture != F3->picture) { F2->breaks |= BREAK_RIGHT; return; }
    if (F0->picture != F2->picture && F1->picture == F3->picture) { F1->breaks |= BREAK_LEFT;  return; }

    const int max_l = pv->results[2 * pv->slot_breaks[f0]], max_r = pv->results[2 * pv->slot_breaks[f0] + 1];
    if (max_l + max_r < pv->half_value) return;               /* mostly quantisation noise */
    if (max_l > 4 * max_r) F1->breaks |= BREAK_LEFT;
    if (max_r > 4 * max_l) F2->breaks |= BREAK_RIGHT;
}

/* pullup_compute_affinity (:382-434): does field f weave better with its predecessor (-1) or its successor (+1)? */
static void settle_affinity(hb_filter_private_t *pv, int f)
{
    dt_field_t *F = &pv->fld[f], *N = &pv->fld[F->next], *NN = &pv->fld[N->next];
    if (F->flags & HAVE_AFFINITY) return;
    F->flags |= HAVE_AFFINITY;

    if (F->picture == NN->picture)                            /* a repeated field brackets its successor */
    {
        F->affinity = 1;
        N->affinity = 0;
        NN->affinity = -1;
        N->flags |= HAVE_AFFINITY;
        NN->flags |= HAVE_AFFINITY;
        return;
    }
    const int max_l = pv->results[2 * pv->slot_affinity[f]], max_r = pv->results[2 * pv->slot_affinity[f] + 1];
    if (max_l + max_r < pv->quarter_value) return;
    if (max_r > 6 * max_l)      F->affinity = -1;
    else if (max_l > 6 * max_r) F->affinity = 1;
}

static int first_break(const hb_filter_private_t *pv, int f, int max)      /* :330-343 */
{
    for (int i = 0; i < max; i++)
    {
        if ((pv->fld[f].breaks & BREAK_RIGHT) || (pv->fld[pv->fld[f].next].breaks & BREAK_LEFT)) return i + 1;
        f = pv->fld[f].next;
    }
    return 0;
}

/* pullup_decide_frame_length (:448-535): how many of the queued fields make the next frame (0: not enough queued).
 * c->strict_pairs is never set by HandBrake, so the branch it guards (:481-488) does not exist here. */
static int decide_frame_length(hb_filter_private_t *pv)
{
    const int n = queue_length(pv);
    if (n < 4) return 0;

    fetch_reductions(pv, n);
    if (pv->failed) return 0;
    for (int i = 0, f = pv->first; i < n - 1; i++, f = pv->fld[f].next)       /* pullup_foo (:436-446) */
    {
        if (i < n - 3) settle_breaks(pv, f);
        settle_affinity(pv, f);
    }

    const dt_field_t *F0 = &pv->fld[pv->first], *F1 = &pv->fld[F0->next], *F2 = &pv->fld[F1->next];
    if (F0->affinity == -1) return 1;

    int where = first_break(pv, pv->first, 3);
    if (where == 1 && pv->strict_breaks < 0) where = 0;

    switch (where)
    {
        case 1:  return (pv->strict_breaks < 1 && F0->affinity == 1 && F1->affinity == -1) ? 2 : 1;
        case 2:  return F1->affinity == 1 ? 1 : 2;
        case 3:  return F2->affinity == 1 ? 2 : 3;
        default: break;
    }
    /* no break within three fields: let the affinities speak */
    if (F1->affinity == 1)  return 1;
    if (F1->affinity == -1) return 2;
    if (F2->affinity == -1) return F0->affinity == 1 ? 3 : 1;
    return 2;
}

/* pullup_get_frame (:851-908): take the frame's fields off the queue and name the two that will be shown */
static dt_frame_t *get_frame(hb_filter_private_t *pv)
{
    dt_frame_t *fr = &pv->frame;
    if (pv->failed || pv->first == DT_NONE) return NULL;     /* no field was ever queued (a failed first submit) */
    const int n = decide_frame_length(pv);
    if (n == 0 || fr->lock) return NULL;
    int aff = pv->fld[pv->fld[pv->first].next].affinity;

    fr->lock++;
    fr->length = n;
    fr->parity = pv->fld[pv->first].parity;
    fr->picture = DT_NONE;
    for (int i = 0; i < n; i++)
    {
        fr->ifields[i] = pv->fld[pv->first].picture;        /* the field's lock travels with it */
        pv->fld[pv->first].picture = DT_NONE;
        pv->first = pv->fld[pv->first].next;
    }
    if (n == 1)
    {
        fr->ofields[fr->parity] = fr->ifields[0];
        fr->ofields[fr->parity ^ 1] = DT_NONE;
    }
    else if (n == 2)
    {
        fr->ofields[fr->parity] = fr->ifields[0];
        fr->ofields[fr->parity ^ 1] = fr->ifields[1];
    }
    else
    {
        if (aff == 0) aff = fr->ifields[0] == fr->ifields[1] ? -1 : 1;
        fr->ofields[fr->parity] = fr->ifields[1 + aff];
        fr->ofields[fr->parity ^ 1] = fr->ifields[1];
    }
    lock_picture(pv, fr->ofields[0], 0);
    lock_picture(pv, fr->ofields[1], 1);
    if (fr->ofields[0] == fr->ofields[1])
    {
        fr->picture = fr->ofields[0];
        lock_picture(pv, fr->picture, 2);
    }
    return fr;
}

/* pullup_pack_frame (:910-935): weave the two fields into one picture -- in place when the other half of one of the two
 * pictures is free, else in a fresh picture */
static int pack_frame(hb_filter_private_t *pv, dt_frame_t *fr)
{
    if (fr->picture != DT_NONE) return 0;
    if (fr->length < 2) return -1;
    for (int i = 0; i < 2; i++)
    {
        if (pv->lock[fr->ofields[i]][i ^ 1]) continue;
        fr->picture = fr->ofields[i];
        lock_picture(pv, fr->picture, 2);
        GPU(hbcu_detelecine_copy_field(pv->gpu, fr->picture, fr->ofields[i ^ 1], i ^ 1));
        return 0;
    }
    fr->picture = get_whole_picture(pv);
    if (fr->picture == DT_NONE) return -1;
    GPU(hbcu_detelecine_copy_field(pv->gpu, fr->picture, fr->ofields[0], 0));
    GPU(hbcu_detelecine_copy_field(pv->gpu, fr->picture, fr->ofields[1], 1));
    return 0;
}

static void release_frame(hb_filter_private_t *pv, dt_frame_t *fr)         /* :937-949 */
{
    for (int i = 0; i < fr->length; i++) release_picture(pv, fr->ifields[i], fr->parity ^ (i & 1));
    release_picture(pv, fr->ofields[0], 0);
    release_picture(pv, fr->ofields[1], 1);
    if (fr->picture != DT_NONE) release_picture(pv, fr->picture, 2);
    fr->lock--;
}

/* ---------------------------------------------------------------- the filter object */
static int detelecine_cuda_init(hb_filter_object_t *filter, hb_filter_init_t *init)
{
    hb_filter_private_t *pv = calloc(1, sizeof(*pv));
    if (pv == NULL)
    {
        hb_error("detelecine(cuda): calloc failed");
        return -1;
    }
    filter->private_data = pv;
    pv->input = *init;
    /* inside a device-resident chain (hw_pix_fmt == AV_PIX_FMT_CUDA) pictures arrive in and leave in HBCU_DEVICE buffers;
     * either kind is accepted per buffer */
    pv->device_out = hbcu_init_wants_device_output(init);

    /* :1025-1047: junk margins of at least one 8-sample column and four line pairs */
    int top = 4, bottom = 4, left = 1, right = 1, plane = 0;
    pv->strict_breaks = -1;
    pv->parity_setting = -1;
    if (filter->settings != NULL)
    {
        hb_dict_extract_int(&top,    filter->settings, "skip-top");
        hb_dict_extract_int(&bottom, filter->settings, "skip-bottom");
        hb_dict_extract_int(&left,   filter->settings, "skip-left");
        hb_dict_extract_int(&right,  filter->settings, "skip-right");
        hb_dict_extract_int(&pv->strict_breaks, filter->settings, "strict-breaks");
        hb_dict_extract_int(&plane, filter->settings, "plane");
        hb_dict_extract_int(&pv->parity_setting, filter->settings, "parity");
    }
    const AVPixFmtDescriptor *desc = av_pix_fmt_desc_get(init->pix_fmt);
    if (desc == NULL || desc->nb_components < 3 || av_pix_fmt_count_planes(init->pix_fmt) < 3)    /* planar YUV only */
    {
        hb_error("detelecine(cuda): unsupported pixel format %d", init->pix_fmt);
        goto fail;
    }
    const int depth = desc->comp[0].depth;
    pv->half_value = (1 << depth) / 2;
    pv->quarter_value = (1 << depth) / 4;
    if (plane >= desc->nb_components || plane < 0) plane = 0;           /* :1076-1079 */

    hbcu_detelecine_config_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.width          = init->geometry.width;
    cfg.height         = init->geometry.height;
    cfg.depth          = depth;
    cfg.chroma_shift_w = desc->log2_chroma_w;
    cfg.chroma_shift_h = desc->log2_chroma_h;
    const char *dev_env = getenv("HBCU_DEVICE");
    cfg.device         = dev_env != NULL ? atoi(dev_env) : 0;
    pv->device         = cfg.device;
    cfg.pictures       = DT_PICTURES;
    cfg.fields         = DT_MAX_FIELDS;
    cfg.results        = 2 * DT_MAX_FIELDS;
    cfg.metric_plane   = plane;
    cfg.junk_top       = top    > 4 ? top    : 4;
    cfg.junk_bottom    = bottom > 4 ? bottom : 4;
    cfg.junk_left      = left   > 1 ? left   : 1;
    cfg.junk_right     = right  > 1 ? right  : 1;
    if (hbcu_detelecine_create(&pv->gpu, &cfg) != 0)
    {
        hb_error("detelecine(cuda): %s", hbcu_last_error());
        goto fail;
    }
    ring_init(pv);
    pv->fakecount = 1;
    pv->output = *init;
    return 0;

fail:
    free(pv);
    filter->private_data = NULL;
    return -1;
}

static void detelecine_cuda_close(hb_filter_object_t *filter)
{
    hb_filter_private_t *pv = filter->private_data;
    if (pv == NULL) return;
    if (pv->pending_out != NULL)
    {
        if (pv->gpu != NULL) hbcu_detelecine_download_end(pv->gpu);
        hb_buffer_close(&pv->pending_out);
    }
    if (pv->gpu != NULL) hbcu_detelecine_destroy(pv->gpu);
    free(pv);
    filter->private_data = NULL;
}

/* the frame parked by the previous call, its copy to the host finished; NULL when there is none */
static hb_buffer_t *take_pending(hb_filter_private_t *pv)
{
    hb_buffer_t *out = pv->pending_out;
    if (out == NULL) return NULL;
    pv->pending_out = NULL;
    if (hbcu_detelecine_download_end(pv->gpu) != 0)
    {
        hb_error("detelecine(cuda): %s", hbcu_last_error());
        pv->failed = 1;
        hb_buffer_close(&out);
        return NULL;
    }
    return out;
}

/* the input buffer goes back to its owner when work() returns: no copy out of it may still be running.  A call that has
 * nothing new to show still hands on the frame the previous call parked. */
static int leave(hb_filter_private_t *pv, int status, hb_buffer_t **buf_out)
{
    if (pv->unsynced)
    {
        GPU(hbcu_detelecine_fetch(pv->gpu, NULL, 0));
        pv->unsynced = 0;
    }
    if (buf_out != NULL && !pv->failed && status == HB_FILTER_OK) *buf_out = take_pending(pv);
    return pv->failed ? HB_FILTER_FAILED : status;
}

static int detelecine_cuda_work(hb_filter_object_t *filter, hb_buffer_t **buf_in, hb_buffer_t **buf_out)
{
    hb_filter_private_t *pv = filter->private_data;
    hb_buffer_t *in = *buf_in;

    if (in->s.flags & HB_BUF_FLAG_EOF)
    {
        hb_buffer_t *last = pv->failed ? NULL : take_pending(pv);
        if (last != NULL) last->next = in;
        *buf_out = last != NULL ? last : in;
        *buf_in = NULL;
        return HB_FILTER_DONE;
    }
    if (pv->failed) return HB_FILTER_FAILED;

    const int picture = get_whole_picture(pv);
    if (picture == DT_NONE)
    {
        hb_log("Could not get buffer from pullup!");
        return HB_FILTER_FAILED;
    }
    const void *planes[3] = { in->plane[0].data, in->plane[1].data, in->plane[2].data };
    const int strides[3] = { in->plane[0].stride, in->plane[1].stride, in->plane[2].stride };
    if (hbcu_buffer_frame(in) != NULL) GPU(hbcu_detelecine_upload_frame(pv->gpu, picture, hbcu_buffer_frame(in)));
    else                               GPU(hbcu_detelecine_upload(pv->gpu, picture, planes, strides));
    pv->unsynced = hbcu_buffer_frame(in) == NULL;       /* a device frame's copy is ordered by the frame's own events */

    /* field order: the TFF flag, else bottom field first unless the user says otherwise (:1166-1184) */
    int parity = 1;
    if (in->s.flags & PIC_FLAG_TOP_FIELD_FIRST) parity = 0;
    else if (pv->parity_setting == 0)           parity = 0;
    if (pv->parity_setting == 1)                parity = 1;

    submit_field(pv, picture, parity);
    submit_field(pv, picture, parity ^ 1);
    if (in->s.flags & PIC_FLAG_REPEAT_FIRST_FIELD) submit_field(pv, picture, parity);
    release_picture(pv, picture, 2);

    dt_frame_t *frame = get_frame(pv);
    if (frame == NULL)
    {
        if (pv->fakecount == 0) return leave(pv, HB_FILTER_OK, buf_out);  /* nothing to show for this input */
        pv->fakecount--;                                                   /* the queue is still filling: pass through */
        const int status = leave(pv, HB_FILTER_OK, NULL);
        if (status == HB_FILTER_OK)
        {
            hb_buffer_t *before = take_pending(pv);                        /* (none while the queue fills; order kept anyway) */
            if (pv->failed) return HB_FILTER_FAILED;
            *buf_in = NULL;
            if (before != NULL) before->next = in;
            *buf_out = before != NULL ? before : in;
        }
        return status;
    }

    /* frames of a single field are dropped; look for up to two more (:1211-1244) */
    if (frame->length < 2)
    {
        release_frame(pv, frame);
        frame = get_frame(pv);
        if (frame == NULL) return leave(pv, HB_FILTER_OK, buf_out);
        if (frame->length < 2)
        {
            release_frame(pv, frame);
            if (!(in->s.flags & PIC_FLAG_REPEAT_FIRST_FIELD)) return leave(pv, HB_FILTER_OK, buf_out);
            frame = get_frame(pv);
            if (frame == NULL) return leave(pv, HB_FILTER_OK, buf_out);
            if (frame->length < 2)
            {
                release_frame(pv, frame);
                return leave(pv, HB_FILTER_OK, buf_out);
            }
        }
    }

    if (frame->picture == DT_NONE && pack_frame(pv, frame) != 0)
    {
        hb_error("detelecine(cuda): no free picture to weave a frame in");
        pv->failed = 1;
        release_frame(pv, frame);
        return leave(pv, HB_FILTER_FAILED, NULL);
    }

    hb_buffer_t *out = pv->device_out ? hbcu_device_frame_buffer_init(pv->output.pix_fmt, in->f.width, in->f.height, pv->device)
                                      : hb_frame_buffer_init(pv->output.pix_fmt, in->f.width, in->f.height);
    if (out == NULL)
    {
        release_frame(pv, frame);
        return leave(pv, HB_FILTER_FAILED, NULL);
    }
    out->f.color_prim      = pv->output.color_prim;
    out->f.color_transfer  = pv->output.color_transfer;
    out->f.color_matrix    = pv->output.color_matrix;
    out->f.color_range     = pv->output.color_range;
    out->f.chroma_location = pv->output.chroma_location;

    if (pv->device_out)
    {
        /* stays in HBM: a device copy queued behind the weave, the consumer orders itself behind the frame's event */
        GPU(hbcu_detelecine_download_frame(pv->gpu, frame->picture, hbcu_buffer_frame(out)));
        if (pv->unsynced)
        {
            GPU(hbcu_detelecine_fetch(pv->gpu, NULL, 0));           /* a HOST input buffer goes back to its owner now */
            pv->unsynced = 0;
        }
    }
    else
    {
        void *oplanes[3] = { out->plane[0].data, out->plane[1].data, out->plane[2].data };
        const int ostrides[3] = { out->plane[0].stride, out->plane[1].stride, out->plane[2].stride };
        /* the previous frame's copy has had a whole call to finish; this one's starts now and is collected by the next call */
        hb_buffer_t *before = take_pending(pv);
        GPU(hbcu_detelecine_download_begin(pv->gpu, frame->picture, oplanes, ostrides));
        if (pv->unsynced)
        {
            GPU(hbcu_detelecine_fetch(pv->gpu, NULL, 0));               /* the host input buffer goes back to its owner now */
            pv->unsynced = 0;
        }
        release_frame(pv, frame);
        if (pv->failed)
        {
            hbcu_detelecine_download_end(pv->gpu);
            hb_buffer_close(&out);
            if (before != NULL) hb_buffer_close(&before);
            return HB_FILTER_FAILED;
        }
        hb_buffer_copy_props(out, in);
        pv->pending_out = out;
        *buf_out = before;
        return HB_FILTER_OK;
    }
    release_frame(pv, frame);
    if (pv->failed)
    {
        hb_buffer_close(&out);
        return HB_FILTER_FAILED;
    }
    hb_buffer_copy_props(out, in);
    *buf_out = out;
    return HB_FILTER_OK;
}
