/* hbcu_device_frames.c -- frames that stay in HBM between two CUDA filters (SURVEY.md 8 f3).
 *
 * libhb moves frames between filters as hb_buffer_t through FIFOs; hardware paths already carry non-host payloads
 * there (storage_type AVFRAME / COREMEDIA, handbrake/internal.h:152-153; release in hb_buffer_close,
 * fifo.c:1016-1034) and put adapter filters at the ends of a hardware chain (platform/macosx/adapter_vt.c).
 * This file is the same pattern for CUDA:
 *   - hbcu_device_frame_buffer_init(): an hb_buffer_t whose planes are device memory (storage = hbcu_frame_t);
 *   - hb_buffer_close()/hb_buffer_shallow_dup() release/retain the frame through the hooks set below;
 *   - hb_filter_hbcu_upload / hb_filter_hbcu_download: the ends of the chain.
 * A CUDA filter emits device buffers when its init sees hw_pix_fmt == AV_PIX_FMT_CUDA, and accepts either kind on
 * input (it looks at storage_type per buffer).  No host thread ever waits for the GPU between two such filters:
 * the order of work is carried by the frame's events (include/hbcu.h, "device frames").
 */
#include "hbcu_device_frames.h"

#define XFER_MAX_PENDING 16

static void release_hook(void *storage) { hbcu_frame_release((hbcu_frame_t *)storage); }
static void retain_hook(void *storage)  { hbcu_frame_retain((hbcu_frame_t *)storage); }

static void install_hooks(void)
{
    hb_shim_set_device_release(release_hook);
    hb_shim_set_device_retain(retain_hook);
}

int hbcu_env_device(void)
{
    const char *dev_env = getenv("HBCU_DEVICE");
    return dev_env != NULL ? atoi(dev_env) : 0;
}

static int parse_device_list(const char *str, int *out)
{
    int n = 0;
    if (str == NULL) return 0;
    while (*str != '\0' && n < HBCU_MAX_DEVICES)
    {
        char *end = NULL;
        const long v = strtol(str, &end, 10);
        if (end == str || v < 0) return -1;
        out[n++] = (int)v;
        str = end;
        if (*str == ',' || *str == '+') str++;
        else if (*str != '\0') return -1;
    }
    return n;
}

int hbcu_settings_devices(const hb_dict_t *settings, int devices[HBCU_MAX_DEVICES])
{
    int n = 0;
    char *list = NULL;
    if (settings != NULL && hb_dict_extract_string(&list, settings, "devices"))
    {
        n = parse_device_list(list, devices);
        free(list);
        if (n <= 0) return -1;
        return n;
    }
    n = parse_device_list(getenv("HBCU_DEVICES"), devices);
    if (n < 0) return -1;
    if (n == 0)
    {
        devices[0] = hbcu_env_device();
        n = 1;
    }
    return n;
}

int hbcu_init_wants_device_output(const hb_filter_init_t *init)
{
    return init != NULL && init->hw_pix_fmt == AV_PIX_FMT_CUDA;
}

hbcu_frame_t *hbcu_buffer_frame(const hb_buffer_t *b)
{
    return (b != NULL && b->storage_type == HBCU_DEVICE) ? (hbcu_frame_t *)b->storage : NULL;
}

/* planes of a YUV frame as a device frame has them: 3, or 2 for a semi-planar format (NV12, P010, P016), whose
 * absent third plane is 0 rows of 0 bytes; row bytes are FFmpeg's linesizes (a row of Cb/Cr pairs is twice as long) */
static int frame_planes(int pix_fmt)
{
    const AVPixFmtDescriptor *desc = av_pix_fmt_desc_get(pix_fmt);
    if (desc == NULL || desc->nb_components < 3) return 0;
    return av_pix_fmt_count_planes(pix_fmt) == 2 ? 2 : 3;
}

hb_buffer_t *hbcu_device_frame_buffer_init(int pix_fmt, int width, int height, int device)
{
    const int nplanes = frame_planes(pix_fmt);
    if (nplanes == 0) return NULL;
    install_hooks();
    hb_buffer_t *b = hb_buffer_init(0);
    if (b == NULL) return NULL;
    b->f.max_plane = nplanes - 1;
    b->s.type      = FRAME_BUF;
    b->f.width     = width;
    b->f.height    = height;
    b->f.fmt       = pix_fmt;
    int row_bytes[3] = {0, 0, 0}, rows[3] = {0, 0, 0}, strides[3] = {0, 0, 0};
    for (int p = 0; p < nplanes; p++)
    {
        b->plane[p].stride = hb_image_stride(pix_fmt, width, p);
        b->plane[p].width  = hb_image_width(pix_fmt, width, p);
        b->plane[p].height = hb_image_height(pix_fmt, height, p);
        b->plane[p].size   = b->plane[p].stride * b->plane[p].height;
        row_bytes[p] = av_image_get_linesize(pix_fmt, width, p);
        rows[p]      = b->plane[p].height;
        strides[p]   = b->plane[p].stride;
        b->size     += b->plane[p].size;
    }
    hbcu_frame_t *f = NULL;
    if (hbcu_frame_alloc(&f, device, row_bytes, rows, strides) != 0)
    {
        hb_error("hbcu: device frame: %s", hbcu_last_error());
        hb_buffer_close(&b);
        return NULL;
    }
    for (int p = 0; p < nplanes; p++) b->plane[p].data = hbcu_frame_plane(f, p);
    b->storage_type = HBCU_DEVICE;
    b->storage = f;
    return b;
}

/* The decoder end of a zero-copy chain (SURVEY.md 8 f4): an AVFrame of AV_PIX_FMT_CUDA -- data[i] device pointers,
 * linesize[i], the frames context's device and stream -- becomes an HBCU_DEVICE hb_buffer_t without a copy
 * (hwaccel.c:15-60 is where libhb receives such frames; nvenc_common.c:329-336 where the encoder asks for them).
 * For NVDEC's semi-planar sw_format (NV12, P010, P016) only data[0..1] / linesize[0..1] are read.
 * `release(opaque)` is the caller's av_frame_free: it runs when the buffer is closed and the last device reader is done. */
hb_buffer_t *hbcu_wrap_cuda_frame(int pix_fmt, int width, int height, int device, void *const data[3], const int linesize[3],
                                  size_t readable_tail_bytes, void *cuda_stream, void (*release)(void *), void *opaque)
{
    const int nplanes = frame_planes(pix_fmt);
    if (nplanes == 0) return NULL;
    install_hooks();
    hb_buffer_t *b = hb_buffer_init(0);
    if (b == NULL) return NULL;
    b->f.max_plane = nplanes - 1;
    b->s.type      = FRAME_BUF;
    b->f.width     = width;
    b->f.height    = height;
    b->f.fmt       = pix_fmt;
    void *planes[3] = {NULL, NULL, NULL};
    int row_bytes[3] = {0, 0, 0}, rows[3] = {0, 0, 0}, strides[3] = {0, 0, 0};
    for (int p = 0; p < nplanes; p++)
    {
        b->plane[p].stride = linesize[p];
        b->plane[p].width  = hb_image_width(pix_fmt, width, p);
        b->plane[p].height = hb_image_height(pix_fmt, height, p);
        b->plane[p].size   = b->plane[p].stride * b->plane[p].height;
        b->plane[p].data   = data[p];
        planes[p]    = data[p];
        strides[p]   = linesize[p];
        row_bytes[p] = av_image_get_linesize(pix_fmt, width, p);
        rows[p]      = b->plane[p].height;
        b->size     += b->plane[p].size;
    }
    hbcu_frame_t *f = NULL;
    if (hbcu_frame_wrap(&f, device, planes, row_bytes, rows, strides, readable_tail_bytes, cuda_stream, release, opaque) != 0)
    {
        hb_error("hbcu: wrapped device frame: %s", hbcu_last_error());
        hb_buffer_close(&b);
        return NULL;
    }
    b->storage_type = HBCU_DEVICE;
    b->storage = f;
    return b;
}

/* ------------------------------------------------------------------ */
/* adapter filters                                                       */
/* ------------------------------------------------------------------ */
typedef struct
{
    hb_buffer_t *in, *out;
    int64_t      ticket;
} xfer_pending_t;

struct hb_filter_private_s
{
    hbcu_xfer_t *x;
    int          download, device;
    int          external;      /* HBCU_UPLOAD_EXTERNAL=1 (test hook): behave like a hardware decoder -- the uploaded frame is
                                 * a surface the adapter owns and goes downstream WRAPPED (hbcu_wrap_cuda_frame) */
    xfer_pending_t pending[XFER_MAX_PENDING];
    int head, count, inflight_max;
    int64_t next_ticket;
    hb_filter_init_t input, output;
};

static int  xfer_init(hb_filter_object_t *filter, hb_filter_init_t *init);
static int  xfer_work(hb_filter_object_t *filter, hb_buffer_t **buf_in, hb_buffer_t **buf_out);
static void xfer_close(hb_filter_object_t *filter);

hb_filter_object_t hb_filter_hbcu_upload =
{
    .id            = HB_FILTER_HBCU_UPLOAD,
    .enforce_order = 0,
    .name          = "Host to CUDA device frames (hbcu)",
    .short_name    = "hbcu-upload",
    .settings      = NULL,
    .init          = xfer_init,
    .work          = xfer_work,
    .close         = xfer_close,
};

hb_filter_object_t hb_filter_hbcu_download =
{
    .id            = HB_FILTER_HBCU_DOWNLOAD,
    .enforce_order = 0,
    .name          = "CUDA device frames to host (hbcu)",
    .short_name    = "hbcu-download",
    .settings      = NULL,
    .init          = xfer_init,
    .work          = xfer_work,
    .close         = xfer_close,
};

static int xfer_init(hb_filter_object_t *filter, hb_filter_init_t *init)
{
    hb_filter_private_t *pv = calloc(1, sizeof(*pv));
    if (pv == NULL) return -1;
    filter->private_data = pv;
    install_hooks();
    pv->download = filter->id == HB_FILTER_HBCU_DOWNLOAD;
    pv->device = hbcu_env_device();
    pv->inflight_max = 6;
    pv->input = *init;
    pv->external = !pv->download && getenv("HBCU_UPLOAD_EXTERNAL") != NULL && atoi(getenv("HBCU_UPLOAD_EXTERNAL")) != 0;
    if (hbcu_xfer_create(&pv->x, pv->device, XFER_MAX_PENDING) != 0)
    {
        hb_error("%s: %s", filter->short_name, hbcu_last_error());
        free(pv);
        filter->private_data = NULL;
        return -1;
    }
    /* downstream of the upload adapter frames are CUDA frames, downstream of the download adapter host frames */
    init->hw_pix_fmt = pv->download ? AV_PIX_FMT_NONE : AV_PIX_FMT_CUDA;
    pv->output = *init;
    return 0;
}

static void xfer_close(hb_filter_object_t *filter)
{
    hb_filter_private_t *pv = filter->private_data;
    if (pv == NULL) return;
    while (pv->count > 0)
    {
        xfer_pending_t *p = &pv->pending[pv->head];
        hbcu_xfer_wait(pv->x, p->ticket);
        hb_buffer_close(&p->in);
        hb_buffer_close(&p->out);
        pv->head = (pv->head + 1) % XFER_MAX_PENDING;
        pv->count--;
    }
    hbcu_xfer_destroy(pv->x);
    free(pv);
    filter->private_data = NULL;
}

static long g_surfaces_returned = 0;
long hbcu_test_surfaces_returned(void) { return g_surfaces_returned; }

static void surface_return(void *opaque)
{
    hb_buffer_t *surface = opaque;       /* the "decoder" gets its surface back: here it simply frees it */
    __sync_fetch_and_add(&g_surfaces_returned, 1);
    hb_buffer_close(&surface);
}

/* test hook: the uploaded frame plays a decoder-owned surface; what goes downstream is a wrapper around its planes */
static hb_buffer_t *as_decoder_surface(hb_filter_private_t *pv, hb_buffer_t *surface)
{
    void *data[3] = {NULL, NULL, NULL};
    int linesize[3] = {0, 0, 0};
    if (hbcu_xfer_wait(pv->x, pv->pending[pv->head].ticket) != 0) return NULL;      /* the "decode" is complete */
    for (int c = 0; c <= surface->f.max_plane; c++)
    {
        data[c]     = surface->plane[c].data;
        linesize[c] = surface->plane[c].stride;
    }
    hb_buffer_t *w = hbcu_wrap_cuda_frame(surface->f.fmt, surface->f.width, surface->f.height, pv->device, data, linesize,
                                          256, NULL, surface_return, surface);
    if (w == NULL) return NULL;
    w->f.color_prim      = surface->f.color_prim;
    w->f.color_transfer  = surface->f.color_transfer;
    w->f.color_matrix    = surface->f.color_matrix;
    w->f.color_range     = surface->f.color_range;
    w->f.chroma_location = surface->f.chroma_location;
    hb_buffer_copy_props(w, surface);
    return w;
}

static int xfer_harvest(hb_filter_private_t *pv, hb_buffer_list_t *list, int all)
{
    while (pv->count > 0)
    {
        xfer_pending_t *p = &pv->pending[pv->head];
        if (p->ticket >= 0)
        {
            /* an upload is finished for the host side once the copy has left the (pinned) input buffer, a download
             * once the data is in the output buffer: both are the ticket's event */
            if (all || pv->count > pv->inflight_max)
            {
                if (hbcu_xfer_wait(pv->x, p->ticket) != 0) return -1;
            }
            else
            {
                const int done = hbcu_xfer_poll(pv->x, p->ticket);
                if (done < 0) return -1;
                if (done == 0) break;
            }
        }
        if (pv->external && p->ticket >= 0 && (p->out = as_decoder_surface(pv, p->out)) == NULL) return -1;
        hb_buffer_list_append(list, p->out);
        p->out = NULL;
        if (p->in != NULL) hb_buffer_close(&p->in);
        pv->head = (pv->head + 1) % XFER_MAX_PENDING;
        pv->count--;
    }
    return 0;
}

static int xfer_work(hb_filter_object_t *filter, hb_buffer_t **buf_in, hb_buffer_t **buf_out)
{
    hb_filter_private_t *pv = filter->private_data;
    hb_buffer_t *in = *buf_in;
    hb_buffer_list_t list;
    hb_buffer_list_clear(&list);
    *buf_in = NULL;
    if (in->s.flags & HB_BUF_FLAG_EOF)
    {
        const int failed = xfer_harvest(pv, &list, 1) != 0;
        hb_buffer_list_append(&list, in);
        *buf_out = hb_buffer_list_clear(&list);
        return failed ? HB_FILTER_FAILED : HB_FILTER_DONE;
    }

    hbcu_frame_t *fin = hbcu_buffer_frame(in);
    xfer_pending_t *p = &pv->pending[(pv->head + pv->count) % XFER_MAX_PENDING];
    p->in = NULL;
    p->out = NULL;
    p->ticket = -1;
    if ((pv->download && fin == NULL) || (!pv->download && fin != NULL))
    {
        /* already where it should be: pass through, in order */
        p->out = in;
    }
    else
    {
        hb_buffer_t *out = pv->download ? hb_frame_buffer_init(in->f.fmt, in->f.width, in->f.height)
                                        : hbcu_device_frame_buffer_init(in->f.fmt, in->f.width, in->f.height, pv->device);
        if (out == NULL)
        {
            hb_buffer_close(&in);
            return HB_FILTER_FAILED;
        }
        out->f.color_prim      = in->f.color_prim;
        out->f.color_transfer  = in->f.color_transfer;
        out->f.color_matrix    = in->f.color_matrix;
        out->f.color_range     = in->f.color_range;
        out->f.chroma_location = in->f.chroma_location;
        hb_buffer_copy_props(out, in);
        hb_buffer_t *host = pv->download ? out : in;
        void *planes[3] = {NULL, NULL, NULL};
        int strides[3] = {0, 0, 0};
        for (int c = 0; c <= host->f.max_plane; c++)
        {
            planes[c]  = host->plane[c].data;
            strides[c] = host->plane[c].stride;
        }
        const int64_t ticket = pv->next_ticket++;
        const int rc = pv->download ? hbcu_xfer_download(pv->x, ticket, fin, planes, strides)
                                    : hbcu_xfer_upload(pv->x, ticket, hbcu_buffer_frame(out), (const void *const *)planes, strides);
        if (rc != 0)
        {
            hb_error("%s: %s", filter->short_name, hbcu_last_error());
            hb_buffer_close(&in);
            hb_buffer_close(&out);
            return HB_FILTER_FAILED;
        }
        p->in = in;
        p->out = out;
        p->ticket = ticket;
    }
    pv->count++;
    if (xfer_harvest(pv, &list, 0) != 0)
    {
        hb_error("%s: %s", filter->short_name, hbcu_last_error());
        hb_buffer_list_close(&list);
        return HB_FILTER_FAILED;
    }
    *buf_out = hb_buffer_list_clear(&list);
    return HB_FILTER_OK;
}
