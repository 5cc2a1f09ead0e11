/* hb_runtime.c -- runtime half of the libhb shim (see handbrake/handbrake.h).
 *
 * Restates only the semantics the video-filter hot path depends on:
 *   frame buffers      libhb/fifo.c:358-441, 618-622, 725-881, 906-959, 1037-1083
 *   buffer lists       libhb/common.c:4002-4232
 *   settings dict      libhb/hb_dict.c:538-605 (extract_* return 1 when key present)
 *   ports              libhb/ports.c (hb_lock/hb_cond/hb_thread over pthreads)
 *
 * Deliberate difference from libhb: hb_frame_buffer_init() returns ZEROED
 * memory.  libhb's pool hands back recycled, uninitialised buffers; EEDI2's
 * edge mask keeps state in such a buffer (eedi2 template :122-195), so a
 * deterministic oracle needs a defined starting state (SURVEY.md 8a/a21).
 */
#define _GNU_SOURCE
#include "handbrake/handbrake.h"

#include <ctype.h>
#include <pthread.h>
#include <sched.h>
#include <stdarg.h>
#include <unistd.h>

/* ------------------------------------------------------------------ */
/* pixel format table                                                   */
/* ------------------------------------------------------------------ */
#define DESC(nm, cw, ch, d, ncomp) \
    { nm, ncomp, cw, ch, 0, { {0, 0, 0, 0, d}, {1, 0, 0, 0, d}, {2, 0, 0, 0, d}, {0, 0, 0, 0, 0} } }

static const AVPixFmtDescriptor desc_yuv420p    = DESC("yuv420p",     1, 1,  8, 3);
static const AVPixFmtDescriptor desc_yuv422p    = DESC("yuv422p",     1, 0,  8, 3);
static const AVPixFmtDescriptor desc_yuv444p    = DESC("yuv444p",     0, 0,  8, 3);
static const AVPixFmtDescriptor desc_gray8      = { "gray", 1, 0, 0, 0, { {0, 0, 0, 0, 8} } };
static const AVPixFmtDescriptor desc_yuv420p10  = DESC("yuv420p10le", 1, 1, 10, 3);
static const AVPixFmtDescriptor desc_yuv422p10  = DESC("yuv422p10le", 1, 0, 10, 3);
static const AVPixFmtDescriptor desc_yuv444p10  = DESC("yuv444p10le", 0, 0, 10, 3);
static const AVPixFmtDescriptor desc_yuv420p12  = DESC("yuv420p12le", 1, 1, 12, 3);
static const AVPixFmtDescriptor desc_yuv420p16  = DESC("yuv420p16le", 1, 1, 16, 3);
#define DESC_A(nm, cw, ch) \
    { nm, 4, cw, ch, 0, { {0, 0, 0, 0, 8}, {1, 0, 0, 0, 8}, {2, 0, 0, 0, 8}, {3, 0, 0, 0, 8} } }
static const AVPixFmtDescriptor desc_yuva420p   = DESC_A("yuva420p", 1, 1);
static const AVPixFmtDescriptor desc_yuva422p   = DESC_A("yuva422p", 1, 0);
static const AVPixFmtDescriptor desc_yuva444p   = DESC_A("yuva444p", 0, 0);
/* libavutil/pixdesc.c: Cb and Cr share plane 1, interleaved (step = one Cb/Cr pair, Cr one sample after Cb) */
#define DESC_SEMI(nm, bytes, sh, d) \
    { nm, 3, 1, 1, 0, { {0, bytes, 0, sh, d}, {1, 2 * (bytes), 0, sh, d}, {1, 2 * (bytes), bytes, sh, d}, {0, 0, 0, 0, 0} } }
static const AVPixFmtDescriptor desc_nv12       = DESC_SEMI("nv12",    1, 0,  8);
static const AVPixFmtDescriptor desc_p010       = DESC_SEMI("p010le",  2, 6, 10);
static const AVPixFmtDescriptor desc_p016       = DESC_SEMI("p016le",  2, 0, 16);

const AVPixFmtDescriptor *av_pix_fmt_desc_get(int pix_fmt)
{
    switch (pix_fmt)
    {
        case AV_PIX_FMT_YUV420P:     return &desc_yuv420p;
        case AV_PIX_FMT_YUV422P:     return &desc_yuv422p;
        case AV_PIX_FMT_YUV444P:     return &desc_yuv444p;
        case AV_PIX_FMT_GRAY8:       return &desc_gray8;
        case AV_PIX_FMT_YUV420P10LE: return &desc_yuv420p10;
        case AV_PIX_FMT_YUV422P10LE: return &desc_yuv422p10;
        case AV_PIX_FMT_YUV444P10LE: return &desc_yuv444p10;
        case AV_PIX_FMT_YUV420P12LE: return &desc_yuv420p12;
        case AV_PIX_FMT_YUV420P16LE: return &desc_yuv420p16;
        case AV_PIX_FMT_YUVA420P:    return &desc_yuva420p;
        case AV_PIX_FMT_YUVA422P:    return &desc_yuva422p;
        case AV_PIX_FMT_YUVA444P:    return &desc_yuva444p;
        case AV_PIX_FMT_NV12:        return &desc_nv12;
        case AV_PIX_FMT_P010LE:      return &desc_p010;
        case AV_PIX_FMT_P016LE:      return &desc_p016;
        default:                     return NULL;
    }
}

enum AVPixelFormat av_get_pix_fmt(const char *name)
{
    static const enum AVPixelFormat known[] = {
        AV_PIX_FMT_YUV420P, AV_PIX_FMT_YUV422P, AV_PIX_FMT_YUV444P, AV_PIX_FMT_GRAY8, AV_PIX_FMT_YUV420P10LE,
        AV_PIX_FMT_YUV422P10LE, AV_PIX_FMT_YUV444P10LE, AV_PIX_FMT_YUV420P12LE, AV_PIX_FMT_YUV420P16LE,
        AV_PIX_FMT_YUVA420P, AV_PIX_FMT_YUVA422P, AV_PIX_FMT_YUVA444P, AV_PIX_FMT_NV12, AV_PIX_FMT_P010LE, AV_PIX_FMT_P016LE,
    };
    if (name == NULL) return AV_PIX_FMT_NONE;
    char native[64];
    snprintf(native, sizeof(native), "%sle", name);
    for (int pass = 0; pass < 2; pass++)
        for (size_t i = 0; i < sizeof(known) / sizeof(known[0]); i++)
            if (strcmp(av_pix_fmt_desc_get(known[i])->name, pass == 0 ? name : native) == 0)
                return known[i];
    return AV_PIX_FMT_NONE;
}

const char *av_get_pix_fmt_name(enum AVPixelFormat pix_fmt)
{
    const AVPixFmtDescriptor *d = av_pix_fmt_desc_get(pix_fmt);
    return d != NULL ? d->name : NULL;
}

int av_pix_fmt_count_planes(int pix_fmt)
{
    const AVPixFmtDescriptor *d = av_pix_fmt_desc_get(pix_fmt);
    if (d == NULL) return -1;
    int seen[4] = {0, 0, 0, 0}, n = 0;
    for (int c = 0; c < d->nb_components; c++)
        if (!seen[d->comp[c].plane]++) n++;
    return n;
}

/* Restatement of common.c:7054-7091.  Weak: the reference build (oracle/Makefile) links the reference's own definition
 * next to this file, and that one must win there. */
__attribute__((weak)) void hb_compute_chroma_smoothing_coefficient(uint32_t chroma_coeffs[2][4], int pix_fmt, int chroma_location)
{
    const AVPixFmtDescriptor *desc = av_pix_fmt_desc_get(pix_fmt);
    const int sw = desc->log2_chroma_w, sh = desc->log2_chroma_h;
    /* the offset into the 1 3 9 27 9 3 1 kernel of the first luma sample of a chroma group: centred by default, one
     * sample further for every side the chroma location pins the sample to */
    int wx = 4 - (1 << sw), wy = 4 - (1 << sh);
    const int left = chroma_location == AVCHROMA_LOC_TOPLEFT || chroma_location == AVCHROMA_LOC_LEFT ||
                     chroma_location == AVCHROMA_LOC_BOTTOMLEFT;
    const int vert = chroma_location == AVCHROMA_LOC_TOPLEFT || chroma_location == AVCHROMA_LOC_TOP ||
                     chroma_location == AVCHROMA_LOC_BOTTOMLEFT || chroma_location == AVCHROMA_LOC_BOTTOM;
    if (left) wx += (1 << sw) - 1;
    if (vert) wy += (1 << sh) - 1;
    static const uint32_t base[7] = {1, 3, 9, 27, 9, 3, 1};
    /* an even offset averages two neighbouring kernel taps (the sample sits between them) */
    for (int i = 0; i < 4; i++)
    {
        chroma_coeffs[0][i] = (base[i + wx] + base[i + wx + ((wx & 1) == 0)]) >> 1;
        chroma_coeffs[1][i] = (base[i + wy] + base[i + wy + ((wy & 1) == 0)]) >> 1;
    }
}

int av_image_get_linesize(int pix_fmt, int width, int plane)
{
    const AVPixFmtDescriptor *d = av_pix_fmt_desc_get(pix_fmt);
    if (d != NULL && d->nb_components == 3 && d->comp[1].plane == d->comp[2].plane)
    {
        /* semi-planar (libavutil/imgutils.c): the largest step of the plane's components times the plane's width in
         * samples; 0 for a plane the format does not have */
        if (plane < 0 || plane > 3)
            return -1;
        int step = 0;
        for (int c = 0; c < d->nb_components; c++)
            if (d->comp[c].plane == plane && d->comp[c].step > step)
                step = d->comp[c].step;
        return step * (plane == 1 || plane == 2 ? -((-width) >> d->log2_chroma_w) : width);
    }
    if (d == NULL || plane < 0 || plane >= d->nb_components)
        return -1;
    int w = width;
    if (plane == 1 || plane == 2)
        w = -((-width) >> d->log2_chroma_w);
    return w * (d->comp[plane].depth > 8 ? 2 : 1);
}

int av_get_cpu_flags(void)
{
#if defined(__SSE2__)
    return 0x0010; /* AV_CPU_FLAG_SSE2 */
#else
    return 0;
#endif
}

/* ------------------------------------------------------------------ */
/* logging / cpu count                                                  */
/* ------------------------------------------------------------------ */
static int g_log_level = 0;
static int g_cpu_count = 0;

void hb_shim_set_log_level(int level) { g_log_level = level; }
void hb_shim_set_cpu_count(int n)     { g_cpu_count = n; }

void hb_log(const char *fmt, ...)
{
    if (g_log_level < 0) return;
    va_list ap;
    va_start(ap, fmt);
    vfprintf(stderr, fmt, ap);
    va_end(ap);
    fputc('\n', stderr);
}

void hb_deep_log(int level, const char *fmt, ...)
{
    if (g_log_level < level) return;
    va_list ap;
    va_start(ap, fmt);
    vfprintf(stderr, fmt, ap);
    va_end(ap);
    fputc('\n', stderr);
}

void hb_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    fputs("ERROR: ", stderr);
    vfprintf(stderr, fmt, ap);
    va_end(ap);
    fputc('\n', stderr);
}

int hb_get_cpu_count(void)
{
    if (g_cpu_count > 0) return g_cpu_count;
    long n = sysconf(_SC_NPROCESSORS_ONLN);
    if (n < 1) n = 1;
    if (n > 128) n = 128;   /* ports.c caps the count as well */
    return (int)n;
}

/* ------------------------------------------------------------------ */
/* locks / conds / threads                                              */
/* ------------------------------------------------------------------ */
struct hb_lock_s   { pthread_mutex_t m; };
struct hb_cond_s   { pthread_cond_t  c; };
struct hb_thread_s { pthread_t t; thread_func_t *fn; void *arg; };

hb_lock_t *hb_lock_init(void)
{
    hb_lock_t *l = calloc(1, sizeof(*l));
    pthread_mutex_init(&l->m, NULL);
    return l;
}
void hb_lock_close(hb_lock_t **l)
{
    if (l == NULL || *l == NULL) return;
    pthread_mutex_destroy(&(*l)->m);
    free(*l);
    *l = NULL;
}
void hb_lock(hb_lock_t *l)   { pthread_mutex_lock(&l->m); }
void hb_unlock(hb_lock_t *l) { pthread_mutex_unlock(&l->m); }

hb_cond_t *hb_cond_init(void)
{
    hb_cond_t *c = calloc(1, sizeof(*c));
    pthread_cond_init(&c->c, NULL);
    return c;
}
void hb_cond_wait(hb_cond_t *c, hb_lock_t *l) { pthread_cond_wait(&c->c, &l->m); }
void hb_cond_signal(hb_cond_t *c)             { pthread_cond_signal(&c->c); }
void hb_cond_broadcast(hb_cond_t *c)          { pthread_cond_broadcast(&c->c); }
void hb_cond_close(hb_cond_t **c)
{
    if (c == NULL || *c == NULL) return;
    pthread_cond_destroy(&(*c)->c);
    free(*c);
    *c = NULL;
}

static void *thread_trampoline(void *p)
{
    hb_thread_t *t = p;
    t->fn(t->arg);
    return NULL;
}

hb_thread_t *hb_thread_init(const char *name, thread_func_t *fn, void *arg, int priority)
{
    (void)name; (void)priority;
    hb_thread_t *t = calloc(1, sizeof(*t));
    t->fn = fn;
    t->arg = arg;
    if (pthread_create(&t->t, NULL, thread_trampoline, t) != 0)
    {
        free(t);
        return NULL;
    }
    return t;
}

void hb_thread_close(hb_thread_t **t)
{
    if (t == NULL || *t == NULL) return;
    pthread_join((*t)->t, NULL);
    free(*t);
    *t = NULL;
}

void hb_yield(void) { sched_yield(); }

/* ------------------------------------------------------------------ */
/* buffers                                                              */
/* ------------------------------------------------------------------ */
static hb_shim_alloc_fn g_alloc = NULL;
static hb_shim_free_fn  g_free  = NULL;
static long g_alive = 0;
static int  g_zero  = 1;   /* zero-fill new buffers (deterministic oracle); libhb's pool does not */

void hb_shim_set_zero_buffers(int on) { g_zero = on; }

static void (*g_device_release)(void *) = NULL;
void hb_shim_set_device_release(void (*release)(void *storage)) { g_device_release = release; }
static void (*g_device_retain)(void *) = NULL;
void hb_shim_set_device_retain(void (*retain)(void *storage)) { g_device_retain = retain; }

void hb_shim_set_frame_allocator(hb_shim_alloc_fn a, hb_shim_free_fn f)
{
    g_alloc = a;
    g_free  = f;
}

long hb_shim_buffers_alive(void) { return __atomic_load_n(&g_alive, __ATOMIC_SEQ_CST); }

/* A small header in front of the payload remembers which allocator owns it. */
typedef struct { hb_shim_free_fn free_fn; void *base; } alloc_tag_t;

hb_buffer_t *hb_buffer_init(int size)
{
    hb_buffer_t *b = calloc(1, sizeof(*b));
    if (b == NULL) return NULL;
    b->size  = size;
    b->alloc = size;
    b->storage_type = STANDARD;
    if (size > 0)
    {
        /* payload 64-byte aligned like av_malloc'ed libhb buffers (fifo.c:404) */
        size_t total = (size_t)size + 64 + 128;
        void *base;
        hb_shim_free_fn ffn = NULL;
        if (g_alloc != NULL && g_free != NULL)
        {
            base = g_alloc(total);
            ffn  = g_free;
            if (base != NULL && g_zero) memset(base, 0, total);
        }
        else
        {
            base = g_zero ? calloc(1, total) : malloc(total);
        }
        if (base == NULL)
        {
            free(b);
            return NULL;
        }
        uintptr_t p = ((uintptr_t)base + sizeof(alloc_tag_t) + 63) & ~(uintptr_t)63;
        alloc_tag_t *tag = (alloc_tag_t *)(p - sizeof(alloc_tag_t));
        tag->free_fn = ffn;
        tag->base    = base;
        b->data = (uint8_t *)p;
        if (ffn != NULL) b->storage_type = HBCU_PINNED;
    }
    __atomic_add_fetch(&g_alive, 1, __ATOMIC_SEQ_CST);
    return b;
}

/* Decoder-style frame buffers for streaming benchmarks: a header over a payload somebody else keeps (libhb wraps
 * decoder memory the same way, hbffmpeg.c:182-239 -- closing the hb_buffer_t hands the memory back to its owner
 * instead of freeing it).  `release` replaces the allocator's free for this payload until reset with NULL. */
void *hb_shim_buffer_set_release(hb_buffer_t *b, hb_shim_free_fn release, hb_shim_free_fn *previous)
{
    if (b == NULL || b->data == NULL) return NULL;
    alloc_tag_t *tag = (alloc_tag_t *)(b->data - sizeof(alloc_tag_t));
    if (previous != NULL) *previous = tag->free_fn;
    tag->free_fn = release;
    return tag->base;
}

hb_buffer_t *hb_shim_frame_header_dup(const hb_buffer_t *master)
{
    hb_buffer_t *b = calloc(1, sizeof(*b));
    if (b == NULL) return NULL;
    *b = *master;
    b->next = NULL;
    __atomic_add_fetch(&g_alive, 1, __ATOMIC_SEQ_CST);
    return b;
}

hb_buffer_t *hb_buffer_eof_init(void)
{
    hb_buffer_t *b = hb_buffer_init(0);
    if (b != NULL) b->s.flags = HB_BUF_FLAG_EOF;
    return b;
}

void hb_buffer_init_planes(hb_buffer_t *b)
{
    uint8_t *data = b->data;
    for (int pp = 0; pp <= b->f.max_plane; pp++)
    {
        b->plane[pp].data   = data;
        b->plane[pp].stride = hb_image_stride(b->f.fmt, b->f.width, pp);
        b->plane[pp].width  = hb_image_width(b->f.fmt, b->f.width, pp);
        b->plane[pp].height = hb_image_height(b->f.fmt, b->f.height, pp);
        b->plane[pp].size   = b->plane[pp].stride * b->plane[pp].height;
        data += b->plane[pp].size;
    }
}

hb_buffer_t *hb_frame_buffer_init(int pix_fmt, int width, int height)
{
    const AVPixFmtDescriptor *desc = av_pix_fmt_desc_get(pix_fmt);
    if (desc == NULL) return NULL;

    int size = 0;
    int max_plane = 0;
    uint8_t seen[4] = {0, 0, 0, 0};
    for (int ii = 0; ii < desc->nb_components; ii++)
    {
        int pp = desc->comp[ii].plane;
        if (pp > max_plane) max_plane = pp;
        if (!seen[pp])
        {
            seen[pp] = 1;
            size += hb_image_stride(pix_fmt, width, pp) * hb_image_height(pix_fmt, height, pp);
        }
    }
    hb_buffer_t *buf = hb_buffer_init(size);
    if (buf == NULL) return NULL;
    buf->f.max_plane = max_plane;
    buf->s.type      = FRAME_BUF;
    buf->f.width     = width;
    buf->f.height    = height;
    buf->f.fmt       = pix_fmt;
    hb_buffer_init_planes(buf);
    return buf;
}

/* closes the whole ->next chain, like libhb (fifo.c:1037-1083) */
void hb_buffer_close(hb_buffer_t **_b)
{
    if (_b == NULL) return;
    hb_buffer_t *b = *_b;
    while (b != NULL)
    {
        hb_buffer_t *next = b->next;
        if (b->storage_type == HBCU_DEVICE)
        {
            /* device frame: plane[].data are device pointers, b->data is NULL (fifo.c:1016-1034 pattern) */
            if (b->storage != NULL && g_device_release != NULL) g_device_release(b->storage);
        }
        else if (b->data != NULL)
        {
            alloc_tag_t *tag = (alloc_tag_t *)(b->data - sizeof(alloc_tag_t));
            if (tag->free_fn != NULL) tag->free_fn(tag->base);
            else                      free(tag->base);
        }
        free(b);
        __atomic_sub_fetch(&g_alive, 1, __ATOMIC_SEQ_CST);
        b = next;
    }
    *_b = NULL;
}

void hb_buffer_copy_props(hb_buffer_t *dst, const hb_buffer_t *src)
{
    dst->s = src->s;   /* side data is FFmpeg-owned and not modelled by the shim */
}

hb_buffer_t *hb_buffer_dup(const hb_buffer_t *src)
{
    if (src == NULL) return NULL;
    if (src->storage_type == HBCU_DEVICE)
    {
        /* another reference on the same device frame */
        hb_buffer_t *ref = hb_buffer_init(0);
        if (ref == NULL || g_device_retain == NULL) { if (ref) hb_buffer_close(&ref); return NULL; }
        ref->f = src->f;
        hb_buffer_copy_props(ref, src);
        memcpy(ref->plane, src->plane, sizeof(ref->plane));
        ref->size = src->size;
        ref->storage_type = HBCU_DEVICE;
        ref->storage = src->storage;
        g_device_retain(ref->storage);
        return ref;
    }
    hb_buffer_t *buf = hb_buffer_init(src->size);
    if (buf == NULL) return NULL;
    buf->f = src->f;
    hb_buffer_copy_props(buf, src);
    if (buf->s.type == FRAME_BUF) hb_buffer_init_planes(buf);
    if (src->size > 0) memcpy(buf->data, src->data, src->size);
    return buf;
}

int hb_buffer_is_writable(const hb_buffer_t *buf)
{
    return buf->storage_type == STANDARD || buf->storage_type == HBCU_PINNED;
}

/* STANDARD buffers have no refcount in libhb either: shallow dup == dup (fifo.c:718-721) */
hb_buffer_t *hb_buffer_shallow_dup(const hb_buffer_t *src) { return hb_buffer_dup(src); }

int hb_buffer_copy(hb_buffer_t *dst, const hb_buffer_t *src)
{
    if (src == NULL || dst == NULL) return -1;
    if (dst->size < src->size) return -1;
    memcpy(dst->data, src->data, src->size);
    dst->f = src->f;
    hb_buffer_copy_props(dst, src);
    if (dst->s.type == FRAME_BUF) hb_buffer_init_planes(dst);
    return 0;
}

/* fifo.c:906-959.  NOTE the reference switches on `depth` after reducing it to
 * bytes-per-sample (1 or 2), so `case 8` never matches and the 16-bit variant
 * runs for every format.  Restated as-is: lapsharp reads the stride region. */
static void mirror_stride_words(uint8_t *data, int width, int height, int stride)
{
    uint16_t *d = (uint16_t *)data;
    stride /= 2;
    const int margin       = stride - width;
    const int margin_front = margin / 2;
    const int margin_back  = margin - margin_front;
    for (int yy = 0; yy < height; yy++)
    {
        int pos = yy * stride + width;
        for (int ii = 0; ii < margin_back; ii++)
            d[pos + ii] = d[pos - ii - 1];
        pos = (yy + 1) * stride - 1;
        for (int ii = 0; ii < margin_front; ii++)
            d[pos - ii] = d[pos + ii + 1];
    }
}

void hb_frame_buffer_mirror_stride(hb_buffer_t *buf)
{
    for (int pp = 0; pp <= buf->f.max_plane; pp++)
    {
        if (buf->plane[pp].data != NULL)
            mirror_stride_words(buf->plane[pp].data, buf->plane[pp].width,
                                buf->plane[pp].height, buf->plane[pp].stride);
    }
}

/* ------------------------------------------------------------------ */
/* buffer lists (singly linked through ->next; count/size bookkeeping)  */
/* ------------------------------------------------------------------ */
static hb_buffer_t *chain_end(hb_buffer_t *buf, int *count, int *size)
{
    hb_buffer_t *end = buf;
    *count = 1;
    *size  = buf->size;
    while (end->next != NULL)
    {
        end = end->next;
        *count += 1;
        *size  += end->size;
    }
    return end;
}

void hb_buffer_list_append(hb_buffer_list_t *list, hb_buffer_t *buf)
{
    if (buf == NULL) return;
    int count, size;
    hb_buffer_t *end = chain_end(buf, &count, &size);
    if (list->tail == NULL) list->head = buf;
    else                    list->tail->next = buf;
    list->tail   = end;
    list->count += count;
    list->size  += size;
}

void hb_buffer_list_prepend(hb_buffer_list_t *list, hb_buffer_t *buf)
{
    if (buf == NULL) return;
    int count, size;
    hb_buffer_t *end = chain_end(buf, &count, &size);
    if (list->tail == NULL) list->tail = end;
    else                    end->next = list->head;
    list->head   = buf;
    list->count += count;
    list->size  += size;
}

hb_buffer_t *hb_buffer_list_head(hb_buffer_list_t *list) { return list ? list->head : NULL; }
hb_buffer_t *hb_buffer_list_tail(hb_buffer_list_t *list) { return list ? list->tail : NULL; }

hb_buffer_t *hb_buffer_list_rem_head(hb_buffer_list_t *list)
{
    if (list == NULL || list->head == NULL) return NULL;
    hb_buffer_t *head = list->head;
    list->head = head->next;
    if (list->head == NULL) list->tail = NULL;
    list->count--;
    list->size -= head->size;
    head->next = NULL;
    return head;
}

hb_buffer_t *hb_buffer_list_rem_tail(hb_buffer_list_t *list)
{
    if (list == NULL || list->tail == NULL) return NULL;
    hb_buffer_t *tail = list->tail;
    if (list->head == tail)
    {
        list->head = list->tail = NULL;
        list->count = 0;
        list->size  = 0;
    }
    else
    {
        hb_buffer_t *p = list->head;
        while (p->next != tail) p = p->next;
        p->next = NULL;
        list->tail = p;
        list->count--;
        list->size -= tail->size;
    }
    tail->next = NULL;
    return tail;
}

hb_buffer_t *hb_buffer_list_rem(hb_buffer_list_t *list, hb_buffer_t *b)
{
    if (list == NULL) return NULL;
    if (b == list->head) return hb_buffer_list_rem_head(list);
    hb_buffer_t *a = list->head;
    while (a != NULL && a->next != b) a = a->next;
    if (a == NULL) return NULL;
    a->next = b->next;
    if (list->tail == b) list->tail = a;
    list->count--;
    list->size -= b->size;
    b->next = NULL;
    return b;
}

hb_buffer_t *hb_buffer_list_clear(hb_buffer_list_t *list)
{
    if (list == NULL) return NULL;
    hb_buffer_t *head = list->head;
    list->head = list->tail = NULL;
    list->count = 0;
    list->size  = 0;
    return head;
}

hb_buffer_t *hb_buffer_list_set(hb_buffer_list_t *list, hb_buffer_t *buf)
{
    if (list == NULL) return NULL;
    hb_buffer_t *old = list->head;
    list->head = buf;
    list->tail = NULL;
    list->count = 0;
    list->size  = 0;
    if (buf != NULL)
        list->tail = chain_end(buf, &list->count, &list->size);
    return old;
}

void hb_buffer_list_close(hb_buffer_list_t *list)
{
    hb_buffer_t *buf = hb_buffer_list_clear(list);
    hb_buffer_close(&buf);
}

int hb_buffer_list_count(hb_buffer_list_t *list) { return list ? list->count : 0; }
int hb_buffer_list_size(hb_buffer_list_t *list)  { return list ? list->size : 0; }

/* ------------------------------------------------------------------ */
/* settings dict: flat list of (key, string) pairs                      */
/* ------------------------------------------------------------------ */
typedef struct dict_entry_s
{
    char *key;
    char *val;
    struct dict_entry_s *next;
} dict_entry_t;

struct hb_value_s { dict_entry_t *head; };

hb_dict_t *hb_dict_init(void) { return calloc(1, sizeof(hb_dict_t)); }

void hb_dict_free(hb_dict_t **pd)
{
    if (pd == NULL || *pd == NULL) return;
    dict_entry_t *e = (*pd)->head;
    while (e != NULL)
    {
        dict_entry_t *n = e->next;
        free(e->key);
        free(e->val);
        free(e);
        e = n;
    }
    free(*pd);
    *pd = NULL;
}

static const dict_entry_t *dict_find(const hb_dict_t *d, const char *key)
{
    if (d == NULL || key == NULL) return NULL;
    for (const dict_entry_t *e = d->head; e != NULL; e = e->next)
        if (strcmp(e->key, key) == 0) return e;
    return NULL;
}

void hb_dict_set_string(hb_dict_t *d, const char *key, const char *value)
{
    for (dict_entry_t *e = d->head; e != NULL; e = e->next)
    {
        if (strcmp(e->key, key) == 0)
        {
            free(e->val);
            e->val = strdup(value);
            return;
        }
    }
    dict_entry_t *e = calloc(1, sizeof(*e));
    e->key  = strdup(key);
    e->val  = strdup(value);
    e->next = d->head;
    d->head = e;
}

void hb_dict_set_int(hb_dict_t *d, const char *key, int64_t value)
{
    char tmp[32];
    snprintf(tmp, sizeof(tmp), "%lld", (long long)value);
    hb_dict_set_string(d, key, tmp);
}

void hb_dict_set_double(hb_dict_t *d, const char *key, double value)
{
    char tmp[64];
    snprintf(tmp, sizeof(tmp), "%.17g", value);
    hb_dict_set_string(d, key, tmp);
}

int hb_dict_extract_int(int *dst, const hb_dict_t *dict, const char *key)
{
    const dict_entry_t *e = dict_find(dict, key);
    if (e == NULL || dst == NULL) return 0;
    /* hb_value_get_int on a string value parses it as a number */
    *dst = (int)strtod(e->val, NULL);
    return 1;
}

int hb_dict_extract_double(double *dst, const hb_dict_t *dict, const char *key)
{
    const dict_entry_t *e = dict_find(dict, key);
    if (e == NULL || dst == NULL) return 0;
    *dst = strtod(e->val, NULL);
    return 1;
}

int hb_dict_extract_bool(int *dst, const hb_dict_t *dict, const char *key)
{
    const dict_entry_t *e = dict_find(dict, key);
    if (e == NULL || dst == NULL) return 0;
    *dst = (!strcasecmp(e->val, "true") || !strcasecmp(e->val, "yes") || strtod(e->val, NULL) != 0);
    return 1;
}

int hb_dict_extract_string(char **dst, const hb_dict_t *dict, const char *key)
{
    const dict_entry_t *e = dict_find(dict, key);
    if (e == NULL || dst == NULL) return 0;
    *dst = strdup(e->val);
    return 1;
}

int hb_dict_extract_rational(hb_rational_t *dst, const hb_dict_t *dict, const char *key)
{
    const dict_entry_t *e = dict_find(dict, key);
    if (e == NULL || dst == NULL) return 0;
    const char *slash = strchr(e->val, '/');
    if (slash == NULL || !isdigit((unsigned char)e->val[0]) || !isdigit((unsigned char)slash[1]))
        return 0;
    /* the parts between the first two slashes must be whole numbers */
    const char *end2 = strchr(slash + 1, '/');
    char *num_end, *den_end;
    const int num = (int)strtol(e->val, &num_end, 0);
    const int den = (int)strtol(slash + 1, &den_end, 0);
    if (num_end != slash || (end2 ? den_end != end2 : *den_end != '\0')) return 0;
    dst->num = num;
    dst->den = den;
    return 1;
}

/* ------------------------------------------------------------------ */
/* lists, FIFOs, interjob                                               */
/* ------------------------------------------------------------------ */
struct hb_list_s { void **items; int count, cap; };

hb_list_t *hb_list_init(void) { return calloc(1, sizeof(hb_list_t)); }
int hb_list_count(const hb_list_t *l) { return l ? l->count : 0; }

void hb_list_add(hb_list_t *l, void *p)
{
    if (l == NULL || p == NULL) return;
    if (l->count == l->cap)
    {
        const int cap = l->cap ? 2 * l->cap : 16;
        void **items = realloc(l->items, sizeof(void *) * cap);
        if (items == NULL) return;
        l->items = items;
        l->cap = cap;
    }
    l->items[l->count++] = p;
}

void hb_list_rem(hb_list_t *l, void *p)
{
    if (l == NULL) return;
    for (int i = 0; i < l->count; i++)
        if (l->items[i] == p)
        {
            memmove(&l->items[i], &l->items[i + 1], sizeof(void *) * (l->count - i - 1));
            l->count--;
            return;
        }
}

void *hb_list_item(const hb_list_t *l, int i)
{
    return (l == NULL || i < 0 || i >= l->count) ? NULL : l->items[i];
}

void hb_list_close(hb_list_t **l)
{
    if (l == NULL || *l == NULL) return;
    free((*l)->items);
    free(*l);
    *l = NULL;
}

struct hb_fifo_s { hb_buffer_list_t list; };

hb_fifo_t *hb_fifo_init(int capacity, int thresh)
{
    (void)capacity; (void)thresh;
    return calloc(1, sizeof(hb_fifo_t));
}
int hb_fifo_size(hb_fifo_t *f) { return f ? hb_buffer_list_count(&f->list) : 0; }
void hb_fifo_push(hb_fifo_t *f, hb_buffer_t *b) { if (f && b) hb_buffer_list_append(&f->list, b); }
hb_buffer_t *hb_fifo_get(hb_fifo_t *f) { return f ? hb_buffer_list_rem_head(&f->list) : NULL; }
void hb_fifo_close(hb_fifo_t **f)
{
    if (f == NULL || *f == NULL) return;
    hb_buffer_list_close(&(*f)->list);
    free(*f);
    *f = NULL;
}

struct hb_handle_s { hb_interjob_t interjob; };
hb_interjob_t *hb_interjob_get(hb_handle_t *h) { return h ? &h->interjob : NULL; }

hb_dict_t *hb_parse_filter_settings(const char *settings)
{
    hb_dict_t *d = hb_dict_init();
    if (settings == NULL || d == NULL) return d;
    char *copy = strdup(settings);
    char *save = NULL;
    for (char *tok = strtok_r(copy, ":", &save); tok != NULL; tok = strtok_r(NULL, ":", &save))
    {
        char *eq = strchr(tok, '=');
        if (eq == NULL) continue;
        *eq = '\0';
        hb_dict_set_string(d, tok, eq + 1);
    }
    free(copy);
    return d;
}
