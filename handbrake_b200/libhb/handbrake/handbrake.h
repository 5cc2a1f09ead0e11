/* handbrake/handbrake.h -- minimal libhb-compatible environment ("the shim").
 *
 * Purpose.  The CUDA filter objects in this directory (nlmeans_cuda.c, ...)
 * are written against libhb's own plugin interface so they can be dropped into
 * libhb/ unchanged.  libhb itself cannot be built in this image (FFmpeg,
 * jansson, x264 ... are fetched from the network by the reference's build),
 * so this header supplies, field for field, the part of libhb's interface the
 * video-filter hot path touches.  It is NOT a copy of the reference headers:
 * only the members/semantics the filters use are restated, each with the
 * reference location it mirrors.  The same header is used by oracle/Makefile
 * to compile the reference's own filter sources unmodified (they
 * `#include "handbrake/handbrake.h"`, which resolves here first).
 *
 * Mirrors (reference: HandBrake's libhb):
 *   hb_buffer_t, hb_buffer_settings_s, hb_image_format_s  handbrake/internal.h:63-165
 *   hb_image_stride/width/height                          handbrake/internal.h:220-254
 *   hb_filter_object_t, hb_filter_init_t, HB_FILTER_*     handbrake/common.h:1628-1711
 *   filter id enum                                        handbrake/common.h:1729-1778
 *   hb_buffer_list_t                                      handbrake/common.h:115-134
 */
#ifndef HBCU_SHIM_HANDBRAKE_H
#define HBCU_SHIM_HANDBRAKE_H

#include <stdint.h>
#include <stddef.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>
#include <math.h>
#include <limits.h>
#include <inttypes.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef __LIBHB__
#define __LIBHB__ 1
#endif

#if defined(__x86_64__) || defined(__i386__)
#define ARCH_X86 1
#define ARCH_X86_64 1
#endif

#define HB_NORMAL_PRIORITY 0
#define HB_LOW_PRIORITY    0

#ifndef MIN
#define MIN(a, b) (((a) < (b)) ? (a) : (b))
#endif
#ifndef MAX
#define MAX(a, b) (((a) > (b)) ? (a) : (b))
#endif
#ifndef ABS
#define ABS(a) ((a) > 0 ? (a) : (-(a)))
#endif
#define MULTIPLE_MOD_UP(a, b) ((b) * (((a) + (b) - 1) / (b)))
#define MULTIPLE_MOD_DOWN(a, b) ((b) * ((a) / (b)))
#define HB_ALIGN(x, a) (((x) + (a) - 1) & ~((a) - 1))

/* settings_template regex fragments (handbrake/common.h) */
#define HB_INT_REG   "(\\+|-)?[0-9]+"
#define HB_FLOAT_REG "(\\+|-)?[0-9]*(\\.[0-9]+)?"
#define HB_BOOL_REG  "(yes|no|true|false|[01])"
#define HB_ALL_REG   "."

/* ---- pixel formats: the subset of FFmpeg's AVPixelFormat the path needs ---- */
enum AVPixelFormat
{
    AV_PIX_FMT_NONE        = -1,
    AV_PIX_FMT_YUV420P     = 0,
    AV_PIX_FMT_YUV422P     = 4,
    AV_PIX_FMT_YUV444P     = 5,
    AV_PIX_FMT_GRAY8       = 8,
    AV_PIX_FMT_YUV420P10LE = 62,
    AV_PIX_FMT_YUV422P10LE = 64,
    AV_PIX_FMT_YUV444P10LE = 68,
    AV_PIX_FMT_YUV420P12LE = 123,
    AV_PIX_FMT_YUV420P16LE = 47,
    /* FFmpeg's hardware pixel format for CUDA frames.  libhb signals hardware frames through
     * hb_filter_init_t.hw_pix_fmt / job->hw_pix_fmt (nvenc_common.c:329-336); the value is only ever compared */
    AV_PIX_FMT_CUDA        = 117,
    /* the overlay formats of libhb's subtitle renderer (rendersub.c): planar YUV with an 8-bit alpha plane */
    AV_PIX_FMT_YUVA420P    = 33,
    AV_PIX_FMT_YUVA422P    = 78,
    AV_PIX_FMT_YUVA444P    = 79,
    /* the semi-planar 4:2:0 formats NVDEC decodes into (AVHWFramesContext.sw_format): Y, then one plane of
     * interleaved Cb/Cr pairs; P010 keeps its 10 bits in the high bits of each 16-bit sample */
    AV_PIX_FMT_NV12        = 23,
    AV_PIX_FMT_P010LE      = 158,
    AV_PIX_FMT_P016LE      = 169,
};
#define AV_PIX_FMT_YUV420P10 AV_PIX_FMT_YUV420P10LE
#define AV_PIX_FMT_YUV420P12 AV_PIX_FMT_YUV420P12LE
#define AV_PIX_FMT_P010      AV_PIX_FMT_P010LE
#define AV_PIX_FMT_P016      AV_PIX_FMT_P016LE

/* FFmpeg's enum AVChromaLocation (libavutil/pixfmt.h) */
enum AVChromaLocation
{
    AVCHROMA_LOC_UNSPECIFIED = 0,
    AVCHROMA_LOC_LEFT        = 1,
    AVCHROMA_LOC_CENTER      = 2,
    AVCHROMA_LOC_TOPLEFT     = 3,
    AVCHROMA_LOC_TOP         = 4,
    AVCHROMA_LOC_BOTTOMLEFT  = 5,
    AVCHROMA_LOC_BOTTOM      = 6,
    AVCHROMA_LOC_NB
};

typedef struct AVComponentDescriptor
{
    int plane;
    int step;
    int offset;
    int shift;
    int depth;
} AVComponentDescriptor;

typedef struct AVPixFmtDescriptor
{
    const char *name;
    uint8_t nb_components;
    uint8_t log2_chroma_w;
    uint8_t log2_chroma_h;
    uint64_t flags;
    AVComponentDescriptor comp[4];
} AVPixFmtDescriptor;

/* AVPixFmtDescriptor.flags bits (libavutil/pixdesc.h) */
#define AV_PIX_FMT_FLAG_BE  (1 << 0)
#define AV_PIX_FMT_FLAG_RGB (1 << 5)

const AVPixFmtDescriptor *av_pix_fmt_desc_get(int pix_fmt);
int av_image_get_linesize(int pix_fmt, int width, int plane);
/* number of distinct planes of the format (libavutil/pixdesc.c), < 0 for an unknown format */
int av_pix_fmt_count_planes(int pix_fmt);
/* libavutil/pixdesc.c: the format of a descriptor name (or of the name with the native-endian suffix "le" appended,
 * so "p010" is p010le and "yuv420p10" is yuv420p10le), AV_PIX_FMT_NONE for a name the table does not know; and the
 * descriptor name of a format, NULL for an unknown one */
enum AVPixelFormat av_get_pix_fmt(const char *name);
const char *av_get_pix_fmt_name(enum AVPixelFormat pix_fmt);

typedef struct AVRational { int num; int den; } AVRational;
typedef struct AVChannelLayout { int order; int nb_channels; uint64_t mask; void *opaque; } AVChannelLayout;

/* ---- opaque libhb types the filters only pass around ---- */
typedef struct hb_job_s       hb_job_t;
typedef struct hb_fifo_s      hb_fifo_t;
typedef struct hb_subtitle_s  hb_subtitle_t;
typedef struct hb_thread_s    hb_thread_t;
typedef struct hb_lock_s      hb_lock_t;
typedef struct hb_cond_s      hb_cond_t;
typedef struct hb_list_s      hb_list_t;
typedef struct hb_value_s     hb_value_t;
typedef hb_value_t            hb_dict_t;
typedef hb_value_t            hb_value_array_t;
typedef void (thread_func_t)(void *);

typedef struct hb_filter_object_s  hb_filter_object_t;
typedef struct hb_filter_private_s hb_filter_private_t;   /* handbrake/hbtypes.h:42 */
typedef struct hb_buffer_s         hb_buffer_t;
typedef struct hb_buffer_settings_s hb_buffer_settings_t;
typedef struct hb_image_format_s   hb_image_format_t;
typedef struct hb_buffer_list_s    hb_buffer_list_t;

typedef struct hb_rational_s { int num; int den; } hb_rational_t;
typedef struct hb_geometry_s { int width; int height; hb_rational_t par; } hb_geometry_t;

/* ---- hb_buffer_t (handbrake/internal.h:63-165) ---- */
struct hb_buffer_settings_s
{
    enum { OTHER_BUF, AUDIO_BUF, VIDEO_BUF, SUBTITLE_BUF, FRAME_BUF } type;

    int           id;
    int64_t       start;
    double        duration;
    int64_t       stop;
    int64_t       renderOffset;
    int64_t       pcr;
    int           scr_sequence;
    int           split;
    uint8_t       discontinuity;
    int           new_chap;
    uint8_t       frametype;

#define PIC_FLAG_TOP_FIELD_FIRST    0x0008
#define PIC_FLAG_PROGRESSIVE_FRAME  0x0010
#define PIC_FLAG_REPEAT_FIRST_FIELD 0x0100
#define PIC_FLAG_REPEAT_FRAME       0x0200
#define HB_BUF_FLAG_EOF             0x0400
#define HB_BUF_FLAG_EOS             0x0800
    uint16_t      flags;

#define HB_COMB_NONE  0
#define HB_COMB_LIGHT 1
#define HB_COMB_HEAVY 2
    uint8_t       combed;
};

struct hb_image_format_s
{
    int x, y, width, height, fmt;
    int color_prim, color_transfer, color_matrix, color_range, chroma_location;
    int max_plane;
    int window_width, window_height;
};

/* storage_type gains the device backings:
 * HBCU_PINNED  : data lives in cudaHostAlloc'ed (page-locked) host memory
 * HBCU_DEVICE  : plane[].data are device pointers; storage = owning context */
struct hb_buffer_s
{
    int           size;
    int           alloc;
    uint8_t     * data;
    int           offset;

    hb_buffer_settings_t s;
    hb_image_format_t    f;

    struct buffer_plane
    {
        uint8_t * data;
        int       stride;
        int       width;
        int       height;
        int       size;
    } plane[4];

    void * storage;
    enum { STANDARD, AVFRAME, COREMEDIA, HBCU_PINNED, HBCU_DEVICE } storage_type;

    hb_buffer_t * palette;
    void       ** side_data;
    int           nb_side_data;

    hb_buffer_t * next;
};

struct hb_buffer_list_s
{
    hb_buffer_t *head;
    hb_buffer_t *tail;
    int count;
    int size;
};

hb_buffer_t * hb_buffer_init(int size);
hb_buffer_t * hb_buffer_eof_init(void);
hb_buffer_t * hb_frame_buffer_init(int pix_fmt, int w, int h);
void          hb_frame_buffer_mirror_stride(hb_buffer_t *buf);
void          hb_buffer_init_planes(hb_buffer_t *b);
void          hb_buffer_close(hb_buffer_t **);
hb_buffer_t * hb_buffer_dup(const hb_buffer_t *src);
hb_buffer_t * hb_buffer_shallow_dup(const hb_buffer_t *src);
int           hb_buffer_copy(hb_buffer_t *dst, const hb_buffer_t *src);
/* fifo.c:624-639: may the holder write into the buffer's planes?  Host buffers (STANDARD, HBCU_PINNED) yes; an
 * HBCU_DEVICE buffer never -- a device frame is written once, by its producer */
int           hb_buffer_is_writable(const hb_buffer_t *buf);
void          hb_buffer_copy_props(hb_buffer_t *dst, const hb_buffer_t *src);

/* allocator hook: lets the CUDA filters make every frame buffer page-locked
 * ("hb_buffer_t gains pinned backing").  NULL hooks = plain calloc/free. */
typedef void *(*hb_shim_alloc_fn)(size_t);
typedef void  (*hb_shim_free_fn)(void *);
void hb_shim_set_frame_allocator(hb_shim_alloc_fn a, hb_shim_free_fn f);
/* new buffers are zero-filled by default (deterministic oracle runs); libhb's own pool hands out
 * recycled memory, so throughput measurements switch this off */
void hb_shim_set_zero_buffers(int on);
/* HBCU_DEVICE buffers: hb_buffer_close() hands b->storage to this hook (fifo.c:1037-1083 does the same for
 * AVFRAME / COREMEDIA storage); set by hbcu_device_frames.c */
void hb_shim_set_device_release(void (*release)(void *storage));
/* hb_buffer_shallow_dup()/hb_buffer_dup() of an HBCU_DEVICE buffer take another reference on the same device frame
 * (frames are written once by their producer, then only read), like av_frame_ref for AVFRAME storage (fifo.c:718-760) */
void hb_shim_set_device_retain(void (*retain)(void *storage));
/* statistics used by the tests (leak check: HB_BUFFER_DEBUG analogue, fifo.c:137-278) */
long hb_shim_buffers_alive(void);
/* decoder-style buffers (streaming benchmarks): see hb_runtime.c */
void        *hb_shim_buffer_set_release(hb_buffer_t *b, hb_shim_free_fn release, hb_shim_free_fn *previous);
hb_buffer_t *hb_shim_frame_header_dup(const hb_buffer_t *master);

void hb_buffer_list_append(hb_buffer_list_t *list, hb_buffer_t *buf);
void hb_buffer_list_prepend(hb_buffer_list_t *list, hb_buffer_t *buf);
hb_buffer_t *hb_buffer_list_head(hb_buffer_list_t *list);
hb_buffer_t *hb_buffer_list_rem_head(hb_buffer_list_t *list);
hb_buffer_t *hb_buffer_list_tail(hb_buffer_list_t *list);
hb_buffer_t *hb_buffer_list_rem_tail(hb_buffer_list_t *list);
hb_buffer_t *hb_buffer_list_rem(hb_buffer_list_t *list, hb_buffer_t *b);
hb_buffer_t *hb_buffer_list_clear(hb_buffer_list_t *list);
hb_buffer_t *hb_buffer_list_set(hb_buffer_list_t *list, hb_buffer_t *buf);
void hb_buffer_list_close(hb_buffer_list_t *list);
int hb_buffer_list_count(hb_buffer_list_t *list);
int hb_buffer_list_size(hb_buffer_list_t *list);

static inline int hb_image_stride(int pix_fmt, int width, int plane)
{
    int linesize = av_image_get_linesize(pix_fmt, width, plane);
    return MULTIPLE_MOD_UP(linesize, 64);
}

static inline int hb_image_width(int pix_fmt, int width, int plane)
{
    const AVPixFmtDescriptor *desc = av_pix_fmt_desc_get(pix_fmt);
    if (desc != NULL && (plane == 1 || plane == 2))
        width = -((-width) >> desc->log2_chroma_w);
    return width;
}

static inline int hb_image_height(int pix_fmt, int height, int plane)
{
    const AVPixFmtDescriptor *desc = av_pix_fmt_desc_get(pix_fmt);
    if (desc != NULL && (plane == 1 || plane == 2))
        height = -((-height) >> desc->log2_chroma_h);
    return height;
}

static inline void hb_image_copy_plane(uint8_t *restrict dst, const uint8_t *restrict src,
                                       const int stride_dst, const int stride_src, const int height)
{
    if (src == dst) return;
    if (stride_src == stride_dst)
    {
        memcpy(dst, src, (size_t)stride_dst * height);
        return;
    }
    const int size = stride_src < stride_dst ? ABS(stride_src) : stride_dst;
    for (int yy = 0; yy < height; yy++)
    {
        memcpy(dst, src, size);
        dst += stride_dst;
        src += stride_src;
    }
}

/* ---- filter plugin ABI (handbrake/common.h:1628-1711) ---- */
#define HB_FILTER_OK      0
#define HB_FILTER_DELAY   1
#define HB_FILTER_FAILED  2
#define HB_FILTER_DROP    3
#define HB_FILTER_DONE    4

typedef struct hb_filter_init_s
{
    hb_job_t      * job;
    int             pix_fmt;
    int             hw_pix_fmt;
    void          * hw_frames_ctx;
    int             color_prim;
    int             color_transfer;
    int             color_matrix;
    int             color_range;
    int             chroma_location;
    hb_geometry_t   geometry;
    int             crop[4];
    int             grayscale;
    hb_rational_t   vrate;
    int             cfr;
    hb_rational_t   time_base;
    int             samplerate;
    int             sample_fmt;
    AVChannelLayout ch_layout;
} hb_filter_init_t;

typedef struct hb_filter_info_s
{
    char             * human_readable_desc;
    hb_filter_init_t   output;
} hb_filter_info_t;

struct hb_filter_object_s
{
    int                   id;
    int                   enforce_order;
    int                   skip;
    int                   aliased;
    char                * name;
    char                * short_name;
    hb_dict_t           * settings;

    int                (* init)       (hb_filter_object_t *, hb_filter_init_t *);
    int                (* init_thread)(hb_filter_object_t *, int);
    int                (* post_init)  (hb_filter_object_t *, hb_job_t *);
    int                (* work)       (hb_filter_object_t *, hb_buffer_t **, hb_buffer_t **);
    int                (* work_thread)(hb_filter_object_t *, hb_buffer_t **, hb_buffer_t **, int);
    void               (* close)      (hb_filter_object_t *);
    hb_filter_info_t * (* info)       (hb_filter_object_t *);

    const char          * settings_template;

    hb_fifo_t           * fifo_in;
    hb_fifo_t           * fifo_out;
    hb_subtitle_t       * subtitle;
    hb_filter_private_t * private_data;
    hb_thread_t         * thread;
    volatile int        * done;
    int                   status;
    int                   chapter_val;
    int64_t               chapter_time;
    hb_filter_object_t  * sub_filter;
};

/* filter ids: same order as handbrake/common.h:1729-1778 (defines chain order) */
enum
{
    HB_FILTER_INVALID = 0,
    HB_FILTER_FIRST = 1,
    HB_FILTER_ADAPTER_VT,
    HB_FILTER_DETELECINE,
    HB_FILTER_COMB_DETECT,
    HB_FILTER_COMB_DETECT_VT,
    HB_FILTER_DECOMB,
    HB_FILTER_YADIF,
    HB_FILTER_YADIF_VT,
    HB_FILTER_BWDIF,
    HB_FILTER_BWDIF_VT,
    HB_FILTER_VFR,
    HB_FILTER_DEBLOCK,
    HB_FILTER_DEBAND,
    HB_FILTER_DENOISE,
    HB_FILTER_HQDN3D = HB_FILTER_DENOISE,
    HB_FILTER_BM3D,
    HB_FILTER_NLMEANS,
    HB_FILTER_CHROMA_SMOOTH,
    HB_FILTER_CHROMA_SMOOTH_VT,
    HB_FILTER_ROTATE,
    HB_FILTER_ROTATE_VT,
    HB_FILTER_RENDER_SUB,
    HB_FILTER_CROP_SCALE,
    HB_FILTER_CROP_SCALE_VT,
    HB_FILTER_LAPSHARP,
    HB_FILTER_LAPSHARP_VT,
    HB_FILTER_UNSHARP,
    HB_FILTER_UNSHARP_VT,
    HB_FILTER_GRAYSCALE,
    HB_FILTER_GRAYSCALE_VT,
    HB_FILTER_PAD,
    HB_FILTER_PAD_VT,
    HB_FILTER_COLORSPACE,
    HB_FILTER_FORMAT,
    HB_FILTER_RPU,
    HB_FILTER_AVFILTER,
    HB_FILTER_LAST,
    HB_FILTER_MT_FRAME
};

/* ---- settings dict (hb_dict.c:538-605 semantics: 1 = key present) ---- */
hb_dict_t *hb_dict_init(void);
void       hb_dict_free(hb_dict_t **);
void       hb_dict_set_string(hb_dict_t *, const char *key, const char *value);
void       hb_dict_set_int(hb_dict_t *, const char *key, int64_t value);
void       hb_dict_set_double(hb_dict_t *, const char *key, double value);
int hb_dict_extract_int(int *dst, const hb_dict_t *dict, const char *key);
int hb_dict_extract_double(double *dst, const hb_dict_t *dict, const char *key);
int hb_dict_extract_bool(int *dst, const hb_dict_t *dict, const char *key);
int hb_dict_extract_string(char **dst, const hb_dict_t *dict, const char *key);
/* "key=value:key=value" -> dict (hb_parse_filter_settings, common.c) */
hb_dict_t *hb_parse_filter_settings(const char *settings);

/* ---- ports.c: threads / locks / logging ---- */
void hb_log(const char *fmt, ...) __attribute__((format(printf, 1, 2)));
void hb_deep_log(int level, const char *fmt, ...) __attribute__((format(printf, 2, 3)));
void hb_error(const char *fmt, ...) __attribute__((format(printf, 1, 2)));
void hb_shim_set_log_level(int level);   /* <0 silences hb_log */

int          hb_get_cpu_count(void);
void         hb_shim_set_cpu_count(int n);   /* 0 = autodetect */
hb_lock_t  * hb_lock_init(void);
void         hb_lock_close(hb_lock_t **);
void         hb_lock(hb_lock_t *);
void         hb_unlock(hb_lock_t *);
hb_cond_t  * hb_cond_init(void);
void         hb_cond_wait(hb_cond_t *, hb_lock_t *);
void         hb_cond_signal(hb_cond_t *);
void         hb_cond_broadcast(hb_cond_t *);
void         hb_cond_close(hb_cond_t **);
hb_thread_t *hb_thread_init(const char *name, thread_func_t *fn, void *arg, int priority);
void         hb_thread_close(hb_thread_t **);
void         hb_yield(void);                 /* ports.h:189 */

/* sub-filter registry used by mt_frame_filter.c (common.c:5331-5517) */
hb_filter_object_t *hb_filter_get(int filter_id);
hb_filter_object_t *hb_filter_init(int filter_id);
void                hb_filter_close(hb_filter_object_t **);

extern hb_filter_object_t hb_filter_nlmeans;
extern hb_filter_object_t hb_filter_comb_detect;
extern hb_filter_object_t hb_filter_decomb;
/* libavutil helpers libhb/denoise.c uses */
#ifndef FFMIN
#define FFMIN(a, b) ((a) > (b) ? (b) : (a))
#define FFMAX(a, b) ((a) > (b) ? (a) : (b))
#endif
#ifndef AV_CEIL_RSHIFT
#define AV_CEIL_RSHIFT(a, b) (-((-(a)) >> (b)))
#endif
static inline void *av_malloc(size_t size) { void *p = NULL; if (posix_memalign(&p, 64, size ? size : 1) != 0) return NULL; return p; }
static inline void av_freep(void *arg) { void **pp = (void **)arg; free(*pp); *pp = NULL; }

/* ---- blend objects: composite a list of YUVA overlays onto a frame (handbrake/common.h:1813-1826) ---- */
typedef struct hb_blend_object_s  hb_blend_object_t;
typedef struct hb_blend_private_s hb_blend_private_t;   /* handbrake/hbtypes.h:46-47 */
struct hb_blend_object_s
{
    char                * name;
    int                (* init)  (hb_blend_object_t *, int in_width, int in_height, int in_pix_fmt, int in_chroma_location,
                                  int in_color_range, int overlay_pix_fmt);
    hb_buffer_t *      (* work)  (hb_blend_object_t *, hb_buffer_t *, hb_buffer_list_t *, int changed);
    void               (* close) (hb_blend_object_t *);
    hb_blend_private_t  * private_data;
};
extern hb_blend_object_t hb_blend;

/* common.c:7054-7091: the per-position weights [0][x] / [1][y] of the luma samples that make up one chroma sample,
 * from the format's subsampling and the chroma location */
void hb_compute_chroma_smoothing_coefficient(uint32_t chroma_coeffs[2][4], int pix_fmt, int chroma_location);

/* ---- what the framerate shaper (vfr.c) and its motion metric (motion_metric.c) use ---- */
#define HB_RATIONAL_REG "([0-9]+/[0-9]+)"                  /* handbrake/common.h */
/* "num/den" (hb_dict.c: both parts digits only); 1 = key present and well-formed */
int hb_dict_extract_rational(hb_rational_t *dst, const hb_dict_t *dict, const char *key);

/* generic pointer list (common.c hb_list_*) */
hb_list_t *hb_list_init(void);
int        hb_list_count(const hb_list_t *l);
void       hb_list_add(hb_list_t *l, void *p);
void       hb_list_rem(hb_list_t *l, void *p);
void      *hb_list_item(const hb_list_t *l, int i);
void       hb_list_close(hb_list_t **l);

/* buffer FIFO (fifo.c hb_fifo_*), single-threaded and never blocking: push appends, get returns NULL when empty,
 * close frees what is left */
hb_fifo_t   *hb_fifo_init(int capacity, int thresh);
int          hb_fifo_size(hb_fifo_t *f);
void         hb_fifo_push(hb_fifo_t *f, hb_buffer_t *b);
hb_buffer_t *hb_fifo_get(hb_fifo_t *f);
void         hb_fifo_close(hb_fifo_t **f);

/* the job's handle and the statistics one pass leaves for the next (handbrake/handbrake.h hb_interjob_t, hb.c) */
typedef struct hb_handle_s hb_handle_t;
struct hb_job_s { hb_handle_t *h; };
typedef struct hb_interjob_s
{
    int           sequence_id;
    int           frame_count;
    int           out_frame_count;
    int64_t       total_time;
    hb_rational_t vrate;
} hb_interjob_t;
hb_interjob_t *hb_interjob_get(hb_handle_t *h);

/* motion metric objects (handbrake/common.h:1799-1811): the frame distance vfr.c picks frames to drop by */
typedef struct hb_motion_metric_object_s  hb_motion_metric_object_t;
typedef struct hb_motion_metric_private_s hb_motion_metric_private_t;   /* handbrake/hbtypes.h:44-45 */
struct hb_motion_metric_object_s
{
    char                       * name;
    int                       (* init)  (hb_motion_metric_object_t *, hb_filter_init_t *);
    float                     (* work)  (hb_motion_metric_object_t *, hb_buffer_t *, hb_buffer_t *);
    void                      (* close) (hb_motion_metric_object_t *);
    hb_motion_metric_private_t * private_data;
};
extern hb_motion_metric_object_t hb_motion_metric;
extern hb_filter_object_t hb_filter_vfr;

extern hb_filter_object_t hb_filter_denoise;
extern hb_filter_object_t hb_filter_detelecine;
extern hb_filter_object_t hb_filter_lapsharp;
extern hb_filter_object_t hb_filter_unsharp;
extern hb_filter_object_t hb_filter_chroma_smooth;
extern hb_filter_object_t hb_filter_mt_frame;

#ifdef __cplusplus
}
#endif

#endif /* HBCU_SHIM_HANDBRAKE_H */
