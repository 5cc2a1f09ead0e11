/* hb_harness.h -- see hb_harness.c.  Plain-C interface for tests and bench. */
#ifndef HBCU_HB_HARNESS_H
#define HBCU_HB_HARNESS_H
#include "handbrake/handbrake.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct hb_harness_io_s
{
    /* input */
    int             pix_fmt, width, height;
    int             n_in;
    const uint8_t  *in;          /* n_in packed planar frames */
    const uint16_t *in_flags;    /* per-frame s.flags, NULL = progressive */
    const uint8_t  *in_combed;   /* per-frame s.combed, NULL = HB_COMB_NONE */
    /* output */
    uint8_t        *out;         /* out_capacity packed planar frames (may be NULL) */
    int             out_capacity;
    uint8_t        *out_combed;
    uint16_t       *out_flags;
    int64_t        *out_start;
    int64_t        *out_stop;
    double         *out_duration;
    int             n_out;
    int             n_dropped;   /* outputs beyond out_capacity */
    int             saw_eof;
    int             init_failed; /* bit k set: filter k's init() returned non-zero */
    int             vrate_num_out, vrate_den_out;
    /* input, optional (NULL / 0: frame i runs from i*3003 to (i+1)*3003 with new_chap = i, at 30000/1001, cfr 0) */
    const int64_t  *in_start;    /* per-frame s.start */
    const int64_t  *in_stop;     /* per-frame s.stop */
    const int      *in_new_chap; /* per-frame s.new_chap */
    int             vrate_num, vrate_den;   /* init->vrate */
    int             cfr;         /* init->cfr */
    int             collect_info;   /* fill info_text */
    /* output */
    int            *out_new_chap;
    int             cfr_out;     /* init->cfr after every filter's init() */
    char            info_text[128];   /* human_readable_desc of the last filter whose info() gives one */
    /* input, optional: init->geometry.par (0 / 0: 1:1) */
    int             par_num, par_den;
    /* output: init->geometry after every filter's init() (the geometry of the frames in `out`) */
    int             par_num_out, par_den_out;
    int             width_out, height_out;
} hb_harness_io_t;

size_t       hb_harness_frame_bytes(int pix_fmt, int w, int h);
hb_buffer_t *hb_harness_frame_from_packed(int pix_fmt, int w, int h, const uint8_t *src);
void         hb_harness_frame_to_packed(const hb_buffer_t *b, uint8_t *dst);
int hb_harness_run(hb_filter_object_t *proto, const char *settings, hb_harness_io_t *io);
int hb_harness_run_chain(int n_filters, hb_filter_object_t *const *protos,
                         const char *const *settings, hb_harness_io_t *io);

/* one motion metric object (hb_motion_metric ...) on one pair of frames: init() with the format and geometry, work() on
 * frames a and b (packed planar, see above) whose luma rows are `pad` bytes longer than the picture, close().  Returns
 * work()'s value; NaN when init() fails. */
float hb_harness_motion_metric(hb_motion_metric_object_t *proto, int pix_fmt, int w, int h, int pad,
                               const uint8_t *a, const uint8_t *b);

/* ---- a stand-in for libhb's render_sub filter (rendersub.c): burns a per-frame schedule of overlays into the frames
 * through a blend object (hb_blend, hb_blend_cuda ...), calling its init / work / close the way rendersub does ---- */
typedef struct hb_harness_overlay_s
{
    int            frame;             /* index of the input frame it is shown on */
    int            x, y, width, height;
    const uint8_t *yuva;              /* the overlay's planes Y, Cb, Cr, A back to back, rows packed at the plane widths */
} hb_harness_overlay_t;

typedef struct hb_harness_blend_s
{
    /* input */
    hb_blend_object_t          *blend;
    int                         overlay_pix_fmt, chroma_location;
    int                         n_overlays;
    const hb_harness_overlay_t *overlays;     /* ordered by frame; within a frame, list order */
    int                         n_changed;
    const int                  *changed;      /* per frame; frames past n_changed pass changed = 1 */
    int                         guard_x, guard_y;   /* > 0: host frames get this many spare samples / rows on every side
                                                     * around the picture while the blend object works on them */
    /* output */
    int                         guard_damaged;  /* frames where a sample outside the picture was written */
    int                         same_buffer;    /* frames whose work() handed back the buffer it was given */
    int                         frames;
} hb_harness_blend_t;

/* the schedule the next chains' hb_filter_render_sub_harness instances use (the caller keeps it alive) */
void hb_harness_set_blend(hb_harness_blend_t *cfg);
extern hb_filter_object_t hb_filter_render_sub_harness;

#ifdef __cplusplus
}
#endif
#endif
