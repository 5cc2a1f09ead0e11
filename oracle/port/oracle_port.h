/* oracle_port.h -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C restatement of the reference's per-pixel algorithms for the hot path
 * (HandBrake libhb), written independently of the
 * reference's data flow (no integral images, no bordered copies) so that it
 * checks the *mathematics*: a mistake shared by the CUDA path and this port is
 * unlikely, and both are pinned against the compiled reference itself
 * (oracle/_ref/libhbref.so, tests/test_oracle.py) plus the golden digests in
 * tests/golden/.  Only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline leg may load this library.
 *
 * Frames are packed planar arrays (Y, U, V; row pitch = width * bps).
 */
#ifndef ORACLE_PORT_H
#define ORACLE_PORT_H
#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct
{
    double strength;      /* as given in the settings (before bit-depth scaling) */
    double origin_tune;
    int    patch_size;
    int    range;
    int    nframes;
    int    prefilter;     /* nlmeans.c:72-83 bit mask (mean 1/2, median 4/8, csm 16/32, reduce 256/512, edgeboost 1024, passthru 2048) */
} oracle_nlmeans_plane_params_t;

/* templates/nlmeans_template.c:103-543: the pre-denoised image the patch distances are taken from.  src, pre: w*h samples,
 * tightly packed.  Returns 1 when `pre` was produced, 0 when the mode has no filter bit (image_pre == image). */
int oracle_nlmeans_prefilter(const void *src, int w, int h, int depth, int filter_type, void *pre);

/* nlmeans.c:343-358: derived weight table for one plane */
void oracle_nlmeans_table(double strength, int patch_size, int depth,
                          float *weight_fact, int *diff_max, float exptable[128]);

/* templates/nlmeans_template.c:593-717 for one plane; frames[f] = current + f following,
 * each w*h samples, tightly packed; sample type uint8_t (depth 8) or uint16_t. */
void oracle_nlmeans_plane(const void *const *frames, int nframes, int w, int h, int depth,
                          const oracle_nlmeans_plane_params_t *pp, void *dst);

/* the same with the weight table given (weight_fact, diff_max, exptable[128] as in hbcu_nlmeans_plane_t); bypass = the
 * plane is copied (strength 0); stale_src = the source patches are read from the unfiltered image (see nlmeans_port.c) */
void oracle_nlmeans_plane_with_table(const void *const *frames, int nframes, int w, int h, int depth,
                                     int patch_size, int range, double origin_tune, int bypass, int prefilter,
                                     float weight_fact, int diff_max, const float *exptable, int stale_src, void *dst);

/* nlmeans.c:464-694 for a whole yuv420p clip: n_in packed frames in, n_in out
 * (look-ahead window, shrinking at EOF). */
int oracle_nlmeans_clip(const uint8_t *in, int n_in, int width, int height, int depth,
                        const oracle_nlmeans_plane_params_t pp[3], uint8_t *out);

/* ---------------- comb detect (libhb/comb_detect.c + templates/comb_detect_template.c) ---------------- */
typedef struct
{
    int mode;               /* bit0 gamma, bit1 filter (comb_detect.c:23-26) */
    int spatial_metric;
    int motion_threshold;   /* as given in the settings (before the depth shift) */
    int spatial_threshold;
    int filter_mode;        /* 1 classic, 2 erode-dilate */
    int block_threshold, block_width, block_height;
} oracle_comb_params_t;

/* one verdict: luma planes prev/cur/next (w*h samples each, tightly packed, uint8_t or uint16_t by depth);
 * mask_out / filtered_out (w*h bytes each) may be NULL.  Returns HB_COMB_NONE/LIGHT/HEAVY (0/1/2). */
int oracle_comb_detect(const void *prev, const void *cur, const void *next, int w, int h, int depth,
                       const oracle_comb_params_t *p, int force_exhaustive,
                       uint8_t *mask_out, uint8_t *filtered_out);

/* gamma table, comb_detect.c:1074-1081: (1<<depth) floats */
void oracle_comb_gamma_lut(int depth, float *out);

/* whole clip through comb_detect_work's ref window (comb_detect.c:1499-1584): verdict per input frame */
int oracle_comb_detect_clip(const uint8_t *in, int n_in, int width, int height, int depth,
                            const oracle_comb_params_t *p, uint8_t *verdicts);

/* ---------------- decomb (libhb/decomb.c + templates/decomb_template.c), EEDI2 excluded ---------------- */
#define ORACLE_DECOMB_YADIF     1
#define ORACLE_DECOMB_BLEND     2
#define ORACLE_DECOMB_CUBIC     4
#define ORACLE_DECOMB_EEDI2     8
#define ORACLE_DECOMB_BOB       16
#define ORACLE_DECOMB_SELECTIVE 32

/* one output field/frame of filter_{8,16} (decomb template :810-898) for all three planes.
 * prev/cur/next/dst: packed planar yuv420 frames; `mode` is the per-frame mode chosen by the
 * caller (decomb template :823-831) with the EEDI2 bit clear (oracle_decomb_clip handles EEDI2 modes); rows the reference leaves
 * unwritten (mode combinations without a line filter) stay as they are in dst. */
void oracle_decomb_field(const uint8_t *prev, const uint8_t *cur, const uint8_t *next, uint8_t *dst,
                         int width, int height, int depth, int filter_mode, int mode, int parity, int tff);

void oracle_decomb_field_eedi2(const uint8_t *prev, const uint8_t *cur, const uint8_t *next, const uint8_t *eedi, uint8_t *dst,
                               int width, int height, int depth, int mode, int parity, int tff);

/* EEDI2 (libhb/templates/eedi2_template.c via eedi2_interpolate_plane): a handle carries the edge-mask
 * state from field to field; one call interpolates field `!tff` of `cur` (packed planar) to a full frame */
void *oracle_eedi2_create(int width, int height, int depth, int mthresh, int vthresh, int lthresh, int dstr, int estr,
                          int nt, int maxd, int pp);
void  oracle_eedi2_destroy(void *e);
void  oracle_eedi2_field(void *e, const uint8_t *cur, int tff, uint8_t *out);
/* the four stages of postproc 2/3 (eedi2 template :1391-1904), exposed so that each can be pinned against the
 * reference's exported function of the same name (the reference's own chain races, see eedi2_port.c) */
void  oracle_eedi2_gaussian_blur1(const void *src, void *tmp, void *dst, int pitch, int height, int width, int bps);
void  oracle_eedi2_calc_derivatives(const void *src, int pitch, int height, int width, int *x2, int *y2, int *xy, int depth);
void  oracle_eedi2_gaussian_blur_sqrt2(const int *src, int *tmp, int *dst, int pitch, int height, int width);
void  oracle_eedi2_post_process_corner(const int *x2, const int *y2, const int *xy, int pitch, const void *mskp, void *dstp,
                                       int height, int width, int field, int depth);

/* whole clip through hb_decomb_work/process_frame (decomb.c:500-612).  flags/combed: per input
 * frame s.flags and s.combed; out must hold 2*n_in frames; returns the number of output frames.
 * out_src (may be NULL) receives the index of the input frame each output came from. */
int oracle_decomb_clip(const uint8_t *in, int n_in, const uint16_t *flags, const uint8_t *combed,
                       int width, int height, int depth, int mode, int parity_setting,
                       uint8_t *out, int *out_src);
/* same with the EEDI2 `postproc` setting (0..3; oracle_decomb_clip uses the default 1) */
int oracle_decomb_clip_pp(const uint8_t *in, int n_in, const uint16_t *flags, const uint8_t *combed,
                          int width, int height, int depth, int mode, int parity_setting, int postproc,
                          uint8_t *out, int *out_src);

/* ---------------- lapsharp (libhb/lapsharp.c) ---------------- */
/* one plane WITH its strides (bytes); kernel_id 0 lap, 1 isolap, 2 log, 3 isolog */
void oracle_lapsharp_plane(const void *src, void *dst, int width, int height, int stride_src, int stride_dst,
                           int depth, int kernel_id, double strength);

/* ---------------- unsharp / chroma_smooth (libhb/unsharp.c, libhb/chroma_smooth.c) ---------------- */
/* one tightly packed plane; smooth = 0 unsharp, 1 chroma_smooth (is_chroma = 0 copies the plane) */
void oracle_unsharp_plane(const void *src, void *dst, int w, int h, int depth, double strength, int size, int smooth, int is_chroma);
/* n packed yuv420p frames; strength/size per plane AFTER the cascade and defaults of unsharp.c:232-260 /
 * chroma_smooth.c:215-241 */
void oracle_unsharp_clip(const uint8_t *in, int n, int width, int height, int depth, const double strength[3], const int size[3],
                         int smooth, uint8_t *out);

/* ---------------- hqdn3d (libhb/denoise.c) ---------------- */
void oracle_hqdn3d_coef(int16_t *ct, int depth, double dist25);      /* hqdn3d_precalc_coef, table of 512 << LUT_BITS entries */
void oracle_hqdn3d_plane(const void *src, void *dst, uint16_t *ant, int *ant_valid, int w, int h, int depth,
                         const int16_t *spatial_tab, const int16_t *temporal_tab);
void oracle_hqdn3d_clip(const uint8_t *in, int n, int width, int height, int depth, const double strengths[6], uint8_t *out);

#ifdef __cplusplus
}
#endif
#endif
