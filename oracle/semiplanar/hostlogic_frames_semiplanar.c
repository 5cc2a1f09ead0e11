/* hostlogic_frames_semiplanar.c -- TEST INFRASTRUCTURE: the device-frame stand-ins of port/hostlogic_frames.c for
 * libhostlogic_semiplanar.so (semiplanar.mk), extended to two-plane frames.
 *
 * A semi-planar frame (NV12, P010, P016: Y, then one plane of Cb/Cr pairs) has no third plane; include/hbcu.h passes it
 * as 0 rows of 0 bytes.  port/hostlogic_frames.c is compiled here as it is, with its frame_alloc renamed: the stand-ins
 * of the planar libraries stay what they are, and this library's frame_alloc accepts the absent plane, keeps stride 0
 * for it and hands out a NULL plane pointer, like hbcu_frame_alloc.  Wrapped frames, the transfers and the accessors
 * need nothing more: an absent plane is 0 rows long and its pointer is the caller's NULL.  Never linked into the
 * product.
 */
#define oracle_hbcu_frame_alloc hostlogic_frame_alloc_three_planes
#include "../port/hostlogic_frames.c"
#undef oracle_hbcu_frame_alloc

int oracle_hbcu_frame_alloc(hbcu_frame_t **out, int device, const int row_bytes[3], const int rows[3], const int strides[3])
{
    const int two_planes = rows[2] == 0 && row_bytes[2] == 0;
    size_t bytes = 0;
    for (int p = 0; p < (two_planes ? 2 : 3); p++)
    {
        if (row_bytes[p] <= 0 || rows[p] <= 0 || strides[p] < row_bytes[p] || strides[p] % 16)
        {
            oracle_hostlogic_set_error("frame_alloc: bad geometry of plane %d", p);
            return -1;
        }
        bytes += (size_t)strides[p] * rows[p];
    }
    struct hbcu_frame_s *f = calloc(1, sizeof(*f));
    f->refs = 1;
    f->device = device;
    f->base = calloc(1, bytes + 64);                    /* device frames start zeroed, like the real pool's */
    size_t off = 0;
    for (int p = 0; p < 3; p++)
    {
        const int absent = two_planes && p == 2;
        f->row_bytes[p] = row_bytes[p]; f->rows[p] = rows[p]; f->strides[p] = absent ? 0 : strides[p];
        f->planes[p] = absent ? NULL : f->base + off;
        off += (size_t)f->strides[p] * rows[p];
    }
    frames_alive++;
    *out = f;
    return 0;
}
