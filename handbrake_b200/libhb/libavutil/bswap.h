/* libavutil/bswap.h -- the byte swap libhb's blend.c uses for semi-planar 16-bit overlays (part of the shim, see
 * handbrake/handbrake.h).  Only av_bswap16 is restated. */
#ifndef HBCU_SHIM_AVUTIL_BSWAP_H
#define HBCU_SHIM_AVUTIL_BSWAP_H

#include <stdint.h>

static inline uint16_t av_bswap16(uint16_t x)
{
    return (uint16_t)((x >> 8) | (x << 8));
}

#endif
