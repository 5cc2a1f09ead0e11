/* libavutil/avutil.h -- the part of FFmpeg's header libhb's vfr.c uses (shim, see handbrake/handbrake.h) */
#ifndef HBCU_SHIM_AVUTIL_H
#define HBCU_SHIM_AVUTIL_H
#include <stdint.h>

#define AV_NOPTS_VALUE ((int64_t)UINT64_C(0x8000000000000000))

#endif
