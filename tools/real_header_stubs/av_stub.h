/* the libav* types libhb's public headers mention, as opaque or minimal declarations: enough for a syntax-only
 * compile of the CUDA filter sources against the REAL handbrake headers (tools/check_real_headers.sh) */
#ifndef AV_STUB_H
#define AV_STUB_H
#include <stdint.h>
#include <stddef.h>
typedef struct AVRational { int num, den; } AVRational;
enum AVPixelFormat { AV_PIX_FMT_NONE = -1, AV_PIX_FMT_YUV420P = 0, AV_PIX_FMT_YUV420P10LE = 62, AV_PIX_FMT_YUV420P10 = 62, AV_PIX_FMT_CUDA = 117, AV_PIX_FMT_NB = 300 };
enum AVSampleFormat { AV_SAMPLE_FMT_NONE = -1, AV_SAMPLE_FMT_FLT = 3 };
enum AVCodecID { AV_CODEC_ID_NONE = 0 };
enum AVColorPrimaries { AVCOL_PRI_UNSPECIFIED = 2 };
enum AVColorTransferCharacteristic { AVCOL_TRC_UNSPECIFIED = 2 };
enum AVColorSpace { AVCOL_SPC_UNSPECIFIED = 2 };
enum AVColorRange { AVCOL_RANGE_UNSPECIFIED = 0 };
enum AVChromaLocation { AVCHROMA_LOC_UNSPECIFIED = 0 };
enum AVHWDeviceType { AV_HWDEVICE_TYPE_NONE = 0 };
enum AVMatrixEncoding { AV_MATRIX_ENCODING_NONE = 0 };
enum AVFrameSideDataType { AV_FRAME_DATA_PANSCAN = 0 };
int av_image_get_linesize(enum AVPixelFormat pix_fmt, int width, int plane);
typedef struct AVComponentDescriptor { int plane, step, offset, shift, depth; } AVComponentDescriptor;
typedef struct AVPixFmtDescriptor { const char *name; uint8_t nb_components, log2_chroma_w, log2_chroma_h; uint64_t flags; AVComponentDescriptor comp[4]; const char *alias; } AVPixFmtDescriptor;
const AVPixFmtDescriptor *av_pix_fmt_desc_get(enum AVPixelFormat pix_fmt);
int av_pix_fmt_count_planes(enum AVPixelFormat pix_fmt);
enum AVPixelFormat av_get_pix_fmt(const char *name);
const char *av_get_pix_fmt_name(enum AVPixelFormat pix_fmt);
typedef struct AVChannelLayout { int order, nb_channels; union { uint64_t mask; void *map; } u; void *opaque; } AVChannelLayout;
typedef struct AVBufferRef AVBufferRef;
typedef struct AVFrame AVFrame;
typedef struct AVPacket AVPacket;
typedef struct AVCodecContext AVCodecContext;
typedef struct AVCodec AVCodec;
typedef struct AVCodecParameters AVCodecParameters;
typedef struct AVFormatContext AVFormatContext;
typedef struct AVStream AVStream;
typedef struct AVDictionary AVDictionary;
typedef struct AVFrameSideData AVFrameSideData;
typedef struct AVMasteringDisplayMetadata AVMasteringDisplayMetadata;
typedef struct AVContentLightMetadata AVContentLightMetadata;
typedef struct AVAmbientViewingEnvironment AVAmbientViewingEnvironment;
typedef struct AVDOVIDecoderConfigurationRecord AVDOVIDecoderConfigurationRecord;
typedef struct AVFilterContext AVFilterContext;
typedef struct AVFilterGraph AVFilterGraph;
typedef struct SwsContext SwsContext;
typedef struct SwrContext SwrContext;
typedef struct AVDownmixInfo AVDownmixInfo;
#define AV_NOPTS_VALUE ((int64_t)UINT64_C(0x8000000000000000))
#define AV_NUM_DATA_POINTERS 8
#endif
