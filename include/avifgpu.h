/*
 * avifgpu.h -- C ABI of the H100-native colour-conversion hot path of the avif-format plug-in.
 *
 * This header is the drop-in boundary: plain pointers and sizes, no C++ / torch types.  Every entry point
 * replaces one seam of the reference (citations are relative to the reference tree, src/common/):
 *
 *   avifgpu_encode_rows*          the per-row loops of CreateHeifImage{Gray,RGB}{Eight,Sixteen,ThirtyTwo}Bit
 *                                 (WriteHeifImage.cpp:169-1139; called from Write.cpp:303-336) and, for
 *                                 AVIFGPU_LAYOUT_PLANAR_YCBCR, additionally the RGB->YCbCr matrix + chroma
 *                                 down-sampling that the reference delegates to libheif inside
 *                                 heif_context_encode_image (Write.cpp:44; matrix chosen at
 *                                 WriteMetadata.cpp:107-149).
 *   avifgpu_decode_rows*          the per-row loops of ReadHeifImage{Gray,RGB}{Eight,Sixteen,ThirtyTwo}Bit
 *                                 (ReadHeifImage.cpp:83-1178; called from Read.cpp:587-630), i.e. the twelve
 *                                 Decode*Row* functions of YUVDecode.h:29-147 plus the planar-RGB branches.
 *   avifgpu_get_yuv_coefficients  GetYUVCoefficiants (YUVCoefficiants.cpp:154-188).
 *   avifgpu_build_yuv_tables      YUVLookupTables::YUVLookupTables (YuvLookupTables.cpp:115-192).
 *   avifgpu_transfer_f32          LinearToPQ / PQToLinear / LinearToSMPTE428 / SMPTE428ToLinear /
 *                                 HLGToLinear / LinearToHLG (ColorTransfer.cpp:69-190), evaluated on the GPU
 *                                 with the device libm of csrc/device_math.cuh (used by the primitive-level
 *                                 parity gates).
 *
 * The "_device" variants take device pointers and a cudaStream_t (as void*) and never synchronise: they are
 * what a caller that keeps frames resident in HBM uses, and what bench.py times for `value`.  The plain
 * variants take HOST pointers, move the row block over PCIe through pinned staging owned by the context and
 * return when the destination host memory is valid: they are what the plug-in's FormatRecord row shuttle
 * binds (see INTEGRATION.md), and what bench.py times for `e2e`.
 *
 * There is no CPU fallback.  If no CUDA device is usable avifgpu_create fails with AVIFGPU_ERR_NO_DEVICE.
 *
 * Error convention (reference: exceptions mapped to OSErr at Write.cpp:345-364 / Read.cpp:659-678): every
 * function returns 0 on success or a negative avifgpu_status; nothing throws across this boundary.  The C++
 * host mirror (avif-format_b200/host) turns the codes back into OSErrException / std::runtime_error.
 */
#ifndef AVIFGPU_H
#define AVIFGPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(_WIN32) && defined(AVIFGPU_BUILDING_LIBRARY)
#define AVIFGPU_EXPORT __declspec(dllexport)
#elif defined(_WIN32)
#define AVIFGPU_EXPORT __declspec(dllimport) /* the plug-in (an MSVC project) consuming avifgpu.dll */
#else
#define AVIFGPU_EXPORT __attribute__((visibility("default")))
#endif

#define AVIFGPU_API_VERSION 13

typedef enum avifgpu_status
{
    AVIFGPU_OK = 0,
    AVIFGPU_ERR_BAD_PARAM = -1,    /* -> formatBadParameters                                   */
    AVIFGPU_ERR_UNSUPPORTED = -2,  /* -> std::runtime_error("Unsupported ...") in the reference */
    AVIFGPU_ERR_NO_DEVICE = -3,    /* -> errPlugInHostInsufficient                              */
    AVIFGPU_ERR_CUDA = -4,         /* -> std::runtime_error                                     */
    AVIFGPU_ERR_OOM = -5,          /* -> memFullErr / std::bad_alloc                            */
    AVIFGPU_ERR_CANCELED = -6      /* -> userCanceledErr (abortProc polled between row blocks)  */
} avifgpu_status;

/* AlphaState.h:24-29 (same order). */
typedef enum avifgpu_alpha_state
{
    AVIFGPU_ALPHA_NONE = 0,
    AVIFGPU_ALPHA_STRAIGHT = 1,
    AVIFGPU_ALPHA_PREMULTIPLIED = 2
} avifgpu_alpha_state;

/* ColorTransfer.h:28-34 (same order). */
typedef enum avifgpu_transfer
{
    AVIFGPU_TRANSFER_PQ = 0,
    AVIFGPU_TRANSFER_HLG = 1,
    AVIFGPU_TRANSFER_SMPTE428 = 2,
    AVIFGPU_TRANSFER_CLIP = 3
} avifgpu_transfer;

/* Numeric values = libheif's heif_chroma for the planar kinds. */
typedef enum avifgpu_chroma
{
    AVIFGPU_CHROMA_MONOCHROME = 0,
    AVIFGPU_CHROMA_420 = 1,
    AVIFGPU_CHROMA_422 = 2,
    AVIFGPU_CHROMA_444 = 3
} avifgpu_chroma;

/* Numeric values = libheif's heif_colorspace. */
typedef enum avifgpu_colorspace
{
    AVIFGPU_COLORSPACE_YCBCR = 0,
    AVIFGPU_COLORSPACE_RGB = 1,
    AVIFGPU_COLORSPACE_MONOCHROME = 2
} avifgpu_colorspace;

typedef enum avifgpu_layout
{
    /* What the reference itself produces: heif_channel_interleaved RGB(A) for colour hosts
     * (WriteHeifImage.cpp:63-85, 639-646) and heif_channel_Y (+ heif_channel_Alpha) planes for gray hosts
     * (WriteHeifImage.cpp:177-194).  plane[0] = interleaved / Y, plane[3] = Alpha (gray only). */
    AVIFGPU_LAYOUT_REFERENCE = 0,
    /* Fused: additionally applies the forward matrix + chroma down-filter and writes heif_channel_Y / Cb /
     * Cr (/ Alpha) planes at image_bit_depth.  plane[0..3] = Y, Cb, Cr, Alpha.  Colour hosts only. */
    AVIFGPU_LAYOUT_PLANAR_YCBCR = 1
} avifgpu_layout;

typedef enum avifgpu_down_filter
{
    AVIFGPU_DOWN_FILTER_BOX = 0,     /* mean of the 2x1 / 2x2 float chroma samples, then quantise */
    AVIFGPU_DOWN_FILTER_TOP_LEFT = 1 /* co-sited top-left sample (libheif 1.14-like)              */
} avifgpu_down_filter;

/* Extra transfer option outside the reference's ColorTransferFunction enum: BASELINE.json config 5
 * (Gray16 -> 12-bit monochrome SMPTE 428-1), a composition this project defines (SURVEY.md section 8c). */
typedef enum avifgpu_gray16_curve
{
    AVIFGPU_GRAY16_LUT = 0,      /* reference behaviour: BuildSixteenBitToHeifImageLookup, WriteHeifImage.cpp:140-166 */
    AVIFGPU_GRAY16_SMPTE428 = 1  /* code = (u16)clamp(LinearToSMPTE428(v/32768f)*max, 0, max)                         */
} avifgpu_gray16_curve;

/* Mirrors heif_color_profile_nclx as far as the path reads it (YuvLookupTables.cpp:143-144,
 * YUVCoefficiants.cpp:110-152, ColorTransfer.cpp:31-67).  present == 0 means "nclx == nullptr". */
typedef struct avifgpu_nclx
{
    int32_t present;
    int32_t color_primaries;          /* H.273 code point */
    int32_t transfer_characteristics; /* H.273 code point */
    int32_t matrix_coefficients;      /* H.273 code point */
    int32_t full_range_flag;
} avifgpu_nclx;

#define AVIFGPU_MAX_PLANES 4

/* A set of image planes.  stride in BYTES (libheif pads rows: heif_image_get_plane's out_stride).
 * Samples deeper than 8 bit are native-endian uint16 with the value in the low bits, unless a decode description's
 * source_layout or an encode description's dest_layout says otherwise. */
typedef struct avifgpu_planes
{
    void* data[AVIFGPU_MAX_PLANES];
    int64_t stride[AVIFGPU_MAX_PLANES];
} avifgpu_planes;

/* Parameter block of the encode direction = FormatRecord fields + SaveUIOptions fields the loops read
 * (AvifFormat.h:87-101, Write.cpp:229-258 fix-ups are the CALLER's job and are mirrored in host/). */
typedef enum avifgpu_hlg_extension
{
    AVIFGPU_HLG_REJECT = 0,                /* what the reference does */
    AVIFGPU_HLG_OETF = 1,                  /* scene-referred input: code = quantise(LinearToHLG(c)) */
    AVIFGPU_HLG_INVERSE_OOTF_THEN_OETF = 2 /* display-referred input: ApplyInverseHLGOOTF(rgb) first; needs nclx primaries */
} avifgpu_hlg_extension;

typedef struct avifgpu_encode_desc
{
    uint32_t struct_size;    /* sizeof(avifgpu_encode_desc) */
    int32_t width;           /* imageSize.h */
    int32_t height;          /* imageSize.v */
    int32_t host_depth;      /* formatRecord->depth: 8, 16 (0..32768) or 32 (float) */
    int32_t host_channels;   /* formatRecord->planes: 1 Gray, 2 Gray+A, 3 RGB, 4 RGB+A */
    int32_t alpha_state;     /* avifgpu_alpha_state */
    int32_t image_bit_depth; /* SaveUIOptions.imageBitDepth: 8, 10 or 12 */
    int32_t transfer;        /* SaveUIOptions.hdrTransferFunction (32-bit hosts only) */
    int32_t pq_peak_nits;    /* SaveUIOptions.pq.nominalPeakBrightness */
    int32_t layout;          /* avifgpu_layout */
    int32_t chroma;          /* avifgpu_chroma, for AVIFGPU_LAYOUT_PLANAR_YCBCR */
    int32_t down_filter;     /* avifgpu_down_filter */
    int32_t gray16_curve;    /* avifgpu_gray16_curve, Gray16 hosts only */
    avifgpu_nclx nclx;       /* matrix for PLANAR_YCBCR (WriteMetadata.cpp:113-146); full range only */
    /* HLG save path (SURVEY.md 8f-4).  The reference ships LinearToHLG and ApplyInverseHLGOOTF (ColorTransfer.cpp:141-164,
     * 207-220) but no caller: with hlg_extension = 0 transfer = AVIFGPU_TRANSFER_HLG is rejected with the reference's own
     * "Unsupported color transfer function." (WriteHeifImage.cpp:1085-1087).  Colour float hosts only. */
    int32_t hlg_extension;       /* avifgpu_hlg_extension */
    float hlg_display_gamma;     /* for AVIFGPU_HLG_INVERSE_OOTF_THEN_OETF (LoadUIOptions.hlg.displayGamma's counterpart) */
    int32_t hlg_peak_nits;       /* nominal peak brightness of the display-referred input */
    /* Colour-profile step on the GPU (SURVEY.md 8f-3), colour float hosts only.  The reference converts every host row
     * with lcms2 before anything else (ColorProfileConversion::ConvertRow at WriteHeifImage.cpp:1028-1031); for a
     * linear-light document in a matrix profile that conversion is one 3x3 matrix, applied here per pixel in binary32,
     * alpha untouched (cmsFLAGS_COPY_ALPHA), before the clamp / premultiply / transfer curve:
     *     r' = (m[0] r + m[1] g) + m[2] b,  g' = (m[3] r + m[4] g) + m[5] b,  b' = (m[6] r + m[7] g) + m[8] b
     * avifgpu_icc_to_rec2020_linear_matrix() derives it from an ICC profile.  Parity unpinned (lcms2 is not in the tree). */
    int32_t row_matrix_enabled;
    float row_matrix[9];
    /* Since API version 11: avifgpu_source_layout bits saying how the YCbCr planes are written (the table below).
     * Non-zero only for AVIFGPU_LAYOUT_PLANAR_YCBCR (AVIFGPU_ERR_UNSUPPORTED otherwise); AVIFGPU_SOURCE_MSB_ALIGNED needs
     * image_bit_depth 10 or 12 and unknown bits are AVIFGPU_ERR_BAD_PARAM.  Only the device-pointer calls write such
     * planes (avifgpu_encode_rows_device, avifgpu_encode_batch_device, avifgpu_encode_batch_indirect); the host-pointer,
     * asynchronous and sharded calls refuse a non-zero layout with AVIFGPU_ERR_UNSUPPORTED and launch nothing.  With
     * AVIFGPU_SOURCE_CHROMA_INTERLEAVED planes.data[2] is ignored and never written; with AVIFGPU_SOURCE_MSB_ALIGNED every
     * sample written, alpha included, is code << (16 - image_bit_depth) with the low bits zero.  A struct_size of
     * AVIFGPU_ENCODE_DESC_V10_SIZE (a caller built against API version 10, which has no such field) is accepted and
     * means AVIFGPU_SOURCE_PLANAR.
     *   surface format           image_bit_depth  dest_layout
     *   NV12 (4:2:0), NV16       8                AVIFGPU_SOURCE_CHROMA_INTERLEAVED
     *   P010 (4:2:0), P210       10               AVIFGPU_SOURCE_CHROMA_INTERLEAVED | AVIFGPU_SOURCE_MSB_ALIGNED
     *   P016 (4:2:0)             12               AVIFGPU_SOURCE_CHROMA_INTERLEAVED | AVIFGPU_SOURCE_MSB_ALIGNED
     *   YUV444_16Bit             10 or 12         AVIFGPU_SOURCE_MSB_ALIGNED
     * Every sample is, bit for bit, the planar, low-bit encode's code of the same description and rows, moved and
     * shifted. */
    int32_t dest_layout;
} avifgpu_encode_desc;

/* sizeof(avifgpu_encode_desc) up to API version 10: everything before dest_layout. */
#define AVIFGPU_ENCODE_DESC_V10_SIZE ((uint32_t)offsetof(avifgpu_encode_desc, dest_layout))

/* Parameter block of the decode direction = heif_image properties + nclx + LoadUIOptions
 * (AvifFormat.h:61-85). */
/* How YCbCr planes sit in memory, a bit set: the planes a decode reads (avifgpu_decode_desc.source_layout) and, since API
 * version 11, the planes an encode writes (avifgpu_encode_desc.dest_layout).  Hardware video decoders (NVDEC through the
 * Video Codec SDK or nvImageCodec, D3D12 and Vulkan video) write their frames this way, and hardware video encoders
 * (NVENC, D3D12 and Vulkan video encode) and HDR swap chains read them:
 *   surface format         bit_depth  source_layout
 *   NV12 (4:2:0), NV16     8          AVIFGPU_SOURCE_CHROMA_INTERLEAVED
 *   P010 / P016 (4:2:0)    10 or 12   AVIFGPU_SOURCE_CHROMA_INTERLEAVED | AVIFGPU_SOURCE_MSB_ALIGNED
 *   YUV444 (8-bit planar)  8          AVIFGPU_SOURCE_PLANAR
 *   YUV444_16Bit           10 or 12   AVIFGPU_SOURCE_MSB_ALIGNED
 * A decode's output is, bit for bit, that of the same decode of the equivalent planar, low-bit source; an encode's planes
 * hold, bit for bit, the planar, low-bit encode's codes, moved and shifted. */
typedef enum avifgpu_source_layout
{
    /* libheif's (and dav1d's) layout: planes Y, Cb, Cr, Alpha; deeper codes in the low bits of a uint16.  The default. */
    AVIFGPU_SOURCE_PLANAR = 0,
    /* Cb and Cr interleaved in plane 1, Cb first (NV12 / NV16 / P010 / P016 / P210 order): a chroma row holds
     * 2 * ((width + xs) >> xs) samples.  planes.data[2] is ignored (neither read nor written); alpha stays plane 3. */
    AVIFGPU_SOURCE_CHROMA_INTERLEAVED = 1,
    /* Every sample of every plane is a uint16 whose top bit_depth bits hold the code, code = sample >> (16 - bit_depth).
     * A decode ignores the low bits, whatever they hold; an encode writes them zero.  Bit depth 10 or 12 only. */
    AVIFGPU_SOURCE_MSB_ALIGNED = 2
} avifgpu_source_layout;

typedef struct avifgpu_decode_desc
{
    uint32_t struct_size;   /* sizeof(avifgpu_decode_desc) */
    int32_t width;
    int32_t height;
    int32_t colorspace;     /* avifgpu_colorspace */
    int32_t chroma;         /* avifgpu_chroma (YCbCr / monochrome); ignored for planar RGB */
    int32_t bit_depth;      /* heif_image_get_bits_per_pixel_range: 8, 10, 12 or 16 */
    int32_t alpha_state;    /* avifgpu_alpha_state */
    int32_t host_depth;     /* 8, 16 or 32: which ReadHeifImage*Bit variant */
    avifgpu_nclx nclx;
    int32_t hlg_apply_ootf;      /* LoadUIOptions.hlg.applyOOTF */
    float hlg_display_gamma;     /* LoadUIOptions.hlg.displayGamma */
    int32_t hlg_peak_nits;       /* LoadUIOptions.hlg.nominalPeakBrightness */
    int32_t pq_peak_nits;        /* LoadUIOptions.pq.nominalPeakBrightness */
    /* Since API version 10: avifgpu_source_layout bits.  Non-zero only for AVIFGPU_COLORSPACE_YCBCR
     * (AVIFGPU_ERR_UNSUPPORTED otherwise); AVIFGPU_SOURCE_MSB_ALIGNED needs bit_depth 10 or 12 and unknown bits are
     * AVIFGPU_ERR_BAD_PARAM.  Only the device-pointer calls read such sources (avifgpu_decode_rows_device,
     * avifgpu_decode_batch_device, avifgpu_decode_batch_indirect); the host-pointer, asynchronous and sharded calls refuse
     * a non-zero layout with AVIFGPU_ERR_UNSUPPORTED and launch nothing.  A struct_size of AVIFGPU_DECODE_DESC_V9_SIZE
     * (a caller built against API version 9, which has no such field) is accepted and means AVIFGPU_SOURCE_PLANAR. */
    int32_t source_layout;
} avifgpu_decode_desc;

/* sizeof(avifgpu_decode_desc) up to API version 9: everything before source_layout. */
#define AVIFGPU_DECODE_DESC_V9_SIZE ((uint32_t)offsetof(avifgpu_decode_desc, source_layout))

typedef struct avifgpu_context avifgpu_context;

/* ---- context --------------------------------------------------------------------------------------- */

AVIFGPU_EXPORT int avifgpu_api_version(void);

/* Binds to CUDA device `device_ordinal` (must be compute capability 10.x).  No CPU fallback. */
AVIFGPU_EXPORT int avifgpu_create(int device_ordinal, avifgpu_context** out_ctx);
AVIFGPU_EXPORT void avifgpu_destroy(avifgpu_context* ctx);

/* Human-readable text for the last failure on this context (never NULL). ctx may be NULL for creation errors. */
AVIFGPU_EXPORT const char* avifgpu_last_error(const avifgpu_context* ctx);
AVIFGPU_EXPORT const char* avifgpu_status_string(int status);

/* Number of kernels this context has launched so far (bench.py's gpu_launches). */
AVIFGPU_EXPORT int64_t avifgpu_launch_count(const avifgpu_context* ctx);

/* Blocks until all work issued through this context has finished. */
AVIFGPU_EXPORT int avifgpu_synchronize(avifgpu_context* ctx);

/* Pinned host memory for row buffers (the plug-in's replacement for its one-row ScopedBufferSuiteBuffer,
 * Write.cpp:297-299 / ReadHeifImage.cpp:113-115). */
AVIFGPU_EXPORT int avifgpu_host_alloc(avifgpu_context* ctx, size_t bytes, void** out_ptr);
AVIFGPU_EXPORT int avifgpu_host_free(avifgpu_context* ctx, void* ptr);

/* ---- geometry helpers (pure host arithmetic, usable without a device) ------------------------------- */

/* Bytes per host pixel (formatRecord->colBytes) for an encode / decode description. */
AVIFGPU_EXPORT int avifgpu_encode_host_col_bytes(const avifgpu_encode_desc* desc);
AVIFGPU_EXPORT int avifgpu_decode_host_col_bytes(const avifgpu_decode_desc* desc);

/* Width / height / bytes-per-sample of plane `index` of the encode destination or decode source.
 * Returns 0 and zeroes the outputs for planes that do not exist in that configuration. */
AVIFGPU_EXPORT int avifgpu_encode_plane_geometry(const avifgpu_encode_desc* desc, int index,
                                                 int32_t* out_width_samples, int32_t* out_height,
                                                 int32_t* out_bytes_per_sample);
AVIFGPU_EXPORT int avifgpu_decode_plane_geometry(const avifgpu_decode_desc* desc, int index,
                                                 int32_t* out_width_samples, int32_t* out_height,
                                                 int32_t* out_bytes_per_sample);

/* ---- parameter derivation (host arithmetic identical to the reference's) ---------------------------- */

/* GetYUVCoefficiants, YUVCoefficiants.cpp:154-188: out_kr_kg_kb[3]. */
AVIFGPU_EXPORT int avifgpu_get_yuv_coefficients(const avifgpu_nclx* nclx, float* out_kr_kg_kb);

/* GetHLGLumaCoefficients, ColorTransfer.cpp:31-45: out_rgb[3]; AVIFGPU_ERR_UNSUPPORTED for other primaries. */
AVIFGPU_EXPORT int avifgpu_get_hlg_luma_coefficients(int32_t color_primaries, float* out_rgb);

/* YUVLookupTables ctor, YuvLookupTables.cpp:115-192.  Each non-NULL table receives 1 << bit_depth floats. */
AVIFGPU_EXPORT int avifgpu_build_yuv_tables(const avifgpu_nclx* nclx, int32_t bit_depth, int32_t monochrome,
                                            float* out_table_y, float* out_table_uv, float* out_table_alpha);

/* ICC profile -> the matrix of avifgpu_encode_desc.row_matrix for an HDR save (document RGB, linear light -> linear
 * Rec.2020, what ColorProfileConversion::InitializeForRec2020Conversion sets up, ColorProfileConversion.cpp:240-266).
 * AVIFGPU_OK: out_matrix9 filled; *out_is_rec2020 = 1 when the profile already is Rec.2020 (the reference then converts
 * nothing, ColorProfileConversion.cpp:128-131).  AVIFGPU_ERR_UNSUPPORTED: not a matrix / TRC RGB profile with identity
 * tone curves (LUT profiles, gamma-encoded profiles: those stay with the host's lcms2).  Pure host arithmetic. */
AVIFGPU_EXPORT int avifgpu_icc_to_rec2020_linear_matrix(const void* icc_profile, size_t size, float* out_matrix9, int32_t* out_is_rec2020);

/* ---- the hot path: host-pointer variants (PCIe inside) ---------------------------------------------- */

/*
 * Converts host rows [y0, y0 + nrows) and stores them into the destination planes.
 *   host_rows   interleaved host pixels of row y0 (formatRecord->data after advanceState for
 *               theRect = {top = y0, bottom = y0 + nrows}); row_stride_bytes = formatRecord->rowBytes.
 *   dst         HOST pointers to the origin (row 0) of each whole-image plane, e.g. heif_image_get_plane().
 * For 4:2:0 output y0 must be even and nrows even unless y0 + nrows == height.
 */
AVIFGPU_EXPORT int avifgpu_encode_rows(avifgpu_context* ctx, const avifgpu_encode_desc* desc,
                                       const void* host_rows, int64_t row_stride_bytes,
                                       int32_t y0, int32_t nrows, const avifgpu_planes* dst);

/*
 * Converts image rows [y0, y0 + nrows) of the source planes into interleaved host rows.
 *   src         HOST pointers to the origin of each whole-image plane (heif_image_get_plane_readonly()):
 *               YCbCr: Y, Cb, Cr, Alpha; monochrome: Y, -, -, Alpha; planar RGB: R, G, B, Alpha.
 *   host_rows   receives row y0 first; row_stride_bytes = formatRecord->rowBytes.
 */
AVIFGPU_EXPORT int avifgpu_decode_rows(avifgpu_context* ctx, const avifgpu_decode_desc* desc,
                                       const avifgpu_planes* src, int32_t y0, int32_t nrows,
                                       void* host_rows, int64_t row_stride_bytes);

/* ---- the hot path: asynchronous host-pointer variants ------------------------------------------------------ */

/*
 * The same conversions, enqueued: the call returns once the work is on the device's queues, so the caller's thread can
 * produce the next row block (the plug-in: advanceState, i.e. Photoshop filling the next rows, Write.cpp:297-336) while
 * the GPU converts and copies this one.  Single-threaded contract like the rest of a context: calls on one context come
 * from one thread at a time.
 *   encode: on return the rows of THIS call may still be read by the copy engine when host_rows is page-locked memory
 *           (avifgpu_host_alloc).  They may be overwritten (two row buffers make a double-buffered shuttle) once one of
 *           these has returned AVIFGPU_OK on this context: the next host-pointer call of either direction -- encode or
 *           decode, synchronous or asynchronous, an empty row block included; avifgpu_wait() with a ticket covering
 *           this call; avifgpu_synchronize().  A call refused with an error does not release them, and neither do the
 *           device-pointer and batch calls.  Pageable rows are consumed before return.
 *           The destination planes are complete after avifgpu_wait(ticket).
 *   decode: the source planes must stay valid and the host rows are complete after avifgpu_wait(ticket).
 * out_ticket (may be NULL) identifies the call; tickets increase by one per host-pointer call on a context.
 */
AVIFGPU_EXPORT int avifgpu_encode_rows_async(avifgpu_context* ctx, const avifgpu_encode_desc* desc,
                                             const void* host_rows, int64_t row_stride_bytes,
                                             int32_t y0, int32_t nrows, const avifgpu_planes* dst, int64_t* out_ticket);
AVIFGPU_EXPORT int avifgpu_decode_rows_async(avifgpu_context* ctx, const avifgpu_decode_desc* desc,
                                             const avifgpu_planes* src, int32_t y0, int32_t nrows,
                                             void* host_rows, int64_t row_stride_bytes, int64_t* out_ticket);
/* Blocks until every host-pointer call up to and including `ticket` has completed and its results are in the
 * caller's memory; ticket <= 0 waits for everything issued so far. */
AVIFGPU_EXPORT int avifgpu_wait(avifgpu_context* ctx, int64_t ticket);

/* ---- the hot path: device-pointer variants (no copies, no synchronisation) --------------------------- */

/* Same contracts, but host_rows / planes are DEVICE pointers valid on the context's device and the work is
 * enqueued on `cuda_stream` (a cudaStream_t; NULL = the legacy default stream).  The decode call also reads the
 * semi-planar and MSB-aligned sources of avifgpu_decode_desc.source_layout, with any row block (an odd y0 of a 4:2:0
 * image included); since API version 11 the encode call writes the semi-planar and MSB-aligned planes of
 * avifgpu_encode_desc.dest_layout, with any row block the planar layout takes.
 *
 * CUDA graph capture.  Both calls may be recorded into a CUDA graph (cudaStreamBeginCapture ... cudaStreamEndCapture,
 * or torch.cuda.graph), in any capture mode, global included.  While `cuda_stream` is capturing a call:
 *   - enqueues kernel launches on `cuda_stream` and nothing else: no allocation, no synchronisation, no copy;
 *   - uses only the first-use state the context already has: step tables, Gray16 LUTs and the verified fast forms
 *     (divisions, premultiplication).  What is missing takes, for this call only, the path that needs no preparation
 *     (the generic exact kernel, or the reference instruction sequence) -- bit-identical outputs, typically slower
 *     kernels.  Nothing is cached, and the call's pixels do not count towards avifgpu_set_table_autobuild.
 *     Prepare before capturing so that the graph holds the tuned kernels: avifgpu_prepare_encode (step tables, Gray16
 *     LUTs), avifgpu_prepare_decode (HLG / PQ / green divisions), and for integer planar encodes with premultiplied
 *     alpha one direct call outside the capture (the premultiply check);
 *   - returns a launch failure without synchronising anything: ending the capture is the caller's business.
 * The graph holds the pointers, strides, row block and description of the captured call: to convert another frame,
 * copy it into the captured buffers and replay.  avifgpu_launch_count counts the captured kernels once, at capture, and
 * not per replay.  The graph refers to the context's tables, which are never freed or moved before avifgpu_destroy:
 * it stays valid, whatever the context prepares later, until then.  The legacy NULL stream cannot be captured; capture
 * on a stream of your own. */
AVIFGPU_EXPORT int avifgpu_encode_rows_device(avifgpu_context* ctx, const avifgpu_encode_desc* desc,
                                              const void* device_rows, int64_t row_stride_bytes,
                                              int32_t y0, int32_t nrows, const avifgpu_planes* device_dst,
                                              void* cuda_stream);

AVIFGPU_EXPORT int avifgpu_decode_rows_device(avifgpu_context* ctx, const avifgpu_decode_desc* desc,
                                              const avifgpu_planes* device_src, int32_t y0, int32_t nrows,
                                              void* device_rows, int64_t row_stride_bytes,
                                              void* cuda_stream);

/* ---- content light level of PQ encodes (since API version 12) ---------------------------------------------------- */

/*
 * The static HDR metadata every PQ stream or still carries -- the HEVC / AV1 content light level SEI or metadata OBU, the
 * AVIF / HEIF `clli` property -- holds two values (CTA-861.3): MaxCLL, the brightest pixel, and MaxFALL, the frame-average
 * light level, where a pixel's light level is max(R, G, B) in cd/m2.  The light-level encode measures them on the codes it
 * writes, in the same pass.
 *
 * Definition.  For every pixel the call converts, k = max(R', G', B') of the pixel's transfer-curve codes at
 * image_bit_depth -- the codes the encode computes before the forward matrix, after the clamp, premultiplication and
 * row_matrix; for Gray / Gray+A hosts k is the Y code; alpha never counts.  The level of code k is
 *     level(k) = (uint32_t)(PQToLinear((float)k / (float)maxCode, 1.0f) * 2^22), truncated,
 * PQToLinear being ColorTransfer.cpp:94-117 with multiplier 1 (the absolute PQ scale, 1.0 = 10000 cd/m2) in binary32 with
 * glibc's powf; it does not depend on pq_peak_nits.  Working on codes makes the statistic exact and independent of the
 * order in which pixels are visited: every route gives the same integers, and NaN, +-inf and negative inputs count with
 * the code the encode gives them.
 *
 * The accumulator is device memory, zeroed by the caller, and collects every call made into it. */
typedef struct avifgpu_light_level
{
    uint32_t max_code;  /* atomicMax of k over the pixels converted */
    uint32_t reserved;  /* never written */
    uint64_t level_sum; /* sum of level(k), units of 2^-22 x 10000 cd/m2 */
    uint64_t pixels;    /* pixels converted */
} avifgpu_light_level;

/*
 * avifgpu_encode_rows_device, plus the content light level of the rows converted, added into *device_acc.
 *   - Same contract as avifgpu_encode_rows_device: any row block, every dest_layout, graph capture under the same rules.
 *     The graph holds the accumulator's address: a replay adds into whatever the accumulator holds when it runs.
 *   - Writes the same planes, bit for bit, with the same number of kernel launches as avifgpu_encode_rows_device.
 *   - Row blocks add up: the blocks of an image accumulate what one call over the whole image does.
 *   - Accepts host_depth 32 with transfer AVIFGPU_TRANSFER_PQ, in any layout, channel count, alpha state, chroma,
 *     down_filter or row_matrix.  Every other description is AVIFGPU_ERR_UNSUPPORTED and launches nothing; a NULL
 *     device_acc is AVIFGPU_ERR_BAD_PARAM.
 *   - The tuned kernels read level(k) from a 2^image_bit_depth-word table the context builds with the step tables
 *     (avifgpu_prepare_encode); a call captured before it exists takes the generic kernel, which evaluates level(k) itself:
 *     the same result, a slower kernel.
 * Since API version 13 the batch calls have light-level forms too (avifgpu_encode_batch_device_light_level,
 * avifgpu_encode_batch_indirect_light_level, below): one accumulator per image; so do the host-pointer, asynchronous
 * and sharded calls (avifgpu_encode_rows_light_level and its siblings, below), into a host accumulator; and so does the
 * sharded device-pointer call (avifgpu_encode_rows_sharded_device_light_level, below), into the owner's memory. */
AVIFGPU_EXPORT int avifgpu_encode_rows_device_light_level(avifgpu_context* ctx, const avifgpu_encode_desc* desc,
                                                          const void* device_rows, int64_t row_stride_bytes,
                                                          int32_t y0, int32_t nrows, const avifgpu_planes* device_dst,
                                                          avifgpu_light_level* device_acc, void* cuda_stream);

/* MaxCLL and MaxFALL in cd/m2 from an accumulator copied to the host (pure host arithmetic):
 *   MaxCLL  = ceil(10000 * level(max_code) / 2^22)
 *   MaxFALL = ceil(10000 * level_sum / (2^22 * pixels)), exact (128-bit integers)
 * Both are 0 when pixels == 0.  AVIFGPU_ERR_BAD_PARAM for a NULL pointer, an image_bit_depth other than 8, 10 or 12, a
 * max_code above 2^image_bit_depth - 1, or a level_sum above 2^22 * pixels (not an accumulator of this depth). */
AVIFGPU_EXPORT int avifgpu_content_light_level(const avifgpu_light_level* acc, int32_t image_bit_depth,
                                               uint16_t* out_max_cll, uint16_t* out_max_fall);

/* ---- the hot path: batches of small device-resident images ------------------------------------------------ */

/* One image of a batch: a whole image of the batch's description with its own size and buffers (device memory).
 *   encode: rows = the source host-layout rows, planes = the destination planes;
 *   decode: planes = the source planes, rows = the destination host-layout rows. */
typedef struct avifgpu_batch_image
{
    int32_t width;
    int32_t height;
    void* rows;
    int64_t row_stride_bytes;
    avifgpu_planes planes;
} avifgpu_batch_image;

/*
 * Converts `count` whole images with one encode description, many per kernel launch: for small images (thumbnails, image
 * sets) a launch per image costs more than the image's own memory traffic.
 *   - All images share `desc`; its width and height are replaced by each image's own.
 *   - Each image is converted whole, like avifgpu_encode_rows_device with y0 = 0 and nrows = height.
 *   - The result equals `count` such calls, one per image, in order, on `cuda_stream`, bit for bit.
 *   - Every image is validated as `desc` with its own size, and its rows and planes are checked for NULL, before
 *     anything is enqueued: one bad image fails the whole call (AVIFGPU_ERR_BAD_PARAM or AVIFGPU_ERR_UNSUPPORTED)
 *     and nothing is launched.  count == 0 is AVIFGPU_OK with no launch; images of width or height 0 are skipped.
 *   - The outputs of different images must not overlap.
 *   - Like the device calls above it does not synchronise, may be captured into a CUDA graph under the same rules,
 *     and avifgpu_launch_count counts what it launched.  The first-use work (premultiply check, Gray16 LUT, step
 *     tables) is done once per call, outside a capture, for the batch's pixels.
 * Images the tuned integer planar kernel takes in a direct call (8/16-bit RGB(A) hosts into planar YCbCr, aligned
 * buffers, width >= 8) are converted in chunks of up to 64 images, at most two launches per chunk: one for every
 * image's aligned interior, one for every image's right strip and odd last 4:2:0 row.  Since API version 11 they also
 * write the semi-planar and MSB-aligned planes of avifgpu_encode_desc.dest_layout, an interleaved chroma plane aligned to
 * the paired stores (twice the planar chroma's alignment, at most 16 bytes).  Every other image takes one direct call,
 * after the chunks.
 */
AVIFGPU_EXPORT int avifgpu_encode_batch_device(avifgpu_context* ctx, const avifgpu_encode_desc* desc,
                                               const avifgpu_batch_image* images, int32_t count, void* cuda_stream);

/* The same for decodes: like `count` calls of avifgpu_decode_rows_device with y0 = 0 and nrows = height, one per image, in
 * order.  Images a tuned decode takes in a direct call go through chunks of up to 64 images, at most two launches
 * per chunk: the integer YCbCr one (8/16-bit hosts reading YCbCr 8/10/12-bit, straight or no alpha, aligned buffers,
 * width >= 8); since API version 8, the float YCbCr one (32-bit hosts reading YCbCr 10/12-bit with PQ, HLG or SMPTE 428,
 * straight or no alpha, aligned buffers, equal Cb / Cr strides, width >= 4; HLG once its divisions are verified); and,
 * since API version 9, the planar-RGB ones (lossless images: 8-bit planes into 8-bit hosts and 10/12-bit planes into
 * 16-bit hosts, or 10/12-bit planes with PQ, HLG or SMPTE 428 into 32-bit hosts; straight or no alpha, aligned buffers,
 * width >= 8).  Since API version 10 the YCbCr routes also take the semi-planar and MSB-aligned sources of
 * avifgpu_decode_desc.source_layout, an interleaved chroma plane aligned to the pair loads (twice the planar chroma's
 * alignment, at most 16 bytes).  Every other image -- monochrome, premultiplied alpha, 16-bit planes, a misaligned buffer --
 * takes one direct call, after the chunks.  The first-use work (the verified divisions) is done once per call, outside a capture. */
AVIFGPU_EXPORT int avifgpu_decode_batch_device(avifgpu_context* ctx, const avifgpu_decode_desc* desc,
                                               const avifgpu_batch_image* images, int32_t count, void* cuda_stream);

/* ---- the hot path: batches described in device memory ---------------------------------------------------------- */

/* Device workspace bytes a device-described batch of up to max_count images needs (1 <= max_count <= 4096).
 * Pure host arithmetic. */
AVIFGPU_EXPORT int avifgpu_batch_workspace_bytes(int32_t max_count, size_t* out_bytes);

/*
 * A batch whose image list and count are device memory, read when the work runs: one CUDA graph captured once converts
 * a different image set on every replay, and images made by earlier GPU work (a resize, a decoder writing into a pool)
 * need no copy to the host and no synchronisation.
 *   - Device inputs.  device_images (max_count avifgpu_batch_image records), *device_count and device_workspace are
 *     device memory, read on `cuda_stream` when the work runs, not when the call is made: write them earlier on the same
 *     stream, or in work ordered before it.  desc->width and desc->height are ignored.
 *   - Host checks, before any launch (each returns its status and launches nothing): ctx, desc, device_images,
 *     device_count or device_workspace NULL; desc invalid (validated as for the other calls, its size ignored);
 *     max_count outside [1, 4096]; workspace_bytes below avifgpu_batch_workspace_bytes(max_count).
 *   - Supported descriptions: encode, 8- or 16-bit RGB(A) hosts into planar YCbCr, any alpha state (since API version 11
 *     in any dest_layout); decode, 8-, 16- or
 *     (since API version 8) 32-bit hosts reading YCbCr, or (since API version 9) planar RGB, with no or straight alpha.
 *     Anything else -- monochrome, premultiplied alpha -- is AVIFGPU_ERR_UNSUPPORTED, with no launch.
 *   - Device-side checks.  With n = *device_count: n < 0 or n > max_count converts nothing and sets all max_count
 *     entries of device_status to AVIFGPU_ERR_BAD_PARAM.  Otherwise image i < n gets device_status[i] = 0, or
 *     AVIFGPU_ERR_BAD_PARAM when its width or height is negative, or when it is non-empty and its rows or a plane the
 *     description has is NULL (the host-described calls' checks); a rejected image is skipped and its outputs are not
 *     touched.  Images of width or height 0 are accepted and write nothing.  device_status may be NULL.
 *   - Outputs: every accepted image equals one *_rows_device call of the whole image, bit for bit.  The outputs of
 *     different images must not overlap.
 *   - Launches: exactly three per call, whatever the batch holds, n = 0 included (plan, interiors, edges);
 *     avifgpu_launch_count rises by 3.
 *   - Capture: the call may be captured under the device calls' rules.  The graph holds the description and the
 *     addresses of the records, count, workspace and status array, not their contents: a replay converts whatever those
 *     buffers hold at that moment.
 *   - First-use work: an encode makes the premultiply check outside a capture; call avifgpu_prepare_decode before
 *     capturing a decode.  An encode captured before the check, or an HLG decode into 32-bit hosts captured before its
 *     divisions are verified, sends every image through the edge kernel: the same output bit for bit, a slower kernel.
 *   - Workspace: one workspace must not serve two calls that can be in flight at the same time.  The library allocates
 *     nothing for this call.
 * Images the tuned integer, float or planar-RGB kernels take in a direct call have their aligned interior converted by the
 * interior kernel, their right strip and odd last 4:2:0 row by the edge kernel; every other image is one whole-image window of the edge
 * kernel, which runs the generic kernels' own per-site / per-pixel code.
 */
AVIFGPU_EXPORT int avifgpu_encode_batch_indirect(avifgpu_context* ctx, const avifgpu_encode_desc* desc,
                                                 const avifgpu_batch_image* device_images, const int32_t* device_count,
                                                 int32_t max_count, void* device_workspace, size_t workspace_bytes,
                                                 int32_t* device_status, void* cuda_stream);
AVIFGPU_EXPORT int avifgpu_decode_batch_indirect(avifgpu_context* ctx, const avifgpu_decode_desc* desc,
                                                 const avifgpu_batch_image* device_images, const int32_t* device_count,
                                                 int32_t max_count, void* device_workspace, size_t workspace_bytes,
                                                 int32_t* device_status, void* cuda_stream);

/* ---- content light level of batches (since API version 13) ------------------------------------------------------- */

/*
 * The batch calls plus each image's content light level: thumbnails, previews, image collections and burst or bracket
 * sets of HDR stills, every one of which carries its own `clli`.
 *   - Statistic: avifgpu_light_level, level(k) and avifgpu_content_light_level as in API version 12.  device_acc[i]
 *     (device memory, zeroed by the caller; calls add into it) gains exactly what one avifgpu_encode_rows_device_light_level
 *     call over image i whole (y0 = 0, nrows = height) adds.  Empty images, images the device-described call rejects
 *     (device_status[i] = AVIFGPU_ERR_BAD_PARAM) and every image of an out-of-range *device_count leave their entry as it is.
 *   - Planes: the host-described call writes, bit for bit, what avifgpu_encode_batch_device writes for the same images
 *     (one direct call per image), padding included; the device-described call writes what the direct call writes for
 *     every accepted image.
 *   - Descriptions: the host-described call accepts what avifgpu_encode_rows_device_light_level accepts (host_depth 32,
 *     AVIFGPU_TRANSFER_PQ; any layout, channel count, alpha state, chroma, down_filter, row_matrix, dest_layout); the
 *     device-described call the planar YCbCr part of that (AVIFGPU_LAYOUT_PLANAR_YCBCR, RGB or RGBA hosts, any
 *     dest_layout).  Anything else is AVIFGPU_ERR_UNSUPPORTED and launches nothing; a NULL device_acc is
 *     AVIFGPU_ERR_BAD_PARAM.  Every check of the plain calls applies as it stands (images validated before any launch,
 *     max_count, workspace size, NULLs).
 *   - Launches: RGB32f and RGBA32f images the direct light-level call tunes (planar YCbCr through the PQ compact step table,
 *     aligned buffers, width >= 4) go in chunks of up to 64 images, at most two launches per chunk (interiors, then right
 *     strips and odd last 4:2:0 rows); every other non-empty image takes one direct light-level call, with that call's
 *     route and launches, after the chunks.  The device-described call makes exactly three launches (plan, interiors,
 *     edges), n = 0 included.  avifgpu_launch_count counts them.
 *   - Capture: as for the device calls; the graph holds the accumulator array's address.  A call captured before
 *     avifgpu_prepare_encode has no step table and no level table and sends every image through the generic per-site code,
 *     which evaluates level(k) itself: the same planes and integers, a slower kernel.
 *   - Workspace: the device-described call's is sized by avifgpu_batch_workspace_bytes, as for the plain call.
 */
AVIFGPU_EXPORT int avifgpu_encode_batch_device_light_level(avifgpu_context* ctx, const avifgpu_encode_desc* desc,
                                                           const avifgpu_batch_image* images, int32_t count,
                                                           avifgpu_light_level* device_acc, void* cuda_stream);
AVIFGPU_EXPORT int avifgpu_encode_batch_indirect_light_level(avifgpu_context* ctx, const avifgpu_encode_desc* desc,
                                                             const avifgpu_batch_image* device_images, const int32_t* device_count,
                                                             int32_t max_count, void* device_workspace, size_t workspace_bytes,
                                                             int32_t* device_status, avifgpu_light_level* device_acc,
                                                             void* cuda_stream);

/* ---- content light level of host-pointer encodes (additions within API version 13) -------------------------------- */

/*
 * avifgpu_encode_rows, avifgpu_encode_rows_async and avifgpu_encode_rows_sharded plus the content light level of the rows
 * converted, added into a HOST accumulator: what an HDR save from host memory (the plug-in's row shuttle, a libheif
 * integrator) needs for its `clli`, with no second pass over the frame on the CPU.  These three calls were added within
 * API version 13: avifgpu_api_version() does not tell whether a library has them; look them up by symbol.
 *   - Same call as the plain one: the contract of avifgpu_encode_rows / _async / _sharded as it stands -- rows, planes,
 *     staging, the release of the previous asynchronous encode's rows, tickets and errors.  The planes are bit-identical
 *     to the plain call's, padding included, with the same number of kernel launches (avifgpu_launch_count).
 *   - The accumulator is host memory and may be pageable.  The caller zeroes it; calls add into it (max_code takes the
 *     max, level_sum and pixels add, reserved is never written), so several calls may share one accumulator -- the row
 *     blocks of one image, say.  For any row block *host_acc gains exactly what avifgpu_encode_rows_device_light_level
 *     adds over the same rows: the same integers, whatever slicing, pipeline slots or group members the call used.
 *   - When it is complete: for the synchronous and sharded calls, on an AVIFGPU_OK return.  For the asynchronous call,
 *     once avifgpu_wait() with a ticket covering the call, or avifgpu_synchronize(), has returned AVIFGPU_OK; until then
 *     the library may write it during any later host-pointer call on the context, on the caller's thread, and the caller
 *     must not read, write or free it -- exactly as for the destination planes.
 *   - Descriptions: what avifgpu_encode_rows_device_light_level accepts (host_depth 32, AVIFGPU_TRANSFER_PQ; any layout,
 *     channel count, alpha state, chroma, down_filter, row_matrix), with dest_layout 0 as for every host-pointer call.
 *   - Refusals: another description is AVIFGPU_ERR_UNSUPPORTED, a NULL host_acc AVIFGPU_ERR_BAD_PARAM, and every check of
 *     the plain call applies.  A refused call launches nothing, leaves *host_acc untouched and releases nothing.
 *   - Failures: a call that fails once it has started queueing work leaves the accumulators of this call and of earlier
 *     unfinished calls on the context unspecified, as the plain call leaves their planes; nothing writes them after the
 *     return.  The sharded call adds into *host_acc only when every member has succeeded: a failure leaves it untouched.
 */
AVIFGPU_EXPORT int avifgpu_encode_rows_light_level(avifgpu_context* ctx, const avifgpu_encode_desc* desc,
                                                   const void* host_rows, int64_t row_stride_bytes, int32_t y0, int32_t nrows,
                                                   const avifgpu_planes* dst, avifgpu_light_level* host_acc);
AVIFGPU_EXPORT int avifgpu_encode_rows_async_light_level(avifgpu_context* ctx, const avifgpu_encode_desc* desc,
                                                         const void* host_rows, int64_t row_stride_bytes, int32_t y0,
                                                         int32_t nrows, const avifgpu_planes* dst, avifgpu_light_level* host_acc,
                                                         int64_t* out_ticket);

/* ---- the hot path across several GPUs of one box (SURVEY.md 8e) ------------------------------------------------ */

/*
 * An image shards by row block (4:2:0: even boundaries, no halo; tables are replicated), so one process can put every
 * GPU of the box behind the same seam: the reference's row loops (WriteHeifImage.cpp:808-988 for a 16-bit RGBA save,
 * ReadHeifImage.cpp:290-400 for a float load, ...) have no cross-row state.  A shard group owns one context per device
 * and splits every call into `size` contiguous row blocks with avifgpu_shard_row_blocks().
 *
 *   host-pointer calls   block r is staged over device r's OWN PCIe link, converted there and copied back into the
 *                        caller's planes / rows: the PCIe-bound end-to-end rate scales with the number of links.
 *   device-pointer call  block r's rows already sit in device r's HBM; every device's conversion kernel stores its
 *                        part of the planes straight into the OWNER device's memory over NVLink / NVSwitch (peer
 *                        mapping inside the process), so the planar image is assembled when the kernels end -- the
 *                        "gather of the final planar buffer" is fused into the conversion, no collective pass.
 */
typedef struct avifgpu_shard_group avifgpu_shard_group;

/* One context per entry of device_ordinals[0 .. count) (distinct CUDA devices, compute capability 10.x); enables peer
 * access between them where the hardware offers it. */
AVIFGPU_EXPORT int avifgpu_shard_group_create(const int32_t* device_ordinals, int32_t count, avifgpu_shard_group** out_group);
AVIFGPU_EXPORT void avifgpu_shard_group_destroy(avifgpu_shard_group* group);
AVIFGPU_EXPORT int32_t avifgpu_shard_group_size(const avifgpu_shard_group* group);
/* The context of member `index` (owned by the group), e.g. for avifgpu_host_alloc or avifgpu_launch_count. */
AVIFGPU_EXPORT avifgpu_context* avifgpu_shard_group_context(avifgpu_shard_group* group, int32_t index);
/* 1 when member `from` can address member `to`'s memory (needed by the device-pointer call), else 0. */
AVIFGPU_EXPORT int avifgpu_shard_group_peer_access(const avifgpu_shard_group* group, int32_t from, int32_t to);
AVIFGPU_EXPORT const char* avifgpu_shard_group_last_error(const avifgpu_shard_group* group);
/* avifgpu_prepare_encode on every member (concurrently). */
AVIFGPU_EXPORT int avifgpu_shard_group_prepare_encode(avifgpu_shard_group* group, const avifgpu_encode_desc* desc);
/* Blocks until every member's work has finished. */
AVIFGPU_EXPORT int avifgpu_shard_group_synchronize(avifgpu_shard_group* group);

/* Row blocks of rows [y0, y0 + nrows) for `parts` members: contiguous, in order, every inner boundary even (a 2x2
 * chroma site never straddles two blocks); trailing blocks may be empty.  Pure host arithmetic. */
AVIFGPU_EXPORT int avifgpu_shard_row_blocks(int32_t y0, int32_t nrows, int32_t parts, int32_t* out_y0, int32_t* out_nrows);

/* avifgpu_encode_rows / avifgpu_decode_rows with the row block split across the group (same arguments, same result,
 * bit for bit).  y0 even for 4:2:0. */
AVIFGPU_EXPORT int avifgpu_encode_rows_sharded(avifgpu_shard_group* group, const avifgpu_encode_desc* desc,
                                               const void* host_rows, int64_t row_stride_bytes,
                                               int32_t y0, int32_t nrows, const avifgpu_planes* dst);
/* avifgpu_encode_rows_sharded plus the content light level of the rows, added into the host accumulator *host_acc (see
 * avifgpu_encode_rows_light_level): each member measures its row block into a partial of its own, and the partials are
 * added into *host_acc once every member has succeeded.  An addition within API version 13. */
AVIFGPU_EXPORT int avifgpu_encode_rows_sharded_light_level(avifgpu_shard_group* group, const avifgpu_encode_desc* desc,
                                                           const void* host_rows, int64_t row_stride_bytes,
                                                           int32_t y0, int32_t nrows, const avifgpu_planes* dst,
                                                           avifgpu_light_level* host_acc);
AVIFGPU_EXPORT int avifgpu_decode_rows_sharded(avifgpu_shard_group* group, const avifgpu_decode_desc* desc,
                                               const avifgpu_planes* src, int32_t y0, int32_t nrows,
                                               void* host_rows, int64_t row_stride_bytes);

/*
 * Device-resident frame, rows distributed: device_rows[r] / row_stride_bytes[r] = the first row of member r's block
 * (avifgpu_shard_row_blocks(0, desc->height, size)) in member r's memory.  owner_planes = whole-image planes in member
 * `owner`'s memory; every member must have peer access to it.  Enqueues one conversion per member on that member's
 * own stream and returns; avifgpu_shard_group_synchronize() (or the next sharded call) orders after it.
 */
AVIFGPU_EXPORT int avifgpu_encode_rows_sharded_device(avifgpu_shard_group* group, const avifgpu_encode_desc* desc,
                                                      const void* const* device_rows, const int64_t* row_stride_bytes,
                                                      const avifgpu_planes* owner_planes, int32_t owner);
/*
 * avifgpu_encode_rows_sharded_device plus the content light level of the whole image, added into *device_acc in the
 * owner's memory: a device-resident HDR frame spread over several GPUs gets its `clli` with no second pass.  An addition
 * within API version 13: look it up by symbol.
 *   - Same call as the plain one: arguments, row blocks, the peer-access requirement and enqueue-and-return as in
 *     avifgpu_encode_rows_sharded_device.  The planes are bit-identical to the plain call's, padding included.
 *   - Launches: every member's avifgpu_launch_count rises by what the plain call adds, and the owner's by one more, for
 *     the merge described below.
 *   - The accumulator is device memory of the owner, zeroed by the caller; calls add into it (max_code takes the max,
 *     level_sum and pixels add, reserved is never written).  It gains exactly what one
 *     avifgpu_encode_rows_device_light_level call over the whole image (y0 = 0, nrows = height) adds on one device, whatever
 *     the number of members and wherever the block boundaries fall.
 *   - How: each member with a non-empty block measures it on its own stream into a partial in its own memory and copies
 *     the partial into the owner's memory (no atomics across devices); the owner's stream then waits for every member and
 *     one single-warp kernel adds the partials into *device_acc.
 *   - When it is complete: after avifgpu_shard_group_synchronize(), like the planes.  Since the owner's stream waits for
 *     every member, work ordered after it -- avifgpu_synchronize() of the owner's context included -- sees both the
 *     accumulator and the planes complete.
 *   - Descriptions: what avifgpu_encode_rows_device_light_level accepts (host_depth 32, AVIFGPU_TRANSFER_PQ; any layout,
 *     channel count, alpha state, chroma, down_filter, row_matrix), with dest_layout 0 as for every sharded call.
 *   - Refusals, before anything is enqueued on any member and leaving *device_acc untouched: another description is
 *     AVIFGPU_ERR_UNSUPPORTED, a NULL device_acc AVIFGPU_ERR_BAD_PARAM, and every check of the plain call applies (an
 *     owner outside the group, a member with no peer access to the owner, ...).
 *   - Failures: the merge is enqueued only once every member's launch has succeeded, so a call that fails while its
 *     members are being enqueued leaves *device_acc untouched, and the planes as the plain call leaves them.
 */
AVIFGPU_EXPORT int avifgpu_encode_rows_sharded_device_light_level(avifgpu_shard_group* group, const avifgpu_encode_desc* desc,
                                                                  const void* const* device_rows, const int64_t* row_stride_bytes,
                                                                  const avifgpu_planes* owner_planes, int32_t owner,
                                                                  avifgpu_light_level* device_acc);

/* ---- preparation (optional) --------------------------------------------------------------------------- */

/* Statistics of the exact float->code step table behind a float-host encode configuration
 * (avif-format_b200/csrc/curve_tables.h).  The table is derived on the device from the exact curve by sweeping
 * every non-negative float, and verified against it the same way, the first time a configuration is used. */
typedef struct avifgpu_curve_stats
{
    int32_t applicable;          /* 1 if this description uses a step table (float host, PQ or SMPTE 428) */
    int32_t valid;               /* 1 if the table was built and verified; 0 -> the exact generic kernel is used */
    int32_t steps;               /* thresholds found */
    int32_t bands;               /* thresholds with a non-empty fuzzy (non-monotone) band */
    uint32_t widest_band_ulps;
    int32_t bucket_count;
    uint64_t swept_inputs;       /* floats evaluated by the sweep */
    uint64_t in_band_inputs;     /* floats the kernel hands to the exact path */
    uint64_t verify_mismatches;  /* must be 0 for valid == 1 */
    double build_ms;
} avifgpu_curve_stats;

/* Builds whatever device-side tables `desc` needs, now.  out_stats may be NULL.
 * The exact step tables of the float PQ / SMPTE 428 encode path cost about 40 ms to build and verify (once per
 * context and configuration) and make that path several times faster, which pays off after roughly two gigapixels:
 * frame pipelines call this up front; a caller that converts one image does not need to (see
 * avifgpu_set_table_autobuild). */
AVIFGPU_EXPORT int avifgpu_prepare_encode(avifgpu_context* ctx, const avifgpu_encode_desc* desc,
                                          avifgpu_curve_stats* out_stats);

/* Does now the first-use work a decode of `desc` would do: the on-device checks behind the tuned float decode's HLG and
 * PQ divisions and the YCbCr decodes' green-channel division (once per context and configuration).
 * Optional, except before capturing a decode into a CUDA graph. */
AVIFGPU_EXPORT int avifgpu_prepare_decode(avifgpu_context* ctx, const avifgpu_decode_desc* desc);

/* Without avifgpu_prepare_encode() the encode calls convert with the exact kernel (glibc-identical powf per sample)
 * until `pixels` pixels of one configuration have gone through this context, and build the step tables then.
 * Default AVIFGPU_TABLE_AUTOBUILD_DEFAULT; 0 = build at first use; negative = never build automatically.
 * Results are bit-identical either way. */
#define AVIFGPU_TABLE_AUTOBUILD_DEFAULT (((int64_t)1) << 31)
AVIFGPU_EXPORT int avifgpu_set_table_autobuild(avifgpu_context* ctx, int64_t pixels);

/* ---- primitive-level entry points (parity gates G2/G5; not on the plug-in's call path) -------------- */

typedef enum avifgpu_function
{
    AVIFGPU_FN_LINEAR_TO_PQ = 0,      /* param = peak nits  ColorTransfer.cpp:69-92   */
    AVIFGPU_FN_PQ_TO_LINEAR = 1,      /* param = peak nits  ColorTransfer.cpp:94-117  */
    AVIFGPU_FN_LINEAR_TO_SMPTE428 = 2,/*                    ColorTransfer.cpp:119-127 */
    AVIFGPU_FN_SMPTE428_TO_LINEAR = 3,/*                    ColorTransfer.cpp:129-139 */
    AVIFGPU_FN_HLG_TO_LINEAR = 4,     /*                    ColorTransfer.cpp:166-190 */
    AVIFGPU_FN_LINEAR_TO_HLG = 5,     /*                    ColorTransfer.cpp:141-164 */
    AVIFGPU_FN_POWF = 6,              /* param = exponent   libm powf                 */
    AVIFGPU_FN_EXPF = 7,              /*                    libm expf                 */
    AVIFGPU_FN_LOGF = 8               /*                    libm logf                 */
} avifgpu_function;

/* out[i] = fn(in[i], param) for n floats; in/out are HOST pointers (copied through the device). */
AVIFGPU_EXPORT int avifgpu_transfer_f32(avifgpu_context* ctx, int32_t function, float param,
                                        const float* in, float* out, size_t n);

/* ApplyHLGOOTF (ColorTransfer.cpp:192-205; inverse = 0) or ApplyInverseHLGOOTF (ColorTransfer.cpp:207-220; inverse = 1)
 * over `pixels` interleaved RGB float triples, luma coefficients from GetHLGLumaCoefficients(color_primaries)
 * (ColorTransfer.cpp:31-45).  rgb_in / rgb_out are HOST pointers (may alias). */
AVIFGPU_EXPORT int avifgpu_hlg_ootf_f32(avifgpu_context* ctx, int32_t inverse, int32_t color_primaries, float display_gamma,
                                        float nominal_peak_nits, const float* rgb_in, float* rgb_out, size_t pixels);

#ifdef __cplusplus
}
#endif

#endif /* AVIFGPU_H */
