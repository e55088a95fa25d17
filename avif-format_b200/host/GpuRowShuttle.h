// GpuRowShuttle.h -- the plug-in's row shuttle entry points, backed by the H100 library (include/avifgpu.h).
//
// Same names, arguments and error behaviour as the reference's
//     CreateHeifImage{Gray,RGB}{Eight,Sixteen,ThirtyTwo}Bit   (src/common/WriteHeifImage.h:29-63)
//     ReadHeifImage{Gray,RGB}{Eight,Sixteen,ThirtyTwo}Bit     (src/common/ReadHeifImage.h:27-63)
// so the call sites in Write.cpp:303-336 and Read.cpp:587-630 do not change.  Differences, all behind the seam:
//   * the host is asked for blocks of rows (theRect top..bottom spanning many rows -- the FormatRecord protocol
//     allows any rectangle) into a pinned staging buffer instead of one row at a time, abortProc is still polled
//     once per block, and each block is one avifgpu_encode_rows / avifgpu_decode_rows call;
//   * colour images are handed to libheif as planar YCbCr at the encoder's chroma format (matrix + down-filter
//     fused on the GPU) instead of interleaved RGB, so heif_context_encode_image's own colour conversion
//     degenerates to a no-op (SURVEY.md 8b); gray images keep the reference's Y (+ Alpha) planes;
//   * two pinned row buffers alternate: while the GPU converts and copies block k (avifgpu_encode_rows_async), the host
//     fills block k+1 through advanceState; on the read side block k+1 converts while the host takes block k;
//   * the optional ICC row transform (ColorProfileConversion::ConvertRow, lcms2: WriteHeifImage.cpp:651, 830, 1015) stays
//     a host-side step over the staged rows.  In the plug-in tree (AVIFGPU_HOST_USE_PLUGIN_HEADERS) the shuttle builds the
//     plug-in's own ColorProfileConversion; elsewhere a RowTransformFactory supplies it.  When the document carries a
//     profile that MAY need converting (HostMetadata.cpp:63-69, ColorProfileConversion.cpp:107-109, 143) and nothing can
//     decide or do it, the shuttle throws OSErrException(formatBadParameters) -- never unconverted pixels.
// One thread at a time, like the plug-in itself (Photoshop calls PluginMain on one thread): the shared context and the
// settings below are process-wide and not synchronised.
// Errors surface exactly like the reference's: OSErrException (userCanceledErr, formatBadParameters, ...),
// std::runtime_error for unsupported configurations, std::bad_alloc for memory.
#ifndef AVIFGPU_HOST_GPU_ROW_SHUTTLE_H
#define AVIFGPU_HOST_GPU_ROW_SHUTTLE_H

#include "compat/PluginTypes.h"

#include <stdint.h>

struct avifgpu_context;

namespace avifgpu_host
{

// Process-wide context for the plug-in (Photoshop calls PluginMain on one thread).  Throws
// OSErrException(errPlugInHostInsufficient) when there is no usable H100: there is no CPU fallback.
avifgpu_context* SharedContext();
void ReleaseSharedContext();

// Upper bound on the rows requested from / delivered to the host per advanceState call (rounded down to an even
// count; default 4096).  The actual block is also bounded by the staging budget.
void SetRowsPerBlock(int32 rows);

// Page-locked bytes per staging buffer (there are two; default 64 MiB each, at least two rows).  A 300 000-pixel RGBA32f
// row is 4.8 MB: the block shrinks, the allocation does not grow.
void SetStagingBudgetBytes(int64_t bytes);

// Several GPUs of this box behind the same entry points (avifgpu_shard_group): every row block is cut into one part per
// device, each staged over that device's own PCIe link.  count <= 1 returns to the single shared context.
void UseDevices(const int32_t* deviceOrdinals, int32_t count);

// The reference's per-row colour-profile conversion (ColorProfileConversion.cpp:159-186), applied in place to every
// staged host row before the conversion.
struct RowTransform
{
    virtual ~RowTransform() = default;
    virtual void ConvertRow(void* row, uint32_t pixelsPerLine, uint32_t bytesPerLine) = 0;
};

// Called once per save when the document has colour-profile metadata and the reference's own test says a conversion
// may be required.  hostBitsPerChannel 8 / 16 / 32; for 32 `transferFunction` is the save option, otherwise ignored.
// Returns the transform, or nullptr when the profile already is what the file will be tagged with (IsSRGBColorProfile /
// IsRec2020ColorProfile in the reference).  Throwing is allowed ("Unable to load the document color profile.").
using RowTransformFactory = RowTransform* (*)(FormatRecordPtr formatRecord, bool hasAlpha, int hostBitsPerChannel,
                                             ColorTransferFunction transferFunction, bool keepEmbeddedColorProfile, void* user);
void SetRowTransformFactory(RowTransformFactory factory, void* user);

// HDR saves (32-bit documents, PQ / SMPTE 428) of a document whose profile is a matrix / TRC RGB profile with linear tone
// curves: the conversion to linear Rec.2020 is a 3x3 matrix, applied on the GPU ahead of the conversion
// (avifgpu_icc_to_rec2020_linear_matrix, avifgpu_encode_desc.row_matrix) instead of a host-side row transform.  On by
// default where the FormatRecord holds the profile bytes; any other profile falls through to the RowTransformFactory.
void SetGpuRowMatrixEnabled(bool enabled);

// 32-bit PQ saves (CreateHeifImageRGBThirtyTwoBit / CreateHeifImageGrayThirtyTwoBit with the PQ transfer) measure the
// image's content light level while they convert (avifgpu_encode_rows_async_light_level, or the sharded form under
// UseDevices) and attach it to the returned image with heif_image_set_content_light_level, which libheif writes as the
// `clli` property.  It covers the pixels encoded: after the host row transform and the GPU row matrix.  Off by default.
void SetContentLightLevelEnabled(bool enabled);

// The content light level (cd/m2) attached by the last CreateHeifImage* call; measured == false when that call attached
// none (another save, the setting off, a cancelled or failed save).
struct ContentLightLevel
{
    bool measured;
    uint16_t maxCll;
    uint16_t maxFall;
};
ContentLightLevel LastContentLightLevel();

// Where the time of the last CreateHeifImage* / ReadHeifImage* call went (seconds).
struct ShuttleTimes
{
    double total;        // inside the entry point
    double host;         // inside formatRecord->advanceState / abortProc (the host producing or consuming rows)
    double transform;    // inside the row transform
    int32 blocks;
    int32 rowsPerBlock;
};
ShuttleTimes LastShuttleTimes();

} // namespace avifgpu_host

ScopedHeifImage CreateHeifImageGrayEightBit(FormatRecordPtr formatRecord, AlphaState alphaState, const VPoint& imageSize, const SaveUIOptions& saveOptions);
ScopedHeifImage CreateHeifImageGraySixteenBit(FormatRecordPtr formatRecord, AlphaState alphaState, const VPoint& imageSize, const SaveUIOptions& saveOptions);
ScopedHeifImage CreateHeifImageGrayThirtyTwoBit(FormatRecordPtr formatRecord, AlphaState alphaState, const VPoint& imageSize, const SaveUIOptions& saveOptions);
ScopedHeifImage CreateHeifImageRGBEightBit(FormatRecordPtr formatRecord, AlphaState alphaState, const VPoint& imageSize, const SaveUIOptions& saveOptions);
ScopedHeifImage CreateHeifImageRGBSixteenBit(FormatRecordPtr formatRecord, AlphaState alphaState, const VPoint& imageSize, const SaveUIOptions& saveOptions);
ScopedHeifImage CreateHeifImageRGBThirtyTwoBit(FormatRecordPtr formatRecord, AlphaState alphaState, const VPoint& imageSize, const SaveUIOptions& saveOptions);

void ReadHeifImageGrayEightBit(const heif_image* image, AlphaState alphaState, const heif_color_profile_nclx* nclxProfile, FormatRecordPtr formatRecord);
void ReadHeifImageGraySixteenBit(const heif_image* image, AlphaState alphaState, const heif_color_profile_nclx* nclxProfile, FormatRecordPtr formatRecord);
void ReadHeifImageGrayThirtyTwoBit(const heif_image* image, AlphaState alphaState, const heif_color_profile_nclx* nclxProfile, const LoadUIOptions& loadOptions, FormatRecordPtr formatRecord);
void ReadHeifImageRGBEightBit(const heif_image* image, AlphaState alphaState, const heif_color_profile_nclx* nclxProfile, FormatRecordPtr formatRecord);
void ReadHeifImageRGBSixteenBit(const heif_image* image, AlphaState alphaState, const heif_color_profile_nclx* nclxProfile, FormatRecordPtr formatRecord);
void ReadHeifImageRGBThirtyTwoBit(const heif_image* image, AlphaState alphaState, const heif_color_profile_nclx* nclxProfile, const LoadUIOptions& loadOptions, FormatRecordPtr formatRecord);

#endif
