// GpuRowShuttle.cpp -- see GpuRowShuttle.h.  Host-side C++ only: every pixel goes through the C ABI of
// libavifgpu.so (include/avifgpu.h); this file owns the FormatRecord protocol, the heif_image plumbing and the
// translation of status codes back into the exceptions the plug-in's session functions catch
// (Write.cpp:345-364, Read.cpp:659-678).
#include "GpuRowShuttle.h"

#include "../../include/avifgpu.h"

#include <algorithm>
#include <chrono>
#include <cstring>
#include <limits>
#include <memory>
#include <new>
#include <string>

#if defined(AVIFGPU_HOST_USE_PLUGIN_HEADERS)
#include "ColorProfileConversion.h"
#include "HostMetadata.h"
#endif

namespace
{
    avifgpu_context* g_context = nullptr;
    avifgpu_shard_group* g_group = nullptr; // several GPUs (avifgpu_host::UseDevices), else nullptr
    int32 g_rowsPerBlock = 4096;
    int64_t g_stagingBudget = 64ll << 20;
    avifgpu_host::RowTransformFactory g_transformFactory = nullptr;
    void* g_transformUser = nullptr;
    avifgpu_host::ShuttleTimes g_times{};
    bool g_gpuRowMatrix = true;
    bool g_contentLightLevel = false;
    avifgpu_host::ContentLightLevel g_lastLightLevel{};

    using Clock = std::chrono::steady_clock;
    double Seconds(Clock::time_point from) { return std::chrono::duration<double>(Clock::now() - from).count(); }

    // Accumulates the time spent inside the host's callbacks.
    struct HostTimer
    {
        Clock::time_point start = Clock::now();
        ~HostTimer() { g_times.host += Seconds(start); }
    };

    // avifgpu status -> the exception the reference would have thrown for the same condition.
    void ThrowIfFailed(avifgpu_context* ctx, int status)
    {
        if (status == AVIFGPU_OK)
        {
            return;
        }
        const std::string message = avifgpu_last_error(ctx);
        switch (status)
        {
        case AVIFGPU_ERR_BAD_PARAM: throw OSErrException(formatBadParameters);
        case AVIFGPU_ERR_NO_DEVICE: throw OSErrException(errPlugInHostInsufficient);
        case AVIFGPU_ERR_OOM: throw std::bad_alloc();
        case AVIFGPU_ERR_CANCELED: throw OSErrException(userCanceledErr);
        default: throw std::runtime_error(message.empty() ? avifgpu_status_string(status) : message);
        }
    }

    // Utilities.cpp:382-416
    VPoint GetImageSizeOf(const FormatRecordPtr formatRecord)
    {
        VPoint size;
        if (formatRecord->HostSupports32BitCoordinates && formatRecord->PluginUsing32BitCoordinates)
        {
            size.h = formatRecord->imageSize32.h;
            size.v = formatRecord->imageSize32.v;
        }
        else
        {
            size.h = formatRecord->imageSize.h;
            size.v = formatRecord->imageSize.v;
        }
        return size;
    }

    void SetRectOf(FormatRecordPtr formatRecord, int32 top, int32 left, int32 bottom, int32 right)
    {
        if (formatRecord->HostSupports32BitCoordinates && formatRecord->PluginUsing32BitCoordinates)
        {
            formatRecord->theRect32.top = top;
            formatRecord->theRect32.left = left;
            formatRecord->theRect32.bottom = bottom;
            formatRecord->theRect32.right = right;
        }
        else
        {
            formatRecord->theRect.top = static_cast<int16>(top);
            formatRecord->theRect.left = static_cast<int16>(left);
            formatRecord->theRect.bottom = static_cast<int16>(bottom);
            formatRecord->theRect.right = static_cast<int16>(right);
        }
    }

    int HeifBitDepth(ImageBitDepth depth)
    {
        // WriteHeifImage.cpp:41-61
        switch (depth)
        {
        case ImageBitDepth::Eight: return 8;
        case ImageBitDepth::Ten: return 10;
        case ImageBitDepth::Twelve: return 12;
        default: throw OSErrException(formatCannotRead);
        }
    }

    // Pinned staging rows owned by the library; replaces the plug-in's one-row ScopedBufferSuiteBuffer.
    class PinnedRows
    {
    public:
        PinnedRows(avifgpu_context* ctx, size_t bytes) : context(ctx)
        {
            ThrowIfFailed(ctx, avifgpu_host_alloc(ctx, bytes, &memory));
        }
        ~PinnedRows() { avifgpu_host_free(context, memory); }
        PinnedRows(const PinnedRows&) = delete;
        PinnedRows& operator=(const PinnedRows&) = delete;
        void* get() const { return memory; }

    private:
        avifgpu_context* context;
        void* memory = nullptr;
    };

    // Rows per advanceState: bounded by the caller's setting and by the page-locked byte budget (an even count, at
    // least two rows -- a 4:2:0 block must hold whole row pairs).  With several GPUs a block feeds all of them.
    int32 BlockRows(int32 height, int64_t rowBytes)
    {
        const int64_t budget = g_stagingBudget * (g_group != nullptr ? avifgpu_shard_group_size(g_group) : 1);
        int64_t rows = std::max<int64_t>(rowBytes, 1) > 0 ? budget / std::max<int64_t>(rowBytes, 1) : height;
        rows = std::min<int64_t>(rows, g_rowsPerBlock);
        rows = std::max<int64_t>(rows & ~1ll, 2);
        return static_cast<int32>(std::min<int64_t>(rows, std::max<int32>(height, 1)));
    }

    // Two page-locked row buffers, kept between calls (page-locking 128 MiB costs tens of milliseconds -- more than
    // converting an 8K frame -- so the shuttle pays it once per process, not once per image; ReleaseSharedContext frees
    // them).  When the allocation fails the block is halved until it fits (down to two rows).
    struct StagingCache
    {
        std::unique_ptr<PinnedRows> buffer[2];
        size_t bytes = 0;
        avifgpu_context* owner = nullptr;
        void Release()
        {
            buffer[0].reset();
            buffer[1].reset();
            bytes = 0;
            owner = nullptr;
        }
    };
    StagingCache g_staging;

    struct StagingPair
    {
        PinnedRows* buffer[2] = { nullptr, nullptr };
        int32 blockRows = 0;
        StagingPair(avifgpu_context* ctx, int64_t rowBytes, int32 height)
        {
            blockRows = BlockRows(height, rowBytes);
            for (;;)
            {
                const size_t bytes = static_cast<size_t>(std::max<int64_t>(rowBytes, 1)) * blockRows;
                if (g_staging.owner == ctx && g_staging.bytes >= bytes)
                {
                    break; // the buffers of an earlier call are large enough
                }
                try
                {
                    g_staging.Release();
                    g_staging.buffer[0].reset(new PinnedRows(ctx, bytes));
                    g_staging.buffer[1].reset(new PinnedRows(ctx, bytes));
                    g_staging.bytes = bytes;
                    g_staging.owner = ctx;
                    break;
                }
                catch (const std::bad_alloc&)
                {
                    g_staging.Release();
                    if (blockRows <= 2)
                    {
                        throw;
                    }
                    blockRows = std::max<int32>((blockRows / 2) & ~1, 2);
                }
            }
            buffer[0] = g_staging.buffer[0].get();
            buffer[1] = g_staging.buffer[1].get();
        }
    };

    // Nothing issued on the context may outlive the buffers and planes of a call, whichever way the call is left.
    struct DrainOnExit
    {
        avifgpu_context* ctx;
        ~DrainOnExit() { avifgpu_wait(ctx, 0); }
    };

    // HostMetadata.cpp:63-69 (the handle-suite availability test is the plug-in's; the compat record has no suites).
    bool RecordHasColorProfile(const FormatRecordPtr formatRecord)
    {
#if defined(AVIFGPU_HOST_USE_PLUGIN_HEADERS)
        return HasColorProfileMetadata(formatRecord);
#else
        return formatRecord->canUseICCProfiles && formatRecord->iCCprofileData != nullptr && formatRecord->iCCprofileSize > 0;
#endif
    }

#if defined(AVIFGPU_HOST_USE_PLUGIN_HEADERS)
    // The plug-in's own converter behind the RowTransform interface.
    struct PluginRowTransform final : avifgpu_host::RowTransform
    {
        ColorProfileConversion converter;
        PluginRowTransform(FormatRecordPtr record, bool hasAlpha, ColorTransferFunction transfer, bool keep) : converter(record, hasAlpha, transfer, keep) {}
        PluginRowTransform(FormatRecordPtr record, bool hasAlpha, int hostBits, bool keep) : converter(record, hasAlpha, hostBits, keep) {}
        void ConvertRow(void* row, uint32_t pixelsPerLine, uint32_t bytesPerLine) override { converter.ConvertRow(row, pixelsPerLine, bytesPerLine); }
    };
#endif

    // The per-save colour-profile step of CreateHeifImageRGB*Bit (WriteHeifImage.cpp:651, 830, 1015), or nullptr when the
    // reference would not convert.  Gray saves never convert (WriteHeifImage.cpp:169-627 construct no converter).
    // `desc` receives the GPU form of the step when the profile allows it (a 3x3 matrix ahead of the conversion,
    // avifgpu_encode_desc.row_matrix) -- then no host-side transform is returned.
    std::unique_ptr<avifgpu_host::RowTransform> MakeRowTransform(FormatRecordPtr formatRecord, bool gray, bool hasAlpha, int hostDepth,
                                                                 const SaveUIOptions& saveOptions, avifgpu_encode_desc* desc)
    {
        if (gray || !RecordHasColorProfile(formatRecord))
        {
            return nullptr;
        }
        // ColorProfileConversion.cpp:107 (32-bit hosts) / :143 (8 and 16-bit hosts)
        const bool mayRequireConversion = hostDepth == 32 ? (saveOptions.hdrTransferFunction != ColorTransferFunction::Clip || !saveOptions.keepColorProfile)
                                                          : !saveOptions.keepColorProfile;
        if (!mayRequireConversion)
        {
            return nullptr;
        }
#if !defined(AVIFGPU_HOST_USE_PLUGIN_HEADERS)
        // HDR save of a linear-light document in a matrix profile: the whole lcms2 transform is one 3x3 matrix, which the
        // GPU applies ahead of the conversion (SURVEY.md 8f-3).  (In the plug-in tree iCCprofileData is a Handle and the
        // plug-in's own lcms2 converter below is the default; the compat record holds the profile bytes directly.)
        if (g_gpuRowMatrix && hostDepth == 32 && saveOptions.hdrTransferFunction != ColorTransferFunction::Clip)
        {
            float matrix[9];
            int32_t alreadyRec2020 = 0;
            if (avifgpu_icc_to_rec2020_linear_matrix(formatRecord->iCCprofileData, static_cast<size_t>(formatRecord->iCCprofileSize), matrix,
                                                     &alreadyRec2020) == AVIFGPU_OK)
            {
                if (!alreadyRec2020) // ColorProfileConversion.cpp:128-131: a Rec.2020 document is not converted
                {
                    desc->row_matrix_enabled = 1;
                    std::memcpy(desc->row_matrix, matrix, sizeof(matrix));
                }
                return nullptr;
            }
        }
#else
        (void)desc;
#endif
        if (g_transformFactory != nullptr)
        {
            return std::unique_ptr<avifgpu_host::RowTransform>(
                g_transformFactory(formatRecord, hasAlpha, hostDepth, saveOptions.hdrTransferFunction, saveOptions.keepColorProfile, g_transformUser));
        }
#if defined(AVIFGPU_HOST_USE_PLUGIN_HEADERS)
        if (hostDepth == 32)
        {
            return std::unique_ptr<avifgpu_host::RowTransform>(new PluginRowTransform(formatRecord, hasAlpha, saveOptions.hdrTransferFunction, saveOptions.keepColorProfile));
        }
        return std::unique_ptr<avifgpu_host::RowTransform>(new PluginRowTransform(formatRecord, hasAlpha, hostDepth, saveOptions.keepColorProfile));
#else
        // A profile that may need converting and nobody to decide or do it: an error, never unconverted pixels tagged sRGB / BT.2020.
        throw OSErrException(formatBadParameters);
#endif
    }

    // Restores the caller's formatRecord->data / rowBytes when the shuttle leaves (normally or by exception).
    struct RecordDataGuard
    {
        FormatRecordPtr record;
        void* data;
        int32 rowBytes;
        explicit RecordDataGuard(FormatRecordPtr r) : record(r), data(r->data), rowBytes(r->rowBytes) {}
        ~RecordDataGuard()
        {
            record->data = data;
            record->rowBytes = rowBytes;
        }
    };

    avifgpu_nclx ToNclx(const heif_color_profile_nclx* profile)
    {
        avifgpu_nclx out{};
        if (profile != nullptr)
        {
            out.present = 1;
            out.color_primaries = static_cast<int32_t>(profile->color_primaries);
            out.transfer_characteristics = static_cast<int32_t>(profile->transfer_characteristics);
            out.matrix_coefficients = static_cast<int32_t>(profile->matrix_coefficients);
            out.full_range_flag = profile->full_range_flag ? 1 : 0;
        }
        return out;
    }

    // ---- encode --------------------------------------------------------------------------------------------------

    // Stamps g_times.total when an entry point is left.
    struct CallTimer
    {
        Clock::time_point start = Clock::now();
        CallTimer() { g_times = avifgpu_host::ShuttleTimes{}; }
        ~CallTimer() { g_times.total = Seconds(start); }
    };

    ScopedHeifImage EncodeThroughGpu(FormatRecordPtr formatRecord, AlphaState alphaState, const VPoint& imageSize,
                                     const SaveUIOptions& saveOptions, int hostDepth, bool gray)
    {
        CallTimer callTimer;
        g_lastLightLevel = avifgpu_host::ContentLightLevel{};
        avifgpu_context* ctx = avifgpu_host::SharedContext();
        const bool hasAlpha = alphaState != AlphaState::None;
        const int bitDepth = HeifBitDepth(saveOptions.imageBitDepth);
        const bool measure = g_contentLightLevel && hostDepth == 32 && saveOptions.hdrTransferFunction == ColorTransferFunction::PQ;
#if !defined(AVIFGPU_HOST_USE_PLUGIN_HEADERS)
        if (measure && heif_image_set_content_light_level == nullptr) // compat/PluginTypes.h declares it weak
        {
            throw std::runtime_error("the libheif linked in has no heif_image_set_content_light_level");
        }
#endif
        const int channels = (gray ? 1 : 3) + (hasAlpha ? 1 : 0);

        avifgpu_encode_desc desc{};
        desc.struct_size = sizeof(desc);
        desc.width = imageSize.h;
        desc.height = imageSize.v;
        desc.host_depth = hostDepth;
        desc.host_channels = channels;
        desc.alpha_state = static_cast<int32_t>(alphaState);
        desc.image_bit_depth = bitDepth;
        desc.transfer = static_cast<int32_t>(saveOptions.hdrTransferFunction);
        desc.pq_peak_nits = saveOptions.pq.nominalPeakBrightness;
        desc.down_filter = AVIFGPU_DOWN_FILTER_BOX;
        desc.gray16_curve = AVIFGPU_GRAY16_LUT;

        heif_image* raw = nullptr;
        heif_chroma chroma = heif_chroma_monochrome;
        if (gray)
        {
            desc.layout = AVIFGPU_LAYOUT_REFERENCE; // Y (+ Alpha) planes, WriteHeifImage.cpp:175-194
            LibHeifException::ThrowIfError(heif_image_create(imageSize.h, imageSize.v, heif_colorspace_monochrome, heif_chroma_monochrome, &raw));
        }
        else
        {
            desc.layout = AVIFGPU_LAYOUT_PLANAR_YCBCR;
            // Write.cpp:96-120: lossless forces 4:4:4; otherwise the save option picks the encoder's chroma format.
            if (saveOptions.lossless)
            {
                chroma = heif_chroma_444;
            }
            else
            {
                switch (saveOptions.chromaSubsampling)
                {
                case ChromaSubsampling::Yuv420: chroma = heif_chroma_420; break;
                case ChromaSubsampling::Yuv422: chroma = heif_chroma_422; break;
                case ChromaSubsampling::Yuv444: chroma = heif_chroma_444; break;
                default: throw OSErrException(formatBadParameters);
                }
            }
            desc.chroma = static_cast<int32_t>(chroma);
            // WriteMetadata.cpp:107-149: the matrix the file will be tagged with
            desc.nclx.present = 1;
            desc.nclx.full_range_flag = 1;
            if (hostDepth == 32 && saveOptions.hdrTransferFunction != ColorTransferFunction::Clip)
            {
                desc.nclx.color_primaries = 9;
                desc.nclx.transfer_characteristics = saveOptions.hdrTransferFunction == ColorTransferFunction::PQ ? 16 : 17;
                desc.nclx.matrix_coefficients = 9;
            }
            else
            {
                desc.nclx.color_primaries = 1;
                desc.nclx.transfer_characteristics = 13;
                desc.nclx.matrix_coefficients = 6;
            }
            if (saveOptions.lossless)
            {
                desc.nclx.matrix_coefficients = 0;
            }
            LibHeifException::ThrowIfError(heif_image_create(imageSize.h, imageSize.v, heif_colorspace_YCbCr, chroma, &raw));
        }
        ScopedHeifImage image(raw);

        avifgpu_planes planes{};
        auto addPlane = [&](heif_channel channel, int index, int width, int height)
        {
            LibHeifException::ThrowIfError(heif_image_add_plane(image.get(), channel, width, height, bitDepth));
            int stride = 0;
            planes.data[index] = heif_image_get_plane(image.get(), channel, &stride);
            planes.stride[index] = stride;
        };
        addPlane(heif_channel_Y, 0, imageSize.h, imageSize.v);
        if (!gray)
        {
            const int cw = (chroma == heif_chroma_444) ? imageSize.h : (imageSize.h + 1) / 2;
            const int ch = (chroma == heif_chroma_420) ? (imageSize.v + 1) / 2 : imageSize.v;
            addPlane(heif_channel_Cb, 1, cw, ch);
            addPlane(heif_channel_Cr, 2, cw, ch);
        }
        if (hasAlpha)
        {
            addPlane(heif_channel_Alpha, 3, imageSize.h, imageSize.v);
        }

        // No avifgpu_prepare_encode() here: one image goes through the exact kernel (PCIe, not the kernel, bounds a
        // single save); the library builds its step tables by itself once a context has seen enough pixels.

        const int64_t rowBytes = static_cast<int64_t>(imageSize.h) * avifgpu_encode_host_col_bytes(&desc);
        if (rowBytes > std::numeric_limits<int32>::max())
        {
            throw std::bad_alloc(); // Write.cpp:286-295
        }
        std::unique_ptr<avifgpu_host::RowTransform> transform = MakeRowTransform(formatRecord, gray, hasAlpha, hostDepth, saveOptions, &desc);
        StagingPair staging(ctx, rowBytes, imageSize.v);
        const int32 blockRows = staging.blockRows;
        g_times.rowsPerBlock = blockRows;
        RecordDataGuard guard(formatRecord);
        avifgpu_light_level light{}; // one accumulator for every block of the image; outlives the drain below
        DrainOnExit drain{ ctx };
        formatRecord->rowBytes = static_cast<int32>(rowBytes);

        int32 block = 0;
        for (int32 top = 0; top < imageSize.v; top += blockRows, ++block)
        {
            void* rows = staging.buffer[block & 1]->get();
            const int32 bottom = std::min(top + blockRows, imageSize.v);
            {
                HostTimer timer;
                if (formatRecord->abortProc())
                {
                    throw OSErrException(userCanceledErr); // WriteHeifImage.cpp:208-211, once per block here
                }
                SetRectOf(formatRecord, top, 0, bottom, imageSize.h);
                formatRecord->data = rows;
                OSErrException::ThrowIfError(formatRecord->advanceState()); // the host fills rows [top, bottom)
            }
            if (transform)
            {
                const Clock::time_point start = Clock::now();
                for (int32 y = 0; y < bottom - top; ++y)
                {
                    // WriteHeifImage.cpp:1028-1031: converter.ConvertRow(formatRecord->data, imageSize.h, formatRecord->rowBytes)
                    transform->ConvertRow(static_cast<uint8_t*>(rows) + static_cast<int64_t>(y) * rowBytes, static_cast<uint32_t>(imageSize.h),
                                          static_cast<uint32_t>(rowBytes));
                }
                g_times.transform += Seconds(start);
            }
            if (g_group != nullptr)
            {
                // every GPU of the group takes a part of the block over its own PCIe link
                const int status = measure ? avifgpu_encode_rows_sharded_light_level(g_group, &desc, rows, rowBytes, top, bottom - top, &planes, &light)
                                           : avifgpu_encode_rows_sharded(g_group, &desc, rows, rowBytes, top, bottom - top, &planes);
                if (status != AVIFGPU_OK)
                {
                    if (status == AVIFGPU_ERR_BAD_PARAM) throw OSErrException(formatBadParameters);
                    if (status == AVIFGPU_ERR_OOM) throw std::bad_alloc();
                    throw std::runtime_error(avifgpu_shard_group_last_error(g_group));
                }
            }
            else
            {
                // returns once the block is queued: the host fills the other buffer while this one is on the wire;
                // the buffer handed over in the previous iteration is free again when this call returns
                ThrowIfFailed(ctx, measure ? avifgpu_encode_rows_async_light_level(ctx, &desc, rows, rowBytes, top, bottom - top, &planes, &light, nullptr)
                                           : avifgpu_encode_rows_async(ctx, &desc, rows, rowBytes, top, bottom - top, &planes, nullptr));
            }
        }
        g_times.blocks = block;
        ThrowIfFailed(ctx, avifgpu_wait(ctx, 0)); // the planes (and the light level) are complete
        if (measure)
        {
            heif_content_light_level clli{};
            ThrowIfFailed(ctx, avifgpu_content_light_level(&light, bitDepth, &clli.max_content_light_level, &clli.max_pic_average_light_level));
            heif_image_set_content_light_level(image.get(), &clli);
            g_lastLightLevel = avifgpu_host::ContentLightLevel{ true, clli.max_content_light_level, clli.max_pic_average_light_level };
        }
        return image;
    }

    // ---- decode --------------------------------------------------------------------------------------------------

    void DecodeThroughGpu(const heif_image* image, AlphaState alphaState, const heif_color_profile_nclx* nclxProfile,
                          const LoadUIOptions* loadOptions, FormatRecordPtr formatRecord, int hostDepth, bool gray)
    {
        CallTimer callTimer;
        avifgpu_context* ctx = avifgpu_host::SharedContext();
        const VPoint imageSize = GetImageSizeOf(formatRecord);
        const bool hasAlpha = alphaState != AlphaState::None;

        avifgpu_decode_desc desc{};
        desc.struct_size = sizeof(desc);
        desc.width = imageSize.h;
        desc.height = imageSize.v;
        desc.alpha_state = static_cast<int32_t>(alphaState);
        desc.host_depth = hostDepth;
        desc.nclx = ToNclx(nclxProfile);
        if (loadOptions != nullptr)
        {
            desc.hlg_apply_ootf = loadOptions->hlg.applyOOTF ? 1 : 0;
            desc.hlg_display_gamma = loadOptions->hlg.displayGamma;
            desc.hlg_peak_nits = loadOptions->hlg.nominalPeakBrightness;
            desc.pq_peak_nits = loadOptions->pq.nominalPeakBrightness;
        }
        else
        {
            desc.hlg_display_gamma = 1.2f;
            desc.hlg_peak_nits = 1000;
            desc.pq_peak_nits = 80;
        }

        avifgpu_planes planes{};
        auto plane = [&](heif_channel channel, int index)
        {
            int stride = 0;
            planes.data[index] = const_cast<uint8_t*>(heif_image_get_plane_readonly(image, channel, &stride));
            planes.stride[index] = stride;
            if (planes.data[index] == nullptr)
            {
                throw std::runtime_error("The image is missing a channel.");
            }
        };
        heif_channel first = heif_channel_Y;
        if (gray)
        {
            desc.colorspace = AVIFGPU_COLORSPACE_MONOCHROME;
            desc.chroma = AVIFGPU_CHROMA_MONOCHROME;
            plane(heif_channel_Y, 0);
        }
        else
        {
            const heif_colorspace colorspace = heif_image_get_colorspace(image);
            if (colorspace == heif_colorspace_YCbCr)
            {
                desc.colorspace = AVIFGPU_COLORSPACE_YCBCR;
                desc.chroma = static_cast<int32_t>(heif_image_get_chroma_format(image));
                plane(heif_channel_Y, 0);
                plane(heif_channel_Cb, 1);
                plane(heif_channel_Cr, 2);
                const int luma = heif_image_get_bits_per_pixel_range(image, heif_channel_Y);
                if (heif_image_get_bits_per_pixel_range(image, heif_channel_Cb) != luma ||
                    heif_image_get_bits_per_pixel_range(image, heif_channel_Cr) != luma)
                {
                    throw std::runtime_error("The chroma channel bit depth does not match the main image."); // ReadHeifImage.cpp:93-97
                }
            }
            else if (colorspace == heif_colorspace_RGB)
            {
                desc.colorspace = AVIFGPU_COLORSPACE_RGB;
                desc.chroma = AVIFGPU_CHROMA_444;
                first = heif_channel_R;
                plane(heif_channel_R, 0);
                plane(heif_channel_G, 1);
                plane(heif_channel_B, 2);
                const int red = heif_image_get_bits_per_pixel_range(image, heif_channel_R);
                if (heif_image_get_bits_per_pixel_range(image, heif_channel_G) != red ||
                    heif_image_get_bits_per_pixel_range(image, heif_channel_B) != red)
                {
                    throw std::runtime_error("The color channel bit depths do not match."); // ReadHeifImage.cpp:591-595
                }
            }
            else
            {
                throw std::runtime_error("Unsupported image color space, expected RGB."); // ReadHeifImage.cpp:575-578
            }
        }
        desc.bit_depth = heif_image_get_bits_per_pixel_range(image, first);
        if (hasAlpha)
        {
            plane(heif_channel_Alpha, 3);
            if (heif_image_get_bits_per_pixel_range(image, heif_channel_Alpha) != desc.bit_depth)
            {
                throw std::runtime_error("The alpha channel bit depth does not match the main image channels.");
            }
        }

        // SetupFormatRecord, ReadHeifImage.cpp:31-50
        formatRecord->loPlane = 0;
        formatRecord->hiPlane = static_cast<int16>(formatRecord->planes - 1);
        formatRecord->planeBytes = static_cast<int16>((formatRecord->depth + 7) / 8);
        formatRecord->colBytes = static_cast<int16>(formatRecord->planes * formatRecord->planeBytes);
        const int64_t rowBytes = static_cast<int64_t>(imageSize.h) * formatRecord->colBytes;
        if (rowBytes > std::numeric_limits<int32>::max())
        {
            throw std::bad_alloc();
        }
        if (hostDepth == 16)
        {
            // ReadHeifImage.cpp:206 (YCbCr: maxData, sic), :499 (gray), :744 (planar RGB: the source range)
            if (gray)
            {
                formatRecord->maxValue = 32768;
            }
            else if (desc.colorspace == AVIFGPU_COLORSPACE_YCBCR)
            {
                formatRecord->maxData = 32768;
            }
            else
            {
                formatRecord->maxValue = (1 << desc.bit_depth) - 1;
            }
        }

        StagingPair staging(ctx, rowBytes, imageSize.v);
        const int32 blockRows = staging.blockRows;
        g_times.rowsPerBlock = blockRows;
        RecordDataGuard guard(formatRecord);
        DrainOnExit drain{ ctx };
        formatRecord->rowBytes = static_cast<int32>(rowBytes);

        // Block k+1 converts and travels while the host takes block k.
        auto issue = [&](int32 top, int32 index, int64_t* ticket)
        {
            const int32 bottom = std::min(top + blockRows, imageSize.v);
            void* rows = staging.buffer[index & 1]->get();
            if (g_group != nullptr)
            {
                const int status = avifgpu_decode_rows_sharded(g_group, &desc, &planes, top, bottom - top, rows, rowBytes);
                if (status != AVIFGPU_OK)
                {
                    if (status == AVIFGPU_ERR_BAD_PARAM) throw OSErrException(formatBadParameters);
                    if (status == AVIFGPU_ERR_OOM) throw std::bad_alloc();
                    throw std::runtime_error(avifgpu_shard_group_last_error(g_group));
                }
                *ticket = 0;
                return;
            }
            ThrowIfFailed(ctx, avifgpu_decode_rows_async(ctx, &desc, &planes, top, bottom - top, rows, rowBytes, ticket));
        };
        int64_t ticket = 0;
        if (imageSize.v > 0)
        {
            issue(0, 0, &ticket);
        }
        int32 block = 0;
        for (int32 top = 0; top < imageSize.v; top += blockRows, ++block)
        {
            const int32 bottom = std::min(top + blockRows, imageSize.v);
            int64_t nextTicket = 0;
            if (bottom < imageSize.v)
            {
                issue(bottom, block + 1, &nextTicket);
            }
            if (g_group == nullptr)
            {
                ThrowIfFailed(ctx, avifgpu_wait(ctx, ticket));
            }
            ticket = nextTicket;
            HostTimer timer;
            formatRecord->data = staging.buffer[block & 1]->get();
            SetRectOf(formatRecord, top, 0, bottom, imageSize.h);
            OSErrException::ThrowIfError(formatRecord->advanceState()); // the host consumes rows [top, bottom)
        }
        g_times.blocks = block;
    }
}

namespace avifgpu_host
{

avifgpu_context* SharedContext()
{
    if (g_context == nullptr)
    {
        avifgpu_context* created = nullptr;
        const int status = avifgpu_create(0, &created);
        if (status != AVIFGPU_OK)
        {
            throw OSErrException(errPlugInHostInsufficient);
        }
        g_context = created;
    }
    return g_context;
}

void ReleaseSharedContext()
{
    g_staging.Release(); // before the context that owns the page-locked memory goes away
    if (g_group != nullptr)
    {
        avifgpu_shard_group_destroy(g_group);
        g_group = nullptr;
        g_context = nullptr; // owned by the group
    }
    if (g_context != nullptr)
    {
        avifgpu_destroy(g_context);
        g_context = nullptr;
    }
}

void SetRowsPerBlock(int32 rows) { g_rowsPerBlock = std::max<int32>(rows, 2); }

void SetStagingBudgetBytes(int64_t bytes) { g_stagingBudget = std::max<int64_t>(bytes, 1); }

void UseDevices(const int32_t* deviceOrdinals, int32_t count)
{
    ReleaseSharedContext();
    if (deviceOrdinals == nullptr || count <= 1)
    {
        return; // the next call creates the single shared context
    }
    avifgpu_shard_group* group = nullptr;
    if (avifgpu_shard_group_create(deviceOrdinals, count, &group) != AVIFGPU_OK)
    {
        throw OSErrException(errPlugInHostInsufficient);
    }
    g_group = group;
    g_context = avifgpu_shard_group_context(group, 0); // staging memory and the geometry helpers go through member 0
}

void SetRowTransformFactory(RowTransformFactory factory, void* user)
{
    g_transformFactory = factory;
    g_transformUser = user;
}

void SetGpuRowMatrixEnabled(bool enabled) { g_gpuRowMatrix = enabled; }

void SetContentLightLevelEnabled(bool enabled) { g_contentLightLevel = enabled; }

ContentLightLevel LastContentLightLevel() { return g_lastLightLevel; }

ShuttleTimes LastShuttleTimes() { return g_times; }

} // namespace avifgpu_host

ScopedHeifImage CreateHeifImageGrayEightBit(FormatRecordPtr formatRecord, AlphaState alphaState, const VPoint& imageSize, const SaveUIOptions& saveOptions)
{
    return EncodeThroughGpu(formatRecord, alphaState, imageSize, saveOptions, 8, true);
}

ScopedHeifImage CreateHeifImageGraySixteenBit(FormatRecordPtr formatRecord, AlphaState alphaState, const VPoint& imageSize, const SaveUIOptions& saveOptions)
{
    return EncodeThroughGpu(formatRecord, alphaState, imageSize, saveOptions, 16, true);
}

ScopedHeifImage CreateHeifImageGrayThirtyTwoBit(FormatRecordPtr formatRecord, AlphaState alphaState, const VPoint& imageSize, const SaveUIOptions& saveOptions)
{
    return EncodeThroughGpu(formatRecord, alphaState, imageSize, saveOptions, 32, true);
}

ScopedHeifImage CreateHeifImageRGBEightBit(FormatRecordPtr formatRecord, AlphaState alphaState, const VPoint& imageSize, const SaveUIOptions& saveOptions)
{
    return EncodeThroughGpu(formatRecord, alphaState, imageSize, saveOptions, 8, false);
}

ScopedHeifImage CreateHeifImageRGBSixteenBit(FormatRecordPtr formatRecord, AlphaState alphaState, const VPoint& imageSize, const SaveUIOptions& saveOptions)
{
    return EncodeThroughGpu(formatRecord, alphaState, imageSize, saveOptions, 16, false);
}

ScopedHeifImage CreateHeifImageRGBThirtyTwoBit(FormatRecordPtr formatRecord, AlphaState alphaState, const VPoint& imageSize, const SaveUIOptions& saveOptions)
{
    return EncodeThroughGpu(formatRecord, alphaState, imageSize, saveOptions, 32, false);
}

void ReadHeifImageGrayEightBit(const heif_image* image, AlphaState alphaState, const heif_color_profile_nclx* nclxProfile, FormatRecordPtr formatRecord)
{
    DecodeThroughGpu(image, alphaState, nclxProfile, nullptr, formatRecord, 8, true);
}

void ReadHeifImageGraySixteenBit(const heif_image* image, AlphaState alphaState, const heif_color_profile_nclx* nclxProfile, FormatRecordPtr formatRecord)
{
    DecodeThroughGpu(image, alphaState, nclxProfile, nullptr, formatRecord, 16, true);
}

void ReadHeifImageGrayThirtyTwoBit(const heif_image* image, AlphaState alphaState, const heif_color_profile_nclx* nclxProfile, const LoadUIOptions& loadOptions, FormatRecordPtr formatRecord)
{
    if (nclxProfile == nullptr)
    {
        throw std::runtime_error("The nclxProfile is null."); // ReadHeifImage.cpp:870-873
    }
    DecodeThroughGpu(image, alphaState, nclxProfile, &loadOptions, formatRecord, 32, true);
}

void ReadHeifImageRGBEightBit(const heif_image* image, AlphaState alphaState, const heif_color_profile_nclx* nclxProfile, FormatRecordPtr formatRecord)
{
    DecodeThroughGpu(image, alphaState, nclxProfile, nullptr, formatRecord, 8, false);
}

void ReadHeifImageRGBSixteenBit(const heif_image* image, AlphaState alphaState, const heif_color_profile_nclx* nclxProfile, FormatRecordPtr formatRecord)
{
    DecodeThroughGpu(image, alphaState, nclxProfile, nullptr, formatRecord, 16, false);
}

void ReadHeifImageRGBThirtyTwoBit(const heif_image* image, AlphaState alphaState, const heif_color_profile_nclx* nclxProfile, const LoadUIOptions& loadOptions, FormatRecordPtr formatRecord)
{
    if (nclxProfile == nullptr)
    {
        throw std::runtime_error("The nclxProfile is null."); // ReadHeifImage.cpp:956-959
    }
    DecodeThroughGpu(image, alphaState, nclxProfile, &loadOptions, formatRecord, 32, false);
}
