// compat/PluginTypes.h -- the plug-in-side types the GPU row shuttle is written against, for builds where the real
// headers (Photoshop SDK PIFormat.h / PITypes.h, libheif/heif.h, and the plug-in's AvifFormat.h, AlphaState.h,
// ColorTransfer.h) are not available.  When the shuttle is dropped into the plug-in tree, define
// AVIFGPU_HOST_USE_PLUGIN_HEADERS and these declarations are replaced by the real ones (same names, same meaning).
//
// Only what the row shuttle touches is declared; field / enumerator names follow the reference
// (src/common/AvifFormat.h:28-101, AlphaState.h:24-29, ColorTransfer.h:28-34) and the public SDK / libheif ABIs.
#ifndef AVIFGPU_HOST_COMPAT_PLUGIN_TYPES_H
#define AVIFGPU_HOST_COMPAT_PLUGIN_TYPES_H

#if defined(AVIFGPU_HOST_USE_PLUGIN_HEADERS)
#include "AvifFormat.h"
#include "AlphaState.h"
#include "ScopedHeif.h"
#include "OSErrException.h"
#include "LibHeifException.h"
#else

#include <stdint.h>

#include <memory>
#include <stdexcept>

// ---- Photoshop SDK subset ----------------------------------------------------------------------------------------
typedef int16_t int16;
typedef int32_t int32;
typedef int16 OSErr;
typedef char* Ptr;
typedef unsigned char Boolean;
struct Point { int16 v; int16 h; };
struct Rect { int16 top, left, bottom, right; };
struct VPoint { int32 v; int32 h; };
struct VRect { int32 top, left, bottom, right; };
enum { noErr = 0, memFullErr = -108, userCanceledErr = -128 };
enum { formatBadParameters = -30500, formatCannotRead = -30501, errPlugInHostInsufficient = -30900 };
enum { plugInModeGrayScale = 1, plugInModeRGBColor = 3, plugInModeGray16 = 10, plugInModeRGB48 = 11, plugInModeGray32 = 13, plugInModeRGB96 = 16 };

typedef struct PSBufferID_* BufferID;
struct BufferProcs
{
    OSErr (*allocateProc)(int32 size, BufferID* bufferID);
    Ptr (*lockProc)(BufferID bufferID, Boolean moveHigh);
    void (*unlockProc)(BufferID bufferID);
    void (*freeProc)(BufferID bufferID);
};

struct FormatRecord
{
    void* data;
    int32 rowBytes;
    int16 colBytes;
    int16 planeBytes;
    int16 loPlane;
    int16 hiPlane;
    int16 planes;
    int16 depth;
    int16 imageMode;
    Point imageSize;
    VPoint imageSize32;
    Rect theRect;
    VRect theRect32;
    Boolean HostSupports32BitCoordinates;
    Boolean PluginUsing32BitCoordinates;
    int32 maxData;
    int32 maxValue;
    int16 transparencyPlane;
    OSErr (*advanceState)(void);
    Boolean (*abortProc)(void);
    void (*progressProc)(int32 done, int32 total);
    BufferProcs* bufferProcs;
    // document colour profile (HostMetadata.cpp:63-69 HasColorProfileMetadata reads exactly these; the handle suite the
    // real test also asks for is not modelled here)
    Boolean canUseICCProfiles;
    void* iCCprofileData; // a Handle in the SDK
    int32 iCCprofileSize;
};
typedef FormatRecord* FormatRecordPtr;

class OSErrException : public std::exception
{
public:
    explicit OSErrException(OSErr err) noexcept : error(err) {}
    OSErr GetErrorCode() const noexcept { return error; }
    static void ThrowIfError(OSErr err) { if (err != noErr) throw OSErrException(err); }
private:
    OSErr error;
};

// ---- libheif subset ------------------------------------------------------------------------------------------------
extern "C" {
enum heif_error_code { heif_error_Ok = 0, heif_error_Memory_allocation_error = 6 };
enum heif_suberror_code { heif_suberror_Unspecified = 0 };
struct heif_error { enum heif_error_code code; enum heif_suberror_code subcode; const char* message; };
enum heif_chroma { heif_chroma_undefined = 99, heif_chroma_monochrome = 0, heif_chroma_420 = 1, heif_chroma_422 = 2, heif_chroma_444 = 3 };
enum heif_colorspace { heif_colorspace_undefined = 99, heif_colorspace_YCbCr = 0, heif_colorspace_RGB = 1, heif_colorspace_monochrome = 2 };
enum heif_channel { heif_channel_Y = 0, heif_channel_Cb = 1, heif_channel_Cr = 2, heif_channel_R = 3, heif_channel_G = 4, heif_channel_B = 5,
                    heif_channel_Alpha = 6, heif_channel_interleaved = 10 };
struct heif_color_profile_nclx
{
    uint8_t version;
    int color_primaries;
    int transfer_characteristics;
    int matrix_coefficients;
    uint8_t full_range_flag;
    float color_primary_red_x, color_primary_red_y, color_primary_green_x, color_primary_green_y;
    float color_primary_blue_x, color_primary_blue_y, color_primary_white_x, color_primary_white_y;
};
struct heif_image;
struct heif_error heif_image_create(int width, int height, enum heif_colorspace colorspace, enum heif_chroma chroma, struct heif_image** out_image);
struct heif_error heif_image_add_plane(struct heif_image* image, enum heif_channel channel, int width, int height, int bit_depth);
uint8_t* heif_image_get_plane(struct heif_image* image, enum heif_channel channel, int* out_stride);
const uint8_t* heif_image_get_plane_readonly(const struct heif_image* image, enum heif_channel channel, int* out_stride);
int heif_image_get_bits_per_pixel_range(const struct heif_image* image, enum heif_channel channel);
enum heif_chroma heif_image_get_chroma_format(const struct heif_image* image);
enum heif_colorspace heif_image_get_colorspace(const struct heif_image* image);
void heif_image_release(const struct heif_image* image);
struct heif_content_light_level
{
    uint16_t max_content_light_level;
    uint16_t max_pic_average_light_level;
};
int heif_image_has_content_light_level(const struct heif_image* image);
void heif_image_get_content_light_level(const struct heif_image* image, struct heif_content_light_level* out);
// Weak: the stand-alone shuttle links against whatever libheif (or stand-in) it is given, and one without content light
// level support leaves this NULL.  The shuttle then refuses a save that would measure, instead of dropping the property.
__attribute__((weak)) void heif_image_set_content_light_level(const struct heif_image* image, const struct heif_content_light_level* in);
}

namespace detail
{
    struct image_deleter { void operator()(heif_image* h) noexcept { if (h) heif_image_release(h); } };
}
using ScopedHeifImage = std::unique_ptr<heif_image, detail::image_deleter>;

class LibHeifException : public std::runtime_error
{
public:
    explicit LibHeifException(const heif_error& e) : std::runtime_error(e.message ? e.message : "libheif error") {}
    static void ThrowIfError(const heif_error& e)
    {
        if (e.code != heif_error_Ok)
        {
            if (e.code == heif_error_Memory_allocation_error && e.subcode == heif_suberror_Unspecified) throw std::bad_alloc();
            throw LibHeifException(e);
        }
    }
};

// ---- plug-in option blocks (AvifFormat.h:28-101, AlphaState.h, ColorTransfer.h) --------------------------------------
enum class AlphaState { None, Straight, Premultiplied };
enum class ColorTransferFunction { PQ, HLG, SMPTE428, Clip };
enum class ChromaSubsampling { Yuv420, Yuv422, Yuv444 };
enum class CompressionSpeed { Fastest, Default, Slowest };
enum class ImageBitDepth { Eight, Ten, Twelve };
struct HLGOptions { bool applyOOTF; float displayGamma; int nominalPeakBrightness; };
struct PQOptions { int nominalPeakBrightness; };
enum class LoadOptionsHDRFormat : int { Unknown = 0, HLG, PQ };
struct LoadUIOptions { LoadOptionsHDRFormat format; HLGOptions hlg; PQOptions pq; };
struct SaveUIOptions
{
    int quality;
    ChromaSubsampling chromaSubsampling;
    CompressionSpeed compressionSpeed;
    ImageBitDepth imageBitDepth;
    ColorTransferFunction hdrTransferFunction;
    PQOptions pq;
    bool lossless;
    bool losslessAlpha;
    bool keepColorProfile;
    bool keepExif;
    bool keepXmp;
    bool premultipliedAlpha;
};

#endif // AVIFGPU_HOST_USE_PLUGIN_HEADERS
#endif
