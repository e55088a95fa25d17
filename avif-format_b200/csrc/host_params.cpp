// host_params.cpp -- see host_params.h.  Compiled by the host compiler with -ffp-contract=off: the few float
// expressions here (matrix coefficients, luminance multipliers) feed the kernels and must round exactly as the
// reference's do.
#include "host_params.h"

#include "batch_plan.h"

#include <cstring>

namespace avifgpu
{

namespace
{
    struct PrimariesRow
    {
        int32_t code;
        float v[8]; // rX rY gX gY bX bY wX wY
    };

    // Chromaticities per H.273 colour-primaries code point as the reference tabulates them
    // (YUVCoefficiants.cpp:56-68; values are the H.273 / libavif ones, kept digit for digit because the
    // chromaticity-derived matrix is computed from them in float).
    const PrimariesRow kPrimaries[] = {
        { 1, { 0.64f, 0.33f, 0.3f, 0.6f, 0.15f, 0.06f, 0.3127f, 0.329f } },
        { 4, { 0.67f, 0.33f, 0.21f, 0.71f, 0.14f, 0.08f, 0.310f, 0.316f } },
        { 5, { 0.64f, 0.33f, 0.29f, 0.60f, 0.15f, 0.06f, 0.3127f, 0.3290f } },
        { 6, { 0.630f, 0.340f, 0.310f, 0.595f, 0.155f, 0.070f, 0.3127f, 0.3290f } },
        { 7, { 0.630f, 0.340f, 0.310f, 0.595f, 0.155f, 0.070f, 0.3127f, 0.3290f } },
        { 8, { 0.681f, 0.319f, 0.243f, 0.692f, 0.145f, 0.049f, 0.310f, 0.316f } },
        { 9, { 0.708f, 0.292f, 0.170f, 0.797f, 0.131f, 0.046f, 0.3127f, 0.3290f } },
        { 10, { 1.0f, 0.0f, 0.0f, 1.0f, 0.0f, 0.0f, 0.3333f, 0.3333f } },
        { 11, { 0.680f, 0.320f, 0.265f, 0.690f, 0.150f, 0.060f, 0.314f, 0.351f } },
        { 12, { 0.680f, 0.320f, 0.265f, 0.690f, 0.150f, 0.060f, 0.3127f, 0.3290f } },
        { 22, { 0.630f, 0.340f, 0.295f, 0.605f, 0.155f, 0.077f, 0.3127f, 0.3290f } },
    };

    struct MatrixRow
    {
        int32_t code;
        float kr;
        float kb;
    };

    // YUVCoefficiants.cpp:94-106
    const MatrixRow kMatrices[] = {
        { 1, 0.2126f, 0.0722f }, { 4, 0.30f, 0.11f },     { 5, 0.299f, 0.114f },
        { 6, 0.299f, 0.114f },   { 7, 0.212f, 0.087f },   { 9, 0.2627f, 0.0593f },
    };

    const float* LookupPrimaries(int32_t code)
    {
        for (const PrimariesRow& row : kPrimaries)
        {
            if (row.code == code)
            {
                return row.v;
            }
        }
        return kPrimaries[0].v; // YUVCoefficiants.cpp:81-82
    }

    int Fail(std::string* error, int status, const char* message)
    {
        if (error)
        {
            *error = message;
        }
        return status;
    }
}

void GetYuvCoefficients(const avifgpu_nclx* nclx, float out[3])
{
    // YUVCoefficiants.cpp:171-174: BT.601 unless the CICP says otherwise
    float kr = 0.299f;
    float kb = 0.114f;
    float kg = 1.0f - kr - kb;

    if (nclx != nullptr && nclx->present)
    {
        if (nclx->matrix_coefficients == 12)
        {
            // YUVCoefficiants.cpp:110-137 (H.273 equations 32-37), float arithmetic in the reference's association
            const float* p = LookupPrimaries(nclx->color_primaries);
            const float rX = p[0], rY = p[1], gX = p[2], gY = p[3], bX = p[4], bY = p[5], wX = p[6], wY = p[7];
            const float rZ = 1.0f - (rX + rY);
            const float gZ = 1.0f - (gX + gY);
            const float bZ = 1.0f - (bX + bY);
            const float wZ = 1.0f - (wX + wY);
            kr = (rY * (wX * (gY * bZ - bY * gZ) + wY * (bX * gZ - gX * bZ) + wZ * (gX * bY - bX * gY))) /
                 (wY * (rX * (gY * bZ - bY * gZ) + gX * (bY * rZ - rY * bZ) + bX * (rY * gZ - gY * rZ)));
            kb = (bY * (wX * (rY * gZ - gY * rZ) + wY * (gX * rZ - rX * gZ) + wZ * (rX * gY - gX * rY))) /
                 (wY * (rX * (gY * bZ - bY * gZ) + gX * (bY * rZ - rY * bZ) + bX * (rY * gZ - gY * rZ)));
            kg = 1.0f - kr - kb;
        }
        else
        {
            for (const MatrixRow& row : kMatrices)
            {
                if (row.code == nclx->matrix_coefficients)
                {
                    kr = row.kr;
                    kb = row.kb;
                    kg = 1.0f - kr - kb;
                    break;
                }
            }
        }
    }
    out[0] = kr;
    out[1] = kg;
    out[2] = kb;
}

bool GetHlgLumaCoefficients(int32_t colorPrimaries, float out[3])
{
    switch (colorPrimaries)
    {
    case 1:
        out[0] = 0.2126f; out[1] = 0.7152f; out[2] = 0.0722f;
        return true;
    case 5:
    case 6:
        out[0] = 0.299f; out[1] = 0.587f; out[2] = 0.114f;
        return true;
    case 9:
        out[0] = 0.2627f; out[1] = 0.6780f; out[2] = 0.0593f;
        return true;
    default:
        return false;
    }
}

bool TransferFromNclx(int32_t transferCharacteristics, int32_t* outTransfer)
{
    switch (transferCharacteristics)
    {
    case 16: *outTransfer = AVIFGPU_TRANSFER_PQ; return true;
    case 18: *outTransfer = AVIFGPU_TRANSFER_HLG; return true;
    case 17: *outTransfer = AVIFGPU_TRANSFER_SMPTE428; return true;
    default: return false;
    }
}

avifpix::RangeParams MakeRangeParams(const avifgpu_nclx* nclx, int bitDepth, bool monochrome)
{
    avifpix::RangeParams r{};
    const bool hasNclx = nclx != nullptr && nclx->present;
    // YuvLookupTables.cpp:143-144: full range and BT.601 when there is no nclx
    r.fullRange = hasNclx ? (nclx->full_range_flag != 0) : 1;
    const int matrix = hasNclx ? nclx->matrix_coefficients : 6;
    r.identityMatrix = (!monochrome && matrix == 0) ? 1 : 0;
    r.maxChannel = (1 << bitDepth) - 1;
    r.maxChannelFloat = static_cast<float>(r.maxChannel);
    switch (bitDepth)
    {
    case 8: r.yLo = 16; r.yHi = 235; r.uvLo = 16; r.uvHi = 240; break;
    case 10: r.yLo = 64; r.yHi = 940; r.uvLo = 64; r.uvHi = 960; break;
    case 12: r.yLo = 256; r.yHi = 3760; r.uvLo = 256; r.uvHi = 3840; break;
    default: r.yLo = 1024; r.yHi = 60160; r.uvLo = 1024; r.uvHi = 61440; break;
    }
    return r;
}

int ValidateEncodeDesc(const avifgpu_encode_desc* d, std::string* error)
{
    if (d == nullptr || (d->struct_size != sizeof(avifgpu_encode_desc) && d->struct_size != AVIFGPU_ENCODE_DESC_V10_SIZE)) return Fail(error, AVIFGPU_ERR_BAD_PARAM, "bad encode desc size");
    if (d->width < 0 || d->height < 0) return Fail(error, AVIFGPU_ERR_BAD_PARAM, "negative image size");
    if (d->host_depth != 8 && d->host_depth != 16 && d->host_depth != 32) return Fail(error, AVIFGPU_ERR_BAD_PARAM, "host depth must be 8, 16 or 32");
    if (d->host_channels < 1 || d->host_channels > 4) return Fail(error, AVIFGPU_ERR_BAD_PARAM, "host channels must be 1..4");
    if (d->image_bit_depth != 8 && d->image_bit_depth != 10 && d->image_bit_depth != 12) return Fail(error, AVIFGPU_ERR_BAD_PARAM, "image bit depth must be 8, 10 or 12");
    const bool expectsAlpha = d->host_channels == 2 || d->host_channels == 4;
    const bool hasAlpha = d->alpha_state != AVIFGPU_ALPHA_NONE;
    if (d->alpha_state < AVIFGPU_ALPHA_NONE || d->alpha_state > AVIFGPU_ALPHA_PREMULTIPLIED || expectsAlpha != hasAlpha)
    {
        return Fail(error, AVIFGPU_ERR_BAD_PARAM, "alpha state does not match the channel count");
    }
    if (d->host_depth == 32)
    {
        if (d->image_bit_depth == 8) return Fail(error, AVIFGPU_ERR_UNSUPPORTED, "32-bit hosts require a 10- or 12-bit image");
        // WriteHeifImage.cpp:578-588 (gray: PQ, Clip), :1079-1091 (colour: PQ, SMPTE428, Clip)
        const bool gray = d->host_channels <= 2;
        // plus, only on request, the HLG save path the reference has the functions for but never calls (avifgpu.h)
        const bool hlg = !gray && d->transfer == AVIFGPU_TRANSFER_HLG &&
                         (d->hlg_extension == AVIFGPU_HLG_OETF || d->hlg_extension == AVIFGPU_HLG_INVERSE_OOTF_THEN_OETF);
        const bool ok = d->transfer == AVIFGPU_TRANSFER_PQ || d->transfer == AVIFGPU_TRANSFER_CLIP ||
                        (!gray && d->transfer == AVIFGPU_TRANSFER_SMPTE428) || hlg;
        if (!ok) return Fail(error, AVIFGPU_ERR_UNSUPPORTED, "Unsupported color transfer function.");
        if (hlg && d->hlg_extension == AVIFGPU_HLG_INVERSE_OOTF_THEN_OETF)
        {
            float luma[3];
            if (!d->nclx.present || !GetHlgLumaCoefficients(d->nclx.color_primaries, luma))
            {
                return Fail(error, AVIFGPU_ERR_UNSUPPORTED, "the inverse HLG OOTF needs nclx colour primaries with known luma coefficients");
            }
            if (!(d->hlg_display_gamma > 0.0f) || d->hlg_peak_nits <= 0)
            {
                return Fail(error, AVIFGPU_ERR_BAD_PARAM, "bad HLG display gamma / peak brightness");
            }
        }
    }
    if (d->layout == AVIFGPU_LAYOUT_PLANAR_YCBCR)
    {
        if (d->host_channels <= 2) return Fail(error, AVIFGPU_ERR_BAD_PARAM, "planar YCbCr needs a colour host");
        if (d->chroma != AVIFGPU_CHROMA_420 && d->chroma != AVIFGPU_CHROMA_422 && d->chroma != AVIFGPU_CHROMA_444) return Fail(error, AVIFGPU_ERR_BAD_PARAM, "bad chroma");
        if (d->nclx.present && !d->nclx.full_range_flag) return Fail(error, AVIFGPU_ERR_UNSUPPORTED, "the encode path is full range only");
        if (d->nclx.present && d->nclx.matrix_coefficients == 0 && d->chroma != AVIFGPU_CHROMA_444) return Fail(error, AVIFGPU_ERR_UNSUPPORTED, "identity (GBR) matrix requires 4:4:4");
    }
    else if (d->layout != AVIFGPU_LAYOUT_REFERENCE)
    {
        return Fail(error, AVIFGPU_ERR_BAD_PARAM, "bad layout");
    }
    const int32_t dest = DestLayoutOf(*d);
    if (dest != AVIFGPU_SOURCE_PLANAR)
    {
        if (dest & ~(AVIFGPU_SOURCE_CHROMA_INTERLEAVED | AVIFGPU_SOURCE_MSB_ALIGNED)) return Fail(error, AVIFGPU_ERR_BAD_PARAM, "unknown destination layout bits");
        if (d->layout != AVIFGPU_LAYOUT_PLANAR_YCBCR) return Fail(error, AVIFGPU_ERR_UNSUPPORTED, "semi-planar and MSB-aligned destinations are planar YCbCr only");
        if ((dest & AVIFGPU_SOURCE_MSB_ALIGNED) && d->image_bit_depth == 8) return Fail(error, AVIFGPU_ERR_BAD_PARAM, "MSB-aligned destinations need a 10- or 12-bit image");
    }
    return AVIFGPU_OK;
}

int32_t DestLayoutOf(const avifgpu_encode_desc& d) { return d.struct_size == sizeof(avifgpu_encode_desc) ? d.dest_layout : AVIFGPU_SOURCE_PLANAR; }

const avifgpu_encode_desc* WidenEncodeDesc(const avifgpu_encode_desc* d, avifgpu_encode_desc* full)
{
    if (d == nullptr || d->struct_size != AVIFGPU_ENCODE_DESC_V10_SIZE)
    {
        return d;
    }
    std::memset(full, 0, sizeof(*full));
    std::memcpy(full, d, AVIFGPU_ENCODE_DESC_V10_SIZE);
    full->struct_size = sizeof(avifgpu_encode_desc);
    full->dest_layout = AVIFGPU_SOURCE_PLANAR;
    return full;
}

int ValidateDecodeDesc(const avifgpu_decode_desc* d, int32_t* outTransfer, std::string* error)
{
    *outTransfer = AVIFGPU_TRANSFER_CLIP;
    if (d == nullptr || (d->struct_size != sizeof(avifgpu_decode_desc) && d->struct_size != AVIFGPU_DECODE_DESC_V9_SIZE)) return Fail(error, AVIFGPU_ERR_BAD_PARAM, "bad decode desc size");
    if (d->width < 0 || d->height < 0) return Fail(error, AVIFGPU_ERR_BAD_PARAM, "negative image size");
    if (d->host_depth != 8 && d->host_depth != 16 && d->host_depth != 32) return Fail(error, AVIFGPU_ERR_BAD_PARAM, "host depth must be 8, 16 or 32");
    if (d->bit_depth != 8 && d->bit_depth != 10 && d->bit_depth != 12 && d->bit_depth != 16) return Fail(error, AVIFGPU_ERR_UNSUPPORTED, "The image has an unsupported bit depth, must be 8, 10, 12 or 16.");
    if (d->colorspace != AVIFGPU_COLORSPACE_YCBCR && d->colorspace != AVIFGPU_COLORSPACE_RGB && d->colorspace != AVIFGPU_COLORSPACE_MONOCHROME) return Fail(error, AVIFGPU_ERR_UNSUPPORTED, "Unsupported image color space, expected RGB.");
    if (d->alpha_state < AVIFGPU_ALPHA_NONE || d->alpha_state > AVIFGPU_ALPHA_PREMULTIPLIED) return Fail(error, AVIFGPU_ERR_BAD_PARAM, "bad alpha state");
    if ((d->host_depth == 8) != (d->bit_depth == 8)) return Fail(error, AVIFGPU_ERR_UNSUPPORTED, "host depth 8 pairs with 8-bit planes only");
    if (d->colorspace == AVIFGPU_COLORSPACE_YCBCR && d->chroma != AVIFGPU_CHROMA_420 && d->chroma != AVIFGPU_CHROMA_422 && d->chroma != AVIFGPU_CHROMA_444) return Fail(error, AVIFGPU_ERR_BAD_PARAM, "bad chroma");
    if (d->host_depth == 32)
    {
        if (!d->nclx.present) return Fail(error, AVIFGPU_ERR_UNSUPPORTED, "The nclxProfile is null.");
        if (!TransferFromNclx(d->nclx.transfer_characteristics, outTransfer)) return Fail(error, AVIFGPU_ERR_UNSUPPORTED, "Unsupported NCLX transfer characteristic.");
        if (d->colorspace == AVIFGPU_COLORSPACE_MONOCHROME && *outTransfer != AVIFGPU_TRANSFER_PQ) return Fail(error, AVIFGPU_ERR_UNSUPPORTED, "Unsupported color transfer function.");
    }
    const int32_t layout = SourceLayoutOf(*d);
    if (layout != AVIFGPU_SOURCE_PLANAR)
    {
        if (layout & ~(AVIFGPU_SOURCE_CHROMA_INTERLEAVED | AVIFGPU_SOURCE_MSB_ALIGNED)) return Fail(error, AVIFGPU_ERR_BAD_PARAM, "unknown source layout bits");
        if (d->colorspace != AVIFGPU_COLORSPACE_YCBCR) return Fail(error, AVIFGPU_ERR_UNSUPPORTED, "semi-planar and MSB-aligned sources are YCbCr only");
        if ((layout & AVIFGPU_SOURCE_MSB_ALIGNED) && d->bit_depth != 10 && d->bit_depth != 12) return Fail(error, AVIFGPU_ERR_BAD_PARAM, "MSB-aligned sources need a 10- or 12-bit image");
    }
    return AVIFGPU_OK;
}

int32_t SourceLayoutOf(const avifgpu_decode_desc& d) { return d.struct_size == sizeof(avifgpu_decode_desc) ? d.source_layout : AVIFGPU_SOURCE_PLANAR; }

const avifgpu_decode_desc* WidenDecodeDesc(const avifgpu_decode_desc* d, avifgpu_decode_desc* full)
{
    if (d == nullptr || d->struct_size != AVIFGPU_DECODE_DESC_V9_SIZE)
    {
        return d;
    }
    std::memset(full, 0, sizeof(*full));
    std::memcpy(full, d, AVIFGPU_DECODE_DESC_V9_SIZE);
    full->struct_size = sizeof(avifgpu_decode_desc);
    full->source_layout = AVIFGPU_SOURCE_PLANAR;
    return full;
}

static void ChromaShifts(int chroma, int* xs, int* ys)
{
    // ReadHeifImage.cpp:52-81
    *xs = (chroma == AVIFGPU_CHROMA_420 || chroma == AVIFGPU_CHROMA_422) ? 1 : 0;
    *ys = (chroma == AVIFGPU_CHROMA_420) ? 1 : 0;
}

PlaneGeometry EncodePlaneGeometry(const avifgpu_encode_desc& d, int index)
{
    PlaneGeometry g;
    const bool hasAlpha = d.alpha_state != AVIFGPU_ALPHA_NONE;
    g.bytesPerSample = d.image_bit_depth > 8 ? 2 : 1;
    if (d.layout == AVIFGPU_LAYOUT_REFERENCE)
    {
        const bool gray = d.host_channels <= 2;
        if (index == 0)
        {
            g.present = true;
            g.widthSamples = gray ? d.width : d.width * d.host_channels;
            g.height = d.height;
        }
        else if (index == 3 && gray && hasAlpha)
        {
            g.present = true;
            g.widthSamples = d.width;
            g.height = d.height;
        }
    }
    else
    {
        int xs, ys;
        ChromaShifts(d.chroma, &xs, &ys);
        if (index == 0 || (index == 3 && hasAlpha))
        {
            g.present = true;
            g.widthSamples = d.width;
            g.height = d.height;
        }
        else if (index == 1 || index == 2)
        {
            // interleaved chroma: plane 1 holds the Cb, Cr pairs and there is no plane 2
            const bool interleaved = (DestLayoutOf(d) & AVIFGPU_SOURCE_CHROMA_INTERLEAVED) != 0;
            g.present = !(interleaved && index == 2);
            g.xs = xs;
            g.ys = ys;
            g.widthSamples = ((d.width + xs) >> xs) * (interleaved ? 2 : 1);
            g.height = (d.height + ys) >> ys;
        }
    }
    if (!g.present)
    {
        g.bytesPerSample = 0;
    }
    return g;
}

PlaneGeometry DecodePlaneGeometry(const avifgpu_decode_desc& d, int index)
{
    PlaneGeometry g;
    const bool hasAlpha = d.alpha_state != AVIFGPU_ALPHA_NONE;
    g.bytesPerSample = d.bit_depth > 8 ? 2 : 1;
    if (index == 0 || (index == 3 && hasAlpha))
    {
        g.present = true;
        g.widthSamples = d.width;
        g.height = d.height;
    }
    else if ((index == 1 || index == 2) && d.colorspace == AVIFGPU_COLORSPACE_YCBCR)
    {
        // interleaved chroma: plane 1 holds the Cb, Cr pairs and there is no plane 2
        const bool interleaved = (SourceLayoutOf(d) & AVIFGPU_SOURCE_CHROMA_INTERLEAVED) != 0;
        int xs, ys;
        ChromaShifts(d.chroma, &xs, &ys);
        g.present = !(interleaved && index == 2);
        g.xs = xs;
        g.ys = ys;
        g.widthSamples = ((d.width + xs) >> xs) * (interleaved ? 2 : 1);
        g.height = (d.height + ys) >> ys;
    }
    else if ((index == 1 || index == 2) && d.colorspace == AVIFGPU_COLORSPACE_RGB)
    {
        g.present = true;
        g.widthSamples = d.width;
        g.height = d.height;
    }
    if (!g.present)
    {
        g.bytesPerSample = 0;
    }
    return g;
}

int EncodeHostColBytes(const avifgpu_encode_desc& d) { return d.host_channels * ((d.host_depth + 7) / 8); }

int DecodeHostChannels(const avifgpu_decode_desc& d)
{
    const bool hasAlpha = d.alpha_state != AVIFGPU_ALPHA_NONE;
    if (d.colorspace == AVIFGPU_COLORSPACE_MONOCHROME)
    {
        return hasAlpha ? 2 : 1;
    }
    return hasAlpha ? 4 : 3;
}

int DecodeHostColBytes(const avifgpu_decode_desc& d) { return DecodeHostChannels(d) * ((d.host_depth + 7) / 8); }

void FillEncodeParams(const avifgpu_encode_desc& d, EncodeParams* p)
{
    std::memset(p, 0, sizeof(*p));
    p->width = d.width;
    p->channels = d.host_channels;
    p->hasAlpha = d.alpha_state != AVIFGPU_ALPHA_NONE;
    p->premultiply = d.alpha_state == AVIFGPU_ALPHA_PREMULTIPLIED;
    p->imageDepth = d.image_bit_depth;
    p->maxCode = (1u << d.image_bit_depth) - 1u;
    p->maxCodeFloat = static_cast<float>(p->maxCode);
    p->transfer = d.transfer;
    p->pqMultiplier = static_cast<float>(d.pq_peak_nits) / 10000.0f; // ColorTransfer.cpp:86
    p->gray16Smpte428 = (d.host_depth == 16 && d.host_channels <= 2 && d.gray16_curve == AVIFGPU_GRAY16_SMPTE428) ? 1 : 0;
    if (d.host_depth == 32 && d.transfer == AVIFGPU_TRANSFER_HLG && d.hlg_extension == AVIFGPU_HLG_INVERSE_OOTF_THEN_OETF)
    {
        p->hlgInverseOotf = 1;
        GetHlgLumaCoefficients(d.nclx.color_primaries, p->hlgLuma);
        p->hlgDisplayGamma = d.hlg_display_gamma;
        p->hlgPeak = static_cast<float>(d.hlg_peak_nits);
    }
    p->rowMatrixEnabled = (d.row_matrix_enabled && d.host_depth == 32 && d.host_channels >= 3) ? 1 : 0;
    for (int i = 0; i < 9; ++i)
    {
        p->rowMatrix[i] = d.row_matrix[i];
    }
    p->planar = d.layout == AVIFGPU_LAYOUT_PLANAR_YCBCR;
    p->destLayout = DestLayoutOf(d);
    if (p->planar)
    {
        int xs, ys;
        ChromaShifts(d.chroma, &xs, &ys);
        p->xs = xs;
        p->ys = ys;
        p->topLeft = d.down_filter == AVIFGPU_DOWN_FILTER_TOP_LEFT;
        float k[3];
        GetYuvCoefficients(&d.nclx, k);
        p->matrix.kr = k[0];
        p->matrix.kg = k[1];
        p->matrix.kb = k[2];
        p->matrix.cbScale = 0.5f / (1.0f - k[2]);
        p->matrix.crScale = 0.5f / (1.0f - k[0]);
        p->matrix.identity = (d.nclx.present && d.nclx.matrix_coefficients == 0) ? 1 : 0;
        // H.273 full range (and libheif's RGB->YCbCr): Ccode = Clip(Round(C) + 2^(depth-1)); neutral grey sits on 2^(depth-1).
        // (The reference DEcoder's chroma zero is max/2, YuvLookupTables.cpp:183: half a code lower -- its own business.)
        p->chromaOffset = p->matrix.identity ? 0.0f : static_cast<float>(1u << (d.image_bit_depth - 1));
    }
}

bool FillDecodeParams(const avifgpu_decode_desc& d, int32_t transfer, DecodeParams* p, std::string* error)
{
    std::memset(p, 0, sizeof(*p));
    p->width = d.width;
    p->colorspace = d.colorspace;
    if (d.colorspace == AVIFGPU_COLORSPACE_YCBCR)
    {
        int xs, ys;
        ChromaShifts(d.chroma, &xs, &ys);
        p->xs = xs;
        p->ys = ys;
    }
    p->hasAlpha = d.alpha_state != AVIFGPU_ALPHA_NONE;
    p->premultiplied = d.alpha_state == AVIFGPU_ALPHA_PREMULTIPLIED;
    p->bitDepth = d.bit_depth;
    p->maxCode = (1u << d.bit_depth) - 1u;
    p->sourceLayout = SourceLayoutOf(d);
    p->range = MakeRangeParams(&d.nclx, d.bit_depth, d.colorspace == AVIFGPU_COLORSPACE_MONOCHROME);
    if (d.colorspace == AVIFGPU_COLORSPACE_RGB)
    {
        p->range.fullRange = 1; // ReadHeifImage.cpp:402-415: plain i / max table
        p->range.identityMatrix = 0;
    }
    float k[3];
    GetYuvCoefficients(&d.nclx, k);
    p->matrix.kr = k[0];
    p->matrix.kg = k[1];
    p->matrix.kb = k[2];
    p->hostDepth = d.host_depth;
    p->transfer = transfer;
    p->pqMultiplier = 10000.0f / static_cast<float>(d.pq_peak_nits); // ColorTransfer.cpp:114
    p->applyOotf = d.hlg_apply_ootf != 0;
    p->gammaMinusOne = d.hlg_display_gamma - 1.0f; // ColorTransfer.cpp:201
    p->hlgPeak = static_cast<float>(d.hlg_peak_nits);
    if (d.host_depth == 32 && transfer == AVIFGPU_TRANSFER_HLG && d.hlg_apply_ootf && d.colorspace != AVIFGPU_COLORSPACE_MONOCHROME)
    {
        float luma[3];
        if (!GetHlgLumaCoefficients(d.nclx.color_primaries, luma))
        {
            if (error)
            {
                *error = "Unsupported color primaries for the HLG Luma Coefficients ";
            }
            return false;
        }
        p->lumaR = luma[0];
        p->lumaG = luma[1];
        p->lumaB = luma[2];
    }
    return true;
}


namespace
{
// The forward matrix's intermediates stay non-negative for kr, kg, kb >= 0 (all of H.273's matrices): the integer kernel's
// biased truncation rests on it.
bool BiasedTruncationHolds(const avifpix::ForwardMatrix& m)
{
    return m.identity || (m.kr >= 0.0f && m.kg >= 0.0f && m.kb >= 0.0f && m.kr < 1.0f && m.kb < 1.0f);
}
} // namespace

EncodeFamily EncodeFamilyOf(const EncodeParams& p, int hostDepth)
{
    const CurveTableView* table = p.curveTable;
    if (hostDepth == 32)
    {
        const bool pq = p.transfer == AVIFGPU_TRANSFER_PQ;
        const bool curve = pq || p.transfer == AVIFGPU_TRANSFER_SMPTE428;
        if (p.rowMatrixEnabled || p.imageDepth <= 8 || p.hlgInverseOotf)
        {
            return EncodeFamily::Generic; // the colour-profile matrix and the inverse OOTF are prologues of the generic kernel only
        }
        if (!p.planar && p.channels == 3 && !p.hasAlpha)
        {
            // the reference's own interleaved RGB codes (WriteHeifImage.cpp:1098-1130): the flat kernel without the matrix
            const bool fits = curve && table != nullptr && table->buckets != nullptr && (FlatCompactFits(*table) || FlatTwoLevelFits(*table));
            return fits ? EncodeFamily::RgbF32Interleaved : EncodeFamily::Generic;
        }
        if (!p.planar && p.channels <= 2)
        {
            // gray knows PQ and clip only (WriteHeifImage.cpp:586-587); PQ needs the verified compact table within the
            // kernel's shared memory
            if (p.transfer == AVIFGPU_TRANSFER_CLIP)
            {
                return EncodeFamily::GrayF32;
            }
            const bool fits = pq && table != nullptr && table->compact != nullptr && table->firstBits != nullptr && table->bandBits != nullptr &&
                              static_cast<size_t>(kGrayF32FixedBytes) + table->compactImageBytes <= static_cast<size_t>(kGrayF32SharedLimit);
            return fits ? EncodeFamily::GrayF32 : EncodeFamily::Generic;
        }
        const bool rgb = p.channels == 3 && !p.hasAlpha;
        const bool rgba = p.channels == 4 && p.hasAlpha;
        if (!p.planar || !(rgb || rgba))
        {
            return EncodeFamily::Generic;
        }
        // planar YCbCr; an exotic matrix takes the generic kernel, which clamps
        if ((!curve && p.transfer != AVIFGPU_TRANSFER_CLIP) || !ForwardMatrixStaysInRange(p.matrix, p.chromaOffset, static_cast<int>(p.maxCode)))
        {
            return EncodeFamily::Generic;
        }
        if (!curve)
        {
            return rgb ? EncodeFamily::RgbF32Clip : EncodeFamily::Generic; // the RGBA kernel is built on the step table
        }
        if (table == nullptr || table->buckets == nullptr)
        {
            return EncodeFamily::Generic; // no verified table for this curve: the generic exact kernel serves it
        }
        if (rgba)
        {
            // built on the compact table + band bitmap, staged next to the kernel's buffers
            const bool fits = table->compact != nullptr && table->firstBits != nullptr && table->bandBits != nullptr &&
                              static_cast<size_t>(RgbaFixedBytes()) + table->compactImageBytes <= static_cast<size_t>(kSharedLimit);
            return fits ? EncodeFamily::RgbaF32Flat : EncodeFamily::Generic;
        }
        // the other destination layouts have no PQ instantiation for the two-level table (kernels_fast_flat.cu)
        const bool fits = FlatCompactFits(*table) || (FlatTwoLevelFits(*table) && (p.destLayout == AVIFGPU_SOURCE_PLANAR || !pq));
        return fits ? EncodeFamily::RgbF32Flat : EncodeFamily::Generic;
    }
    if (hostDepth != 8 && hostDepth != 16)
    {
        return EncodeFamily::Generic;
    }
    if (hostDepth == 16 && p.imageDepth > 8 && p.channels == 1 && !p.planar)
    {
        return p.gray16Lut != nullptr ? EncodeFamily::Gray16Lut : EncodeFamily::Generic;
    }
    if (!p.planar && (p.channels == 1 || p.channels == 2))
    {
        // premultiplication and the Gray16 SMPTE 428 composition stay with the generic kernel
        return !p.premultiply && !p.gray16Smpte428 && p.imageDepth <= 12 ? EncodeFamily::GrayInt : EncodeFamily::Generic;
    }
    const bool rgbInt = p.planar && (p.channels == 3 || p.channels == 4) && (!p.premultiply || (p.channels == 4 && p.verifiedPremultiply)) &&
                        p.imageDepth <= 12 && BiasedTruncationHolds(p.matrix) && ForwardMatrixStaysInRange(p.matrix, p.chromaOffset, static_cast<int>(p.maxCode));
    return rgbInt ? EncodeFamily::RgbInt : EncodeFamily::Generic;
}

F32DecodeFactors F32DecodeFactorsOf(const avifpix::InverseMatrix& matrix)
{
    F32DecodeFactors f;
    f.rGain = (2 * (1 - matrix.kr));
    f.bGain = (2 * (1 - matrix.kb));
    f.gCr = matrix.kr * (1 - matrix.kr);
    f.gCb = matrix.kb * (1 - matrix.kb);
    f.kgReciprocal = 1.0f / matrix.kg;
    return f;
}

namespace
{
// True when every clamped channel sum Y + offset of the configuration is +0 or a normal float.  Table entries are 0 or at
// least 2^-14 in magnitude (depth <= 12: k / max, k / max - 0.5); with the matrix factors at least 2^-16 every product is 0 or
// at least 2^-30, a sum of two such floats is a multiple of 2^-53 (0 or at least that), the green term after its division a
// float of at least 2^-54, and Y minus it a multiple of 2^-77: nowhere near 2^-126.  Every H.273 matrix passes.
bool ChannelSumsStayNormal(int bitDepth, const F32DecodeFactors& f, float kg)
{
    const float least = 1.0f / 65536.0f;
    const auto moderate = [least](float v) { return v >= least && v <= 4.0f; };
    return bitDepth <= 12 && moderate(f.rGain) && moderate(f.bGain) && moderate(f.gCr) && moderate(f.gCb) && moderate(kg) &&
           moderate(f.kgReciprocal / 65536.0f * 4.0f);
}
} // namespace

namespace
{
// The float YCbCr decode: 10/12-bit YCbCr (+ straight alpha) into 32-bit hosts with the PQ, HLG or SMPTE 428 curve; for
// HLG the context's verified divisions, and with the OOTF an exponent and luma coefficients the branch-free powf covers;
// for PQ and SMPTE 428 a matrix whose channel sums are never subnormal.
bool YccF32Applies(const DecodeParams& p)
{
    if (p.colorspace != AVIFGPU_COLORSPACE_YCBCR || p.hostDepth != 32 || (p.hasAlpha && p.premultiplied) || p.bitDepth > 12 || p.bitDepth <= 8)
    {
        return false;
    }
    if (p.transfer != AVIFGPU_TRANSFER_PQ && p.transfer != AVIFGPU_TRANSFER_HLG && p.transfer != AVIFGPU_TRANSFER_SMPTE428)
    {
        return false;
    }
    if (p.transfer == AVIFGPU_TRANSFER_HLG && !p.verifiedHlgDivisions)
    {
        return false; // the tuned kernel is built on the verified constant divisions; the generic kernel divides
    }
    if (p.transfer == AVIFGPU_TRANSFER_HLG && p.applyOotf && !avifmath::PowfStraightLineCovers(p.gammaMinusOne, false))
    {
        return false; // the tuned kernel's OOTF is the branch-free powf (device_math.cuh PowfStraightLine): moderate exponents only
    }
    if (p.transfer == AVIFGPU_TRANSFER_HLG && p.applyOotf &&
        !(p.lumaR >= 0.0f && p.lumaG >= 0.0f && p.lumaB >= 0.0f && p.lumaR + p.lumaG + p.lumaB <= 2.5f))
    {
        return false; // the OOTF's luma must stay inside the kernel's log2 table (below 2.75) and non-negative
    }
    if (!avifmath::PowfStraightLineCovers(avifpix::PqConstants::inv_m2, true) || !avifmath::PowfStraightLineCovers(avifpix::PqConstants::inv_m1, true) ||
        !avifmath::PowfStraightLineCovers(2.6f, true))
    {
        return false; // constants of the curves: cannot happen, but the kernel's powf rests on it
    }
    if (p.transfer != AVIFGPU_TRANSFER_HLG && !ChannelSumsStayNormal(p.bitDepth, F32DecodeFactorsOf(p.matrix), p.matrix.kg))
    {
        return false; // PQ's and SMPTE 428's branch-free powf takes +0 or NORMAL bases (the generic kernel has the full powf)
    }
    return true;
}
} // namespace

DecodeFamily DecodeFamilyOf(const DecodeParams& p)
{
    if (p.hostDepth == 32)
    {
        const bool tenOrTwelve = p.bitDepth > 8 && p.bitDepth <= 12;
        switch (p.colorspace)
        {
        case AVIFGPU_COLORSPACE_YCBCR: return YccF32Applies(p) ? DecodeFamily::YccF32 : DecodeFamily::Generic;
        case AVIFGPU_COLORSPACE_MONOCHROME:
            // the reference's gray float path knows PQ only (YuvDecode.cpp:214-221)
            return tenOrTwelve && p.transfer == AVIFGPU_TRANSFER_PQ ? DecodeFamily::MonoF32 : DecodeFamily::Generic;
        case AVIFGPU_COLORSPACE_RGB:
            // premultiplied alpha too: the table kernel un-premultiplies in the integer domain
            return tenOrTwelve && (p.transfer == AVIFGPU_TRANSFER_PQ || p.transfer == AVIFGPU_TRANSFER_HLG || p.transfer == AVIFGPU_TRANSFER_SMPTE428)
                       ? DecodeFamily::PlanarRgbF32
                       : DecodeFamily::Generic;
        default: return DecodeFamily::Generic;
        }
    }
    // 8-bit hosts read 8-bit planes, 16-bit hosts 10/12-bit planes (ReadHeifImage.cpp:83, 186, 561-861)
    if ((p.hostDepth != 8 && p.hostDepth != 16) || p.bitDepth > 12 || (p.hasAlpha && p.premultiplied) || (p.hostDepth == 8) != (p.bitDepth <= 8))
    {
        return DecodeFamily::Generic;
    }
    switch (p.colorspace)
    {
    case AVIFGPU_COLORSPACE_YCBCR: return DecodeFamily::YccInt;
    case AVIFGPU_COLORSPACE_MONOCHROME: return DecodeFamily::MonoInt;
    case AVIFGPU_COLORSPACE_RGB: return DecodeFamily::PlanarRgbInt;
    default: return DecodeFamily::Generic;
    }
}

namespace
{
// Adds image i's plan to `plan`: its interior and windows to the last chunk (a new one when that is full), or the image to
// the direct calls when it is non-empty and has no interior.
void AddToBatch(const BatchImagePlan& image, int32_t i, BatchPlan* plan)
{
    if (image.interior.width == 0)
    {
        if (image.windows > 0)
        {
            plan->fallback.push_back(i);
        }
        return;
    }
    if (plan->chunks.empty() || plan->chunks.back().images == kBatchChunkImages)
    {
        plan->chunks.emplace_back();
    }
    BatchChunk& c = plan->chunks.back();
    c.interior[c.images] = image.interior;
    c.interior[c.images].firstUnit = c.interiorUnits;
    c.interiorUnits += image.interiorUnits;
    c.imageIndex[c.images++] = i;
    for (int k = 0; k < image.windows; ++k)
    {
        c.window[c.windows] = image.window[k];
        c.window[c.windows].firstUnit = c.windowUnits;
        c.windowUnits += image.windowUnits[k];
        c.windowImage[c.windows++] = i;
    }
}
} // namespace

void PlanEncodeBatch(const EncodeParams& shared, int hostDepth, int planeMask, const avifgpu_batch_image* images, int32_t count, BatchPlan* plan)
{
    plan->chunks.clear();
    plan->fallback.clear();
    const EncodeFamily family = EncodeBatchFamilyOf(shared, hostDepth);
    for (int32_t i = 0; i < count; ++i)
    {
        AddToBatch(PlanBatchEncodeImage(shared, hostDepth, family, planeMask, images[i]), i, plan);
    }
}

void PlanEncodeLightBatch(const EncodeParams& shared, int planeMask, const avifgpu_batch_image* images, int32_t count, BatchPlan* plan)
{
    plan->chunks.clear();
    plan->fallback.clear();
    const EncodeFamily family = EncodeLightBatchFamilyOf(shared, 32);
    for (int32_t i = 0; i < count; ++i)
    {
        AddToBatch(PlanBatchEncodeImage(shared, 32, family, planeMask, images[i], kLightBatchUnitPixels), i, plan);
    }
}

void PlanDecodeBatch(const DecodeParams& shared, int planeMask, const avifgpu_batch_image* images, int32_t count, BatchPlan* plan)
{
    plan->chunks.clear();
    plan->fallback.clear();
    const DecodeFamily family = DecodeBatchFamilyOf(shared);
    for (int32_t i = 0; i < count; ++i)
    {
        AddToBatch(PlanBatchDecodeImage(shared, family, planeMask, images[i]), i, plan);
    }
}

} // namespace avifgpu
