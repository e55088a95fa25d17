// tests/native/launch_window_check.cpp -- host-side check of EncodeWindow / DecodeWindow (csrc/kernel_params.h), the
// sub-rectangles the tuned launchers hand to the generic kernel for their edge strips.
// Every valid encode and decode description is filled by FillEncodeParams / FillDecodeParams on fake, padded planes;
// every window of a grid of row blocks must point where EncodePlaneGeometry / DecodePlaneGeometry and
// Encode/DecodeHostColBytes put that pixel of the image, and a window of a window must equal the composed window.
// Prints "encode descriptions=N windows=M" and "decode descriptions=N windows=M"; exit code 1 on any mismatch.
#include "host_params.h"

#include <cstdio>
#include <cstring>

using namespace avifgpu;

namespace
{

constexpr int kWidth = 37;
constexpr int kHeight = 19;
constexpr int kBlockStarts[] = { 0, 1, 2, 5 };
constexpr int kWindowX[] = { 0, 1, 3, 8, 16, kWidth - 1 };
constexpr int kWindowY[] = { 0, 1, 2, 3, 7 };
constexpr int kInnerX[] = { 0, 1, 3 };
constexpr int kInnerY[] = { 0, 1, 2 };

long long g_windows = 0;
long long g_failures = 0;

void Fail(const char* what, const char* direction, int index, int y, int x0, int y0)
{
    if (++g_failures <= 20)
    {
        std::printf("MISMATCH %s %s: description %d, block start %d, window (%d, %d)\n", direction, what, index, y, x0, y0);
    }
}

uintptr_t Address(const void* p) { return reinterpret_cast<uintptr_t>(p); }

// A plane of the image at a fake base address, with a padded row stride.
struct FakePlane
{
    PlaneGeometry g;
    uintptr_t base = 0;
    int64_t stride = 0;

    // Samples of one pixel (or chroma site) in this plane: 1, or the channel count of an interleaved plane.
    int SamplesPerSite(int width) const { return g.widthSamples / ((width + g.xs) >> g.xs); }

    // Where pixel (x, y) of the image lives, from the geometry alone.
    uintptr_t At(int width, int x, int y) const
    {
        return base + static_cast<uintptr_t>((y >> g.ys) * stride) +
               static_cast<uintptr_t>((x >> g.xs) * SamplesPerSite(width) * g.bytesPerSample);
    }
};

FakePlane MakePlane(const PlaneGeometry& g, int k)
{
    FakePlane f;
    f.g = g;
    if (g.present)
    {
        f.base = (static_cast<uintptr_t>(k) + 1) << 32;
        f.stride = static_cast<int64_t>(g.widthSamples) * g.bytesPerSample + 64 + 16 * k;
    }
    return f;
}

const uintptr_t kRowsBase = static_cast<uintptr_t>(9) << 32;

// The part of a window both directions share: rows, planes, size.
template <typename Params>
void CheckCommon(const Params& w, const Params& block, const FakePlane planes[4], uintptr_t rowsAt, int width, int rows,
                 const char* direction, int index, int y, int x0, int y0, int ix, int iy)
{
    if (Address(w.rows) != rowsAt) Fail("rows", direction, index, y, x0, y0);
    if (w.rowStride != block.rowStride) Fail("row stride", direction, index, y, x0, y0);
    for (int k = 0; k < 4; ++k)
    {
        if (!planes[k].g.present)
        {
            if (w.plane[k] != nullptr) Fail("absent plane", direction, index, y, x0, y0);
            continue;
        }
        if (Address(w.plane[k]) != planes[k].At(kWidth, ix, iy)) Fail("plane", direction, index, y, x0, y0);
        if (w.planeStride[k] != block.planeStride[k]) Fail("plane stride", direction, index, y, x0, y0);
    }
    if (w.width != width || w.rowCount != rows) Fail("size", direction, index, y, x0, y0);
}

// One window [x0, x0 + width) x [y0, y0 + rows) of the block starting at image row y, and windows of it.  A window
// whose x0 (or, without a row phase, y0) splits a chroma site has no window of its own: (x0 & siteMaskX) != 0 or
// (y0 & siteMaskY) != 0.
template <typename Params, typename Window, typename Extra>
void CheckWindows(const Params& block, const FakePlane planes[4], int colBytes, int y, int siteMaskX, int siteMaskY,
                  const char* direction, int index, Window window, Extra extra)
{
    for (int x0 : kWindowX)
    {
        for (int y0 : kWindowY)
        {
            const int blockRows = kHeight - y;
            if (y0 >= blockRows)
            {
                continue;
            }
            for (int width : { kWidth - x0, (kWidth - x0 + 1) / 2 })
            {
                const int rows = blockRows - y0;
                const Params w = window(block, x0, y0, width, rows);
                ++g_windows;
                const uintptr_t rowsAt = kRowsBase + static_cast<uintptr_t>((y + y0) * block.rowStride) + static_cast<uintptr_t>(x0 * colBytes);
                CheckCommon(w, block, planes, rowsAt, width, rows, direction, index, y, x0, y0, x0, y + y0);
                extra(w, y + y0, index, y, x0, y0);
                for (int x1 : kInnerX)
                {
                    for (int y1 : kInnerY)
                    {
                        if (x1 >= width || y1 >= rows || (x0 & siteMaskX) != 0 || (y0 & siteMaskY) != 0)
                        {
                            continue;
                        }
                        const Params nested = window(w, x1, y1, width - x1, rows - y1);
                        const Params composed = window(block, x0 + x1, y0 + y1, width - x1, rows - y1);
                        ++g_windows;
                        bool same = nested.rows == composed.rows && nested.width == composed.width && nested.rowCount == composed.rowCount;
                        for (int k = 0; k < 4; ++k)
                        {
                            same = same && nested.plane[k] == composed.plane[k];
                        }
                        if (!same) Fail("window of a window", direction, index, y, x0 + x1, y0 + y1);
                        const uintptr_t nestedRowsAt = rowsAt + static_cast<uintptr_t>(y1 * block.rowStride) + static_cast<uintptr_t>(x1 * colBytes);
                        CheckCommon(nested, block, planes, nestedRowsAt, width - x1, rows - y1, direction, index, y, x0 + x1, y0 + y1, x0 + x1, y + y0 + y1);
                        extra(nested, y + y0 + y1, index, y, x0 + x1, y0 + y1);
                        extra(composed, y + y0 + y1, index, y, x0 + x1, y0 + y1);
                    }
                }
            }
        }
    }
}

void CheckEncode()
{
    int descriptions = 0;
    for (int hostDepth : { 8, 16, 32 })
    for (int channels = 1; channels <= 4; ++channels)
    for (int alpha : { AVIFGPU_ALPHA_NONE, AVIFGPU_ALPHA_STRAIGHT, AVIFGPU_ALPHA_PREMULTIPLIED })
    for (int layout : { AVIFGPU_LAYOUT_REFERENCE, AVIFGPU_LAYOUT_PLANAR_YCBCR })
    for (int chroma : { AVIFGPU_CHROMA_444, AVIFGPU_CHROMA_422, AVIFGPU_CHROMA_420 })
    for (int depth : { 8, 10, 12 })
    {
        avifgpu_encode_desc d;
        std::memset(&d, 0, sizeof(d));
        d.struct_size = sizeof(d);
        d.width = kWidth;
        d.height = kHeight;
        d.host_depth = hostDepth;
        d.host_channels = channels;
        d.alpha_state = alpha;
        d.image_bit_depth = depth;
        d.transfer = AVIFGPU_TRANSFER_PQ;
        d.pq_peak_nits = 10000;
        d.layout = layout;
        d.chroma = chroma;
        if (layout == AVIFGPU_LAYOUT_REFERENCE && chroma != AVIFGPU_CHROMA_444)
        {
            continue; // chroma means nothing to the reference layout: enumerate it once
        }
        if (ValidateEncodeDesc(&d, nullptr) != AVIFGPU_OK)
        {
            continue;
        }
        const int index = descriptions++;
        FakePlane planes[4];
        for (int k = 0; k < 4; ++k)
        {
            planes[k] = MakePlane(EncodePlaneGeometry(d, k), k);
        }
        const int colBytes = EncodeHostColBytes(d);
        for (int y : kBlockStarts)
        {
            EncodeParams p;
            FillEncodeParams(d, &p);
            if ((y & p.ys) != 0)
            {
                continue; // an encode block starts on a chroma row
            }
            p.rowStride = static_cast<int64_t>(kWidth) * colBytes + 48;
            p.rows = reinterpret_cast<const void*>(kRowsBase + static_cast<uintptr_t>(y * p.rowStride));
            p.rowCount = kHeight - y;
            for (int k = 0; k < 4; ++k)
            {
                if (planes[k].g.present)
                {
                    p.plane[k] = reinterpret_cast<void*>(planes[k].At(kWidth, 0, y));
                    p.planeStride[k] = planes[k].stride;
                }
            }
            const auto window = [hostDepth](const EncodeParams& b, int x0, int y0, int width, int rows)
            { return EncodeWindow(b, hostDepth, x0, y0, width, rows); };
            const auto noExtra = [](const EncodeParams&, int, int, int, int, int) {};
            CheckWindows(p, planes, colBytes, y, planes[1].g.xs, planes[1].g.ys, "encode", index, window, noExtra);
        }
    }
    std::printf("encode descriptions=%d windows=%lld\n", descriptions, g_windows);
}

void CheckDecode()
{
    const long long before = g_windows;
    int descriptions = 0;
    for (int colorspace : { AVIFGPU_COLORSPACE_YCBCR, AVIFGPU_COLORSPACE_RGB, AVIFGPU_COLORSPACE_MONOCHROME })
    for (int alpha : { AVIFGPU_ALPHA_NONE, AVIFGPU_ALPHA_STRAIGHT, AVIFGPU_ALPHA_PREMULTIPLIED })
    for (int chroma : { AVIFGPU_CHROMA_444, AVIFGPU_CHROMA_422, AVIFGPU_CHROMA_420 })
    for (int depth : { 8, 10, 12, 16 })
    for (int hostDepth : { 8, 16, 32 })
    {
        avifgpu_decode_desc d;
        std::memset(&d, 0, sizeof(d));
        d.struct_size = sizeof(d);
        d.width = kWidth;
        d.height = kHeight;
        d.colorspace = colorspace;
        d.chroma = colorspace == AVIFGPU_COLORSPACE_MONOCHROME ? AVIFGPU_CHROMA_MONOCHROME : chroma;
        if (colorspace != AVIFGPU_COLORSPACE_YCBCR && chroma != AVIFGPU_CHROMA_444)
        {
            continue; // chroma means nothing to these colour spaces: enumerate each once
        }
        d.bit_depth = depth;
        d.alpha_state = alpha;
        d.host_depth = hostDepth;
        d.nclx.present = 1;
        d.nclx.color_primaries = 9;
        d.nclx.transfer_characteristics = 16;
        d.nclx.matrix_coefficients = 9;
        d.nclx.full_range_flag = 1;
        d.pq_peak_nits = 10000;
        d.hlg_display_gamma = 1.2f;
        d.hlg_peak_nits = 1000;
        int32_t transfer;
        DecodeParams p;
        if (ValidateDecodeDesc(&d, &transfer, nullptr) != AVIFGPU_OK || !FillDecodeParams(d, transfer, &p, nullptr))
        {
            continue;
        }
        const int index = descriptions++;
        FakePlane planes[4];
        for (int k = 0; k < 4; ++k)
        {
            planes[k] = MakePlane(DecodePlaneGeometry(d, k), k);
        }
        const int chromaRows = planes[1].g.ys; // the image's vertical chroma shift: 0 unless 4:2:0
        const int colBytes = DecodeHostColBytes(d);
        for (int y : kBlockStarts)
        {
            p.rowStride = static_cast<int64_t>(kWidth) * colBytes + 48;
            p.rows = reinterpret_cast<void*>(kRowsBase + static_cast<uintptr_t>(y * p.rowStride));
            p.rowCount = kHeight - y;
            p.yPhase = y & p.ys;
            for (int k = 0; k < 4; ++k)
            {
                if (planes[k].g.present)
                {
                    p.plane[k] = reinterpret_cast<const void*>(planes[k].At(kWidth, 0, y));
                    p.planeStride[k] = planes[k].stride;
                }
            }
            const auto window = [](const DecodeParams& b, int x0, int y0, int width, int rows) { return DecodeWindow(b, x0, y0, width, rows); };
            const auto phase = [chromaRows](const DecodeParams& w, int imageRow, int index, int y, int x0, int y0)
            {
                if (w.yPhase != (imageRow & chromaRows)) Fail("yPhase", "decode", index, y, x0, y0);
            };
            CheckWindows(p, planes, colBytes, y, planes[1].g.xs, 0, "decode", index, window, phase);
        }
    }
    std::printf("decode descriptions=%d windows=%lld\n", descriptions, g_windows - before);
}

} // namespace

int main()
{
    CheckEncode();
    CheckDecode();
    if (g_failures != 0)
    {
        std::printf("%lld mismatches\n", g_failures);
        return 1;
    }
    return 0;
}
