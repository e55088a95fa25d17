// tests/native/indirect_plan_check.cpp -- host-side check of the per-image planning step both batch APIs share
// (PlanBatchEncodeImage / PlanBatchDecodeImage, csrc/batch_plan.h) and of the device-described batch's workspace, compiled
// with the host compiler from the same __host__ __device__ functions the plan kernel runs.  For every supported encode
// and decode description (with and without the verified premultiply) and seeded random image sets of sizes 0 to 600,
// negative sizes, NULL rows, NULL planes and misaligned pointers and strides, on fake padded planes:
//   - a rejected image (negative size; non-empty with NULL rows or a NULL plane the description has) gets BAD_PARAM and
//     no record, an empty image OK and no record;
//   - every pixel of an accepted image is covered exactly once by its interior and windows, judged from the records'
//     rows pointers, and each record's luma and chroma planes sit at its first pixel and chroma site;
//   - an image has an interior exactly when EncodeBlockInterior / DecodeBlockInterior of the batched family of its own block (built here as a
//     direct call builds it) takes it, that interior is the predicate's rectangle, and its windows are the strips around
//     it; any other image is exactly one whole-image window; every unit count matches its record;
//   - with the records laid out at the exclusive prefix sums of their units (IndirectWorkspaceLayout), FindRecord finds
//     the owner of every unit from any earlier starting record.
// Prints "encode descriptions=N images=K" and "decode descriptions=N images=K"; exit code 1 on any failure.
#include "batch_plan.h"
#include "host_params.h"

#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

using namespace avifgpu;

namespace
{

long long g_failures = 0;

void Fail(const char* what, int description, int image)
{
    if (++g_failures <= 20)
    {
        std::printf("FAIL %s: description %d, image %d\n", what, description, image);
    }
}

bool SameRecord(const BatchRecord& a, const BatchRecord& b)
{
    // every field but the first unit, which the plan sets after its scan
    BatchRecord x = a, y = b;
    x.firstUnit = y.firstUnit = 0;
    return std::memcmp(&x, &y, sizeof(x)) == 0;
}

// Random batch_image records for a description with these plane geometries and bytes per host pixel.
std::vector<avifgpu_batch_image> RandomImages(std::mt19937& rng, int n, int colBytes, const int planeMask, const int planeXs[4], const int sampleBytes,
                                              std::vector<int>* expectRejected)
{
    std::vector<avifgpu_batch_image> images(n);
    expectRejected->assign(n, 0);
    for (int i = 0; i < n; ++i)
    {
        avifgpu_batch_image& im = images[i];
        std::memset(&im, 0, sizeof(im));
        const int kind = static_cast<int>(rng() % 12);
        im.width = kind == 0 ? static_cast<int>(rng() % 9) : static_cast<int>(rng() % 601);
        im.height = kind == 1 ? 1 + static_cast<int>(rng() % 2) : static_cast<int>(rng() % 601);
        if (kind == 2) im.width = 0;
        if (kind == 3) im.height = 0;
        if (kind == 4) (rng() % 2 ? im.width : im.height) = -1 - static_cast<int>(rng() % 5);
        const bool misaligned = kind == 5, oddStride = kind == 6;
        const uintptr_t base = static_cast<uintptr_t>(i + 1) << 36;
        im.rows = reinterpret_cast<void*>(base + (misaligned ? 2 : 0));
        const int w = im.width > 0 ? im.width : 1;
        im.row_stride_bytes = (static_cast<int64_t>(w) * colBytes + 63) / 64 * 64 + 64 + (oddStride ? 2 : 0);
        for (int k = 0; k < 4; ++k)
        {
            if ((planeMask >> k) & 1)
            {
                im.planes.data[k] = reinterpret_cast<void*>(base + (static_cast<uintptr_t>(k + 1) << 30) + (kind == 7 && k == 1 ? 4 : 0));
                im.planes.stride[k] = (static_cast<int64_t>((w + planeXs[k]) >> planeXs[k]) * sampleBytes + 63) / 64 * 64 + 64 + (kind == 10 && k == 0 ? 2 : 0);
            }
            else if (rng() % 2)
            {
                im.planes.data[k] = reinterpret_cast<void*>(base + (static_cast<uintptr_t>(k + 1) << 30)); // ignored: not a plane of the description
            }
        }
        const bool empty = im.width <= 0 || im.height <= 0;
        if (kind == 8) im.rows = nullptr;
        if (kind == 9)
        {
            int k = static_cast<int>(rng() % 4);
            while (!((planeMask >> k) & 1)) k = (k + 1) % 4;
            im.planes.data[k] = nullptr;
        }
        (*expectRejected)[i] = im.width < 0 || im.height < 0 || (!empty && (kind == 8 || kind == 9));
    }
    return images;
}

// Checks the plan `q` of an accepted, non-empty image against its own block `p` and `inner`, the single-image predicate's
// interior of that block.  A window has units of (1 << edgeXs) x (1 << edgeYs) pixels.
template <typename Params>
void CheckImagePlan(const char* direction, const BatchImagePlan& q, const Params& p, Interior inner, int colBytes, int sampleBytes, int edgeXs,
                    int edgeYs, int description, int image)
{
    char what[96];
    const auto fail = [&](const char* check)
    {
        std::snprintf(what, sizeof(what), "%s %s", direction, check);
        Fail(what, description, image);
    };
    // the records, as rectangles of the image read back from their rows pointers
    BatchRecord records[3];
    int count = 0;
    if (inner.width > 0)
    {
        if (q.interior.width != inner.width || q.interior.rowCount != inner.rows || q.interior.rows != p.rows ||
            q.interiorUnits != BatchInteriorUnits(inner.width, inner.rows, p.ys))
            fail("interior");
        if (q.interior.width == 0)
        {
            fail("image the predicate batches has no interior");
            return;
        }
        records[count++] = q.interior;
        const int strips = (inner.width < p.width ? 1 : 0) + (inner.rows < p.rowCount ? 1 : 0);
        if (q.windows != strips)
        {
            fail("window count");
            return;
        }
    }
    else if (q.interior.width != 0 || q.interiorUnits != 0 || q.windows != 1 || !SameRecord(q.window[0], RecordOf(p)) ||
             q.windowUnits[0] != BatchEdgeUnits(p.width, p.rowCount, edgeXs, edgeYs) || q.windowUnits[1] != 0)
    {
        fail("fallback is not one whole-image window");
        return;
    }
    for (int k = 0; k < q.windows; ++k)
    {
        if (q.windowUnits[k] != BatchEdgeUnits(q.window[k].width, q.window[k].rowCount, edgeXs, edgeYs)) fail("window");
        records[count++] = q.window[k];
    }
    if (q.windows < 2 && q.windowUnits[1] != 0) fail("missing window has units");
    int x0[3], y0[3];
    int64_t area = 0;
    for (int j = 0; j < count; ++j)
    {
        const BatchRecord& r = records[j];
        const int64_t offset = static_cast<int64_t>(reinterpret_cast<uintptr_t>(r.rows) - reinterpret_cast<uintptr_t>(p.rows));
        y0[j] = static_cast<int>(offset / p.rowStride);
        x0[j] = static_cast<int>(offset % p.rowStride) / colBytes;
        if (offset < 0 || (offset % p.rowStride) % colBytes || r.width <= 0 || r.rowCount <= 0 || x0[j] + r.width > p.width ||
            y0[j] + r.rowCount > p.rowCount)
        {
            fail("record outside its image");
            return;
        }
        area += static_cast<int64_t>(r.width) * r.rowCount;
        const uintptr_t luma = reinterpret_cast<uintptr_t>(p.plane[0]) + static_cast<uintptr_t>(y0[j] * p.planeStride[0] + x0[j] * sampleBytes);
        const uintptr_t chroma = reinterpret_cast<uintptr_t>(p.plane[1]) +
                                 static_cast<uintptr_t>((y0[j] >> p.ys) * p.planeStride[1] + (x0[j] >> p.xs) * sampleBytes);
        if (reinterpret_cast<uintptr_t>(r.plane[0]) != luma || reinterpret_cast<uintptr_t>(r.plane[1]) != chroma || (x0[j] & ((1 << p.xs) - 1)) ||
            (y0[j] & ((1 << p.ys) - 1)))
            fail("planes of a record");
        for (int i = 0; i < j; ++i)
        {
            const bool apart = x0[i] + records[i].width <= x0[j] || x0[j] + r.width <= x0[i] || y0[i] + records[i].rowCount <= y0[j] ||
                               y0[j] + r.rowCount <= y0[i];
            if (!apart) fail("records overlap");
        }
    }
    // disjoint rectangles inside the image whose areas add up to it cover every pixel exactly once
    if (area != static_cast<int64_t>(p.width) * p.rowCount) fail("pixel not covered exactly once");
}

// The plan kernel's output for `plans`, laid out serially, and FindRecord against a linear search over every unit.
void CheckLayoutAndSearch(std::mt19937& rng, const std::vector<BatchImagePlan>& plans, int description)
{
    const int n = static_cast<int>(plans.size());
    std::vector<int64_t> interiorFirst(n), windowFirst(2 * static_cast<size_t>(n));
    std::vector<int64_t> interiorUnits(n), windowUnits(2 * static_cast<size_t>(n));
    int64_t interiorTotal = 0, windowTotal = 0;
    for (int i = 0; i < n; ++i)
    {
        interiorFirst[i] = interiorTotal;
        interiorUnits[i] = plans[i].interiorUnits;
        interiorTotal += plans[i].interiorUnits;
        for (int k = 0; k < 2; ++k)
        {
            windowFirst[2 * i + k] = windowTotal;
            windowUnits[2 * i + k] = plans[i].windowUnits[k];
            windowTotal += plans[i].windowUnits[k];
        }
    }
    const auto check = [&](const std::vector<int64_t>& first, const std::vector<int64_t>& units, int64_t total)
    {
        const int count = static_cast<int>(first.size());
        if (count == 0 || total == 0) return;
        int owner = 0, record = 0;
        for (int64_t u = 0; u < total; u += 1 + static_cast<int64_t>(rng() % 97))
        {
            while (u >= first[owner] + units[owner]) ++owner;
            record = FindRecord(first.data(), count, rng() % 4 == 0 ? 0 : record, u);
            if (record != owner) Fail("FindRecord", description, owner);
        }
    };
    check(interiorFirst, interiorUnits, interiorTotal);
    check(windowFirst, windowUnits, windowTotal);
}

} // namespace

int main()
{
    std::mt19937 rng(4321);
    // the workspace sections are 256-byte aligned, in order, and large enough
    for (int m : { 1, 2, 63, 64, 1000, kIndirectMaxImages })
    {
        const IndirectLayout l = IndirectWorkspaceLayout(m);
        const size_t offsets[5] = { l.interiorFirst, l.windowFirst, l.interior, l.window, l.bytes };
        const size_t need[4] = { 8u * m, 16u * m, sizeof(BatchRecord) * m, 2 * sizeof(BatchRecord) * m };
        if (l.interiorFirst < sizeof(IndirectHeader)) Fail("layout header", m, 0);
        for (int k = 0; k < 4; ++k)
            if (offsets[k] % 256 || offsets[k + 1] < offsets[k] + need[k]) Fail("layout", m, k);
    }

    int descriptions = 0;
    long long images = 0;
    for (int hostDepth : { 8, 16 })
        for (int channels : { 3, 4 })
            for (int alpha : { 0, 1, 2 })
                for (int depth : { 8, 10, 12 })
                    for (int chroma : { 1, 2, 3 })
                        for (int matrix : { 1, 0, 9 })
                        {
                            avifgpu_encode_desc d{};
                            d.struct_size = sizeof(d);
                            d.host_depth = hostDepth;
                            d.host_channels = channels;
                            d.alpha_state = alpha;
                            d.image_bit_depth = depth;
                            d.transfer = AVIFGPU_TRANSFER_CLIP;
                            d.pq_peak_nits = 80;
                            d.layout = AVIFGPU_LAYOUT_PLANAR_YCBCR;
                            d.chroma = chroma;
                            d.nclx = avifgpu_nclx{ 1, 1, 13, matrix, 1 };
                            if (ValidateEncodeDesc(&d, nullptr) != AVIFGPU_OK)
                            {
                                continue;
                            }
                            ++descriptions;
                            int planeMask = 0, planeXs[4] = { 0, 0, 0, 0 };
                            for (int k = 0; k < 4; ++k)
                            {
                                const PlaneGeometry g = EncodePlaneGeometry(d, k);
                                planeMask |= g.present ? 1 << k : 0;
                                planeXs[k] = g.xs;
                            }
                            for (int verified : { 0, 1 })
                            {
                                EncodeParams shared;
                                FillEncodeParams(d, &shared);
                                shared.verifiedPremultiply = verified;
                                const EncodeFamily family = EncodeBatchFamilyOf(shared, hostDepth);
                        const bool tuned = family == EncodeFamily::RgbInt;
                                const int n = 1 + static_cast<int>(rng() % 120);
                                std::vector<int> rejected;
                                const std::vector<avifgpu_batch_image> batch =
                                    RandomImages(rng, n, EncodeHostColBytes(d), planeMask, planeXs, depth > 8 ? 2 : 1, &rejected);
                                images += n;
                                std::vector<BatchImagePlan> plans(n);
                                for (int i = 0; i < n; ++i)
                                {
                                    const BatchImagePlan& q = plans[i] = PlanBatchEncodeImage(shared, hostDepth, family, planeMask, batch[i]);
                                    if (q.status != (rejected[i] ? AVIFGPU_ERR_BAD_PARAM : AVIFGPU_OK)) Fail("encode status", descriptions, i);
                                    if (rejected[i] || batch[i].width == 0 || batch[i].height == 0)
                                    {
                                        if (q.windows != 0 || q.interiorUnits != 0 || q.windowUnits[0] != 0 || q.windowUnits[1] != 0 || q.interior.width != 0)
                                            Fail("encode records of a rejected or empty image", descriptions, i);
                                        continue;
                                    }
                                    // the image's own block, as the direct call of it builds it
                                    avifgpu_encode_desc di = d;
                                    di.width = batch[i].width;
                                    di.height = batch[i].height;
                                    EncodeParams p;
                                    FillEncodeParams(di, &p);
                                    p.verifiedPremultiply = verified;
                                    p.rows = batch[i].rows;
                                    p.rowStride = batch[i].row_stride_bytes;
                                    p.rowCount = di.height;
                                    for (int k = 0; k < 4; ++k)
                                    {
                                        if ((planeMask >> k) & 1)
                                        {
                                            p.plane[k] = batch[i].planes.data[k];
                                            p.planeStride[k] = batch[i].planes.stride[k];
                                        }
                                    }
                                    CheckImagePlan("encode", q, p, EncodeBlockInterior(EncodeBatchFamilyOf(p, hostDepth), p, hostDepth), EncodeHostColBytes(d), depth > 8 ? 2 : 1, p.xs, p.ys,
                                                   descriptions, i);
                                }
                                CheckLayoutAndSearch(rng, plans, descriptions);
                            }
                        }
    std::printf("encode descriptions=%d images=%lld\n", descriptions, images);

    int decodeDescriptions = 0;
    long long decodeImages = 0;
    for (int hostDepth : { 8, 16 })
        for (int bitDepth : { 8, 10, 12, 16 })
            for (int alpha : { 0, 1 })
                for (int chroma : { 1, 2, 3 })
                {
                    avifgpu_decode_desc d{};
                    d.struct_size = sizeof(d);
                    d.colorspace = AVIFGPU_COLORSPACE_YCBCR;
                    d.chroma = chroma;
                    d.bit_depth = bitDepth;
                    d.alpha_state = alpha;
                    d.host_depth = hostDepth;
                    d.nclx = avifgpu_nclx{ 1, 1, 13, 1, 1 };
                    d.pq_peak_nits = 80;
                    int32_t transfer = 0;
                    DecodeParams shared{};
                    if (ValidateDecodeDesc(&d, &transfer, nullptr) != AVIFGPU_OK || !FillDecodeParams(d, transfer, &shared, nullptr))
                    {
                        continue;
                    }
                    ++decodeDescriptions;
                    int planeMask = 0, planeXs[4] = { 0, 0, 0, 0 };
                    for (int k = 0; k < 4; ++k)
                    {
                        const PlaneGeometry g = DecodePlaneGeometry(d, k);
                        planeMask |= g.present ? 1 << k : 0;
                        planeXs[k] = g.xs;
                    }
                    const DecodeFamily family = DecodeBatchFamilyOf(shared);
                    const bool tuned = family == DecodeFamily::YccInt;
                    for (int trial = 0; trial < 4; ++trial)
                    {
                        const int n = 1 + static_cast<int>(rng() % 120);
                        std::vector<int> rejected;
                        const std::vector<avifgpu_batch_image> batch = RandomImages(rng, n, DecodeHostColBytes(d), planeMask, planeXs, bitDepth > 8 ? 2 : 1, &rejected);
                        decodeImages += n;
                        std::vector<BatchImagePlan> plans(n);
                        for (int i = 0; i < n; ++i)
                        {
                            const BatchImagePlan& q = plans[i] = PlanBatchDecodeImage(shared, family, planeMask, batch[i]);
                            if (q.status != (rejected[i] ? AVIFGPU_ERR_BAD_PARAM : AVIFGPU_OK)) Fail("decode status", decodeDescriptions, i);
                            if (rejected[i] || batch[i].width == 0 || batch[i].height == 0)
                            {
                                if (q.windows != 0 || q.interiorUnits != 0 || q.windowUnits[0] != 0 || q.windowUnits[1] != 0 || q.interior.width != 0)
                                    Fail("decode records of a rejected or empty image", decodeDescriptions, i);
                                continue;
                            }
                            avifgpu_decode_desc di = d;
                            di.width = batch[i].width;
                            di.height = batch[i].height;
                            DecodeParams p;
                            FillDecodeParams(di, transfer, &p, nullptr);
                            p.rows = batch[i].rows;
                            p.rowStride = batch[i].row_stride_bytes;
                            p.rowCount = di.height;
                            for (int k = 0; k < 4; ++k)
                            {
                                if ((planeMask >> k) & 1)
                                {
                                    p.plane[k] = batch[i].planes.data[k];
                                    p.planeStride[k] = batch[i].planes.stride[k];
                                }
                            }
                            CheckImagePlan("decode", q, p, DecodeBlockInterior(DecodeBatchFamilyOf(p), p), DecodeHostColBytes(d), bitDepth > 8 ? 2 : 1, 0, 0, decodeDescriptions, i);
                        }
                        CheckLayoutAndSearch(rng, plans, decodeDescriptions);
                    }
                }
    std::printf("decode descriptions=%d images=%lld\n", decodeDescriptions, decodeImages);
    return g_failures == 0 ? 0 : 1;
}
