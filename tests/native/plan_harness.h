// tests/native/plan_harness.h -- the checks of the batch planning (csrc/batch_plan.h, csrc/host_params.cpp) that every
// batched description gets, whichever direction and family it takes.  Test code, header only.
//
// For one description and one seeded batch of fake images on fake padded planes (MakeBatch), CheckBatch runs:
//   CheckImageStep       the per-image step (PlanBatchEncodeImage / PlanBatchDecodeImage) that the plan kernel of the
//                        device-described batch runs: statuses, the route's interior, its strips, unit counts, placement;
//   CheckLayoutAndSearch the step's records at their prefix sums, as the plan kernel lays them out, and FindRecord;
//   CheckHostPlan        the chunks and direct calls of the host-described batch (PlanEncodeBatch / PlanDecodeBatch).
// A record's rectangle is read back from its rows pointer and its planes are held to EncodeWindow / DecodeWindow, so every
// pixel's coverage is judged from what the kernels are handed.
#ifndef AVIF_TESTS_PLAN_HARNESS_H
#define AVIF_TESTS_PLAN_HARNESS_H

#include "batch_plan.h"
#include "host_params.h"

#include <sys/mman.h>
#include <unistd.h>

#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

namespace avifgpu
{

inline long long g_failures = 0;

inline void Fail(const char* what, int description, int index)
{
    if (++g_failures <= 20)
    {
        std::printf("FAIL %s: description %d, batch or image %d\n", what, description, index);
    }
}

// ---- what differs by direction ----

inline PlaneGeometry Geometry(const avifgpu_encode_desc& d, int k) { return EncodePlaneGeometry(d, k); }
inline PlaneGeometry Geometry(const avifgpu_decode_desc& d, int k) { return DecodePlaneGeometry(d, k); }
inline int HostColBytes(const avifgpu_encode_desc& d) { return EncodeHostColBytes(d); }
inline int HostColBytes(const avifgpu_decode_desc& d) { return DecodeHostColBytes(d); }

inline EncodeParams Window(const EncodeParams& p, int hostDepth, int x0, int y0, int width, int rows)
{
    return EncodeWindow(p, hostDepth, x0, y0, width, rows);
}
inline DecodeParams Window(const DecodeParams& p, int, int x0, int y0, int width, int rows) { return DecodeWindow(p, x0, y0, width, rows); }

// The interior the route gives a block: the batched family's block half.
inline Interior RouteInterior(const EncodeParams& p, int hostDepth) { return EncodeBlockInterior(EncodeBatchFamilyOf(p, hostDepth), p, hostDepth); }
inline Interior RouteInterior(const DecodeParams& p, int) { return DecodeBlockInterior(DecodeBatchFamilyOf(p), p); }

inline BatchImagePlan PlanImage(const EncodeParams& shared, int hostDepth, int planeMask, const avifgpu_batch_image& image)
{
    return PlanBatchEncodeImage(shared, hostDepth, EncodeBatchFamilyOf(shared, hostDepth), planeMask, image);
}
inline BatchImagePlan PlanImage(const DecodeParams& shared, int, int planeMask, const avifgpu_batch_image& image)
{
    return PlanBatchDecodeImage(shared, DecodeBatchFamilyOf(shared), planeMask, image);
}

inline void PlanBatch(const EncodeParams& shared, int hostDepth, int planeMask, const std::vector<avifgpu_batch_image>& images, BatchPlan* plan)
{
    PlanEncodeBatch(shared, hostDepth, planeMask, images.data(), static_cast<int32_t>(images.size()), plan);
}
inline void PlanBatch(const DecodeParams& shared, int, int planeMask, const std::vector<avifgpu_batch_image>& images, BatchPlan* plan)
{
    PlanDecodeBatch(shared, planeMask, images.data(), static_cast<int32_t>(images.size()), plan);
}

// Interior units are UnitPixels pixels of one row (row pair for 4:2:0); edge units are runs of chroma sites (encode) or
// pixels (decode) of one row (pair).
inline int UnitPixels(const EncodeParams&, int) { return kBatchUnitPixels; }
inline int UnitPixels(const DecodeParams& p, int) { return DecodeBatchUnitPixels(DecodeBatchFamilyOf(p)); }
inline int64_t EdgeUnits(const EncodeParams& p, int width, int rows) { return BatchEdgeUnits(width, rows, p.xs, p.ys); }
inline int64_t EdgeUnits(const DecodeParams&, int width, int rows) { return BatchEdgeUnits(width, rows, 0, 0); }

inline bool Interleaved(const EncodeParams& p) { return SourceInterleaved(p.destLayout); }
inline bool Interleaved(const DecodeParams& p) { return SourceInterleaved(p.sourceLayout); }
inline int SampleBytes(const EncodeParams& p) { return p.imageDepth > 8 ? 2 : 1; }
inline int SampleBytes(const DecodeParams& p) { return p.bitDepth > 8 ? 2 : 1; }

// The alignment the tuned kernels' pair loads and stores need of interleaved plane 1, restated from them: twice the planar
// chroma's bytes per thread, at most 16 (16-bit 4:4:4 is two 128-bit accesses).  Encodes: integer hosts write 4 or 8 sites
// of 1 or 2 bytes, float hosts 2 or 4 sites of 2 bytes.  Decodes: integer hosts read 4 or 8 sites of 1 or 2 bytes, float
// hosts 4 or 8 bytes.
inline int PairAlignment(const EncodeParams& p, bool floatHost = false)
{
    const int planar = floatHost ? (p.xs ? 4 : 8) : (p.xs ? 4 : 8) * (p.imageDepth > 8 ? 2 : 1);
    return 2 * planar > 16 ? 16 : 2 * planar;
}
inline int PairAlignment(const DecodeParams& p)
{
    if (p.hostDepth == 32)
    {
        return 2 * (p.xs ? 4 : 8);
    }
    const int planar = (p.xs ? 4 : 8) * (p.hostDepth == 8 ? 1 : 2);
    return 2 * planar > 16 ? 16 : 2 * planar;
}

// ---- the fake batch ----

// One description as the planners see it: its block with the context's first-use state, its host depth, its planes
// (bit k: plane k), the bytes of one host pixel and of one pixel of plane 0 (from the host plane geometry).
template <typename Params>
struct Case
{
    Params shared;
    int hostDepth;
    int planeMask;
    int colBytes;
    int plane0Bytes;
    int index; // the description's number in its slice, for failure messages
};

template <typename Desc, typename Params>
Case<Params> CaseOf(const Desc& d, const Params& shared, int index)
{
    Desc onePixel = d;
    onePixel.width = 1;
    const PlaneGeometry g0 = Geometry(onePixel, 0);
    Case<Params> c{ shared, d.host_depth, 0, HostColBytes(d), g0.widthSamples * g0.bytesPerSample, index };
    for (int k = 0; k < 4; ++k)
    {
        c.planeMask |= Geometry(d, k).present ? 1 << k : 0;
    }
    return c;
}

// What the generator did to an image beyond its size.  kNegativeSize, kNullRows and kNullPlane are rejected, and the host
// planner never sees them: the host-described API validates every image before it plans the batch.
enum Shape
{
    kAligned,
    kOneRow,
    kRowsBy2,
    kRowsBy4,
    kRowsBy8,
    kOddRowStride,
    kPlane0By2,
    kPlaneBy2,      // a random plane of the description
    kPlaneBy8,
    kUnequalChroma, // Cr's stride is not Cb's
    kPairPointer,   // interleaved plane 1 misaligned by half its pair alignment
    kPairStride,
    kEmpty,
    kNegativeSize,
    kNullRows,
    kNullPlane,     // a plane the description has
    kShapes
};

template <typename Params>
struct FakeImage
{
    avifgpu_batch_image record; // what the caller passes
    Params p;                   // its own block, as a direct call of it builds it (accepted images)
    int shape;
    bool rejected;              // the API answers BAD_PARAM
};

constexpr int kEdgeWidths[] = { 1, 2, 3, 7, 8, 9, 255, 256, 257, 512, 513 };

// `n` images of the description `d`: widths 1 to 9, the edge widths and random ones up to 600, heights 1 to 9, rows at
// (i + 1) << 36 and plane k at that plus (k + 1) << 30, strides padded past 64-byte multiples, then the image's shape;
// every other image also sets the planes the description does not have, which the planners must ignore.
template <typename Desc, typename Params>
std::vector<FakeImage<Params>> MakeBatch(std::mt19937_64& rng, const Desc& d, const Case<Params>& c, int n)
{
    std::vector<FakeImage<Params>> images(n);
    for (int i = 0; i < n; ++i)
    {
        FakeImage<Params>& im = images[i];
        avifgpu_batch_image& r = im.record;
        std::memset(&r, 0, sizeof(r));
        const int roll = static_cast<int>(rng() % (2 * kShapes)); // half the images aligned
        const int shape = im.shape = roll < kShapes ? roll : kAligned;
        const int widthKind = static_cast<int>(rng() % 4);
        Desc di = d;
        di.width = widthKind == 0   ? 1 + static_cast<int>(rng() % 9)
                   : widthKind == 1 ? kEdgeWidths[rng() % (sizeof(kEdgeWidths) / sizeof(kEdgeWidths[0]))]
                                    : 1 + static_cast<int>(rng() % 600);
        di.height = shape == kOneRow ? 1 : 1 + static_cast<int>(rng() % 9);
        r.width = di.width;
        r.height = di.height;
        const uintptr_t base = static_cast<uintptr_t>(i + 1) << 36;
        r.rows = reinterpret_cast<void*>(base + (shape == kRowsBy2 ? 2 : shape == kRowsBy4 ? 4 : shape == kRowsBy8 ? 8 : 0));
        r.row_stride_bytes = (static_cast<int64_t>(di.width) * c.colBytes + 63) / 64 * 64 + 64 + (shape == kOddRowStride ? 2 : 0);
        const int oddPlane = static_cast<int>(rng() % 4);
        const bool extraPlanes = rng() % 2;
        for (int k = 0; k < 4; ++k)
        {
            const PlaneGeometry g = Geometry(di, k);
            if (g.present)
            {
                const uintptr_t off = (shape == kPlane0By2 && k == 0) || (shape == kPlaneBy2 && k == oddPlane) ? 2 : shape == kPlaneBy8 && k == oddPlane ? 8 : 0;
                r.planes.data[k] = reinterpret_cast<void*>(base + (static_cast<uintptr_t>(k + 1) << 30) + off);
                r.planes.stride[k] = (static_cast<int64_t>(g.widthSamples) * g.bytesPerSample + 63) / 64 * 64 + 128;
            }
            else if (extraPlanes)
            {
                r.planes.data[k] = reinterpret_cast<void*>(base + (static_cast<uintptr_t>(k + 1) << 30));
                r.planes.stride[k] = 64;
            }
        }
        if (shape == kUnequalChroma && ((c.planeMask >> 2) & 1))
        {
            r.planes.stride[2] += 64;
        }
        if ((shape == kPairPointer || shape == kPairStride) && Interleaved(c.shared))
        {
            const int half = PairAlignment(c.shared) / 2;
            if (shape == kPairPointer)
            {
                r.planes.data[1] = static_cast<uint8_t*>(r.planes.data[1]) + half;
            }
            else
            {
                r.planes.stride[1] += half;
            }
        }
        if (shape == kEmpty)
        {
            (rng() % 2 ? r.width : r.height) = 0;
        }
        if (shape == kNegativeSize)
        {
            (rng() % 2 ? r.width : r.height) = -1 - static_cast<int>(rng() % 5);
        }
        if (shape == kNullRows)
        {
            r.rows = nullptr;
        }
        if (shape == kNullPlane)
        {
            int k = static_cast<int>(rng() % 4);
            while (!((c.planeMask >> k) & 1))
            {
                k = (k + 1) % 4;
            }
            r.planes.data[k] = nullptr;
        }
        im.rejected = shape == kNegativeSize || shape == kNullRows || shape == kNullPlane;
        im.p = c.shared;
        im.p.width = r.width;
        im.p.rowCount = r.height;
        im.p.rows = r.rows;
        im.p.rowStride = r.row_stride_bytes;
        for (int k = 0; k < 4; ++k)
        {
            if ((c.planeMask >> k) & 1)
            {
                im.p.plane[k] = r.planes.data[k];
                im.p.planeStride[k] = r.planes.stride[k];
            }
        }
    }
    return images;
}

// ---- record placement and coverage ----

struct Rect
{
    int x0, y0, width, rows;
    bool operator==(const Rect& o) const { return x0 == o.x0 && y0 == o.y0 && width == o.width && rows == o.rows; }
};

// The rectangle of `p` that the record `r` starts, read back from its rows pointer; false (and a failure) when it is not
// inside the image on a chroma site (a row pair for 4:2:0) or its planes are not where the window of that rectangle puts
// them.  Planes 0 and 1 are also restated here: interleaved chroma moves by two samples per site and has no plane 2.
template <typename Params>
bool Place(const Case<Params>& c, const Params& p, const BatchRecord& r, Rect* rect)
{
    const int64_t offset = static_cast<int64_t>(reinterpret_cast<uintptr_t>(r.rows) - reinterpret_cast<uintptr_t>(p.rows));
    const int y0 = static_cast<int>(offset / p.rowStride), column = static_cast<int>(offset % p.rowStride);
    const int x0 = column / c.colBytes;
    if (offset < 0 || column % c.colBytes || r.width <= 0 || r.rowCount <= 0 || x0 + r.width > p.width || y0 + r.rowCount > p.rowCount ||
        (x0 & ((1 << p.xs) - 1)) || (y0 & ((1 << p.ys) - 1)) || r.rowStride != p.rowStride)
    {
        Fail("record outside its image or off a chroma site", c.index, -1);
        return false;
    }
    *rect = Rect{ x0, y0, r.width, r.rowCount };
    const Params w = Window(p, c.hostDepth, x0, y0, r.width, r.rowCount);
    for (int k = 0; k < 4; ++k)
    {
        if (r.plane[k] != w.plane[k] || r.planeStride[k] != p.planeStride[k])
        {
            Fail("record plane not where the window puts it", c.index, -1);
            return false;
        }
    }
    const auto moved = [&](int k) { return static_cast<const uint8_t*>(r.plane[k]) - static_cast<const uint8_t*>(p.plane[k]); };
    if (moved(0) != static_cast<int64_t>(y0) * p.planeStride[0] + static_cast<int64_t>(x0) * c.plane0Bytes)
    {
        Fail("plane 0 not at the record's first pixel", c.index, -1);
        return false;
    }
    if (p.plane[1] != nullptr)
    {
        const int64_t expected = static_cast<int64_t>(y0 >> p.ys) * p.planeStride[1] + static_cast<int64_t>(x0 >> p.xs) * (Interleaved(p) ? 2 : 1) * SampleBytes(p);
        if (moved(1) != expected || (Interleaved(p) && r.plane[2] != nullptr))
        {
            Fail("plane 1 not at the record's first site", c.index, -1);
            return false;
        }
    }
    return true;
}

// Rectangles inside a width x rows image that are pairwise disjoint and whose areas add up to it cover every pixel once.
inline bool CoveredOnce(const std::vector<Rect>& rects, int width, int rows)
{
    int64_t area = 0;
    for (size_t j = 0; j < rects.size(); ++j)
    {
        const Rect& a = rects[j];
        area += static_cast<int64_t>(a.width) * a.rows;
        for (size_t i = 0; i < j; ++i)
        {
            const Rect& b = rects[i];
            if (a.x0 < b.x0 + b.width && b.x0 < a.x0 + a.width && a.y0 < b.y0 + b.rows && b.y0 < a.y0 + a.rows)
            {
                return false;
            }
        }
    }
    return area == static_cast<int64_t>(width) * rows;
}

// ---- the three checks ----

// The per-image step for every image: BAD_PARAM and no record for a rejected image, OK and no record for an empty one; a
// batched image's interior is the route's and its windows are exactly InteriorStrips; any other image is one whole-image
// window; unit counts match the records, and the records cover the image exactly once.
template <typename Params>
std::vector<BatchImagePlan> CheckImageStep(const Case<Params>& c, const std::vector<FakeImage<Params>>& images)
{
    std::vector<BatchImagePlan> plans(images.size());
    for (size_t i = 0; i < images.size(); ++i)
    {
        const FakeImage<Params>& im = images[i];
        const Params& p = im.p;
        const BatchImagePlan& q = plans[i] = PlanImage(c.shared, c.hostDepth, c.planeMask, im.record);
        if (q.status != (im.rejected ? AVIFGPU_ERR_BAD_PARAM : AVIFGPU_OK))
        {
            Fail("step status", c.index, static_cast<int>(i));
        }
        if (im.rejected || p.width == 0 || p.rowCount == 0)
        {
            if (q.windows != 0 || q.interior.width != 0 || q.interiorUnits != 0 || q.windowUnits[0] != 0 || q.windowUnits[1] != 0)
            {
                Fail("step records of a rejected or empty image", c.index, static_cast<int>(i));
            }
            continue;
        }
        const Interior inner = RouteInterior(p, c.hostDepth);
        std::vector<Rect> rects;
        Rect rect{ 0, 0, 0, 0 };
        if (inner.width > 0)
        {
            if (!Place(c, p, q.interior, &rect) || !(rect == Rect{ 0, 0, inner.width, inner.rows }) ||
                q.interiorUnits != BatchInteriorUnits(inner.width, inner.rows, p.ys, UnitPixels(p, c.hostDepth)))
            {
                Fail("step interior units or rectangle", c.index, static_cast<int>(i));
            }
            rects.push_back(rect);
            Strip strip[2];
            if (q.windows != InteriorStrips(p.width, p.rowCount, inner, strip))
            {
                Fail("step windows are not the strips", c.index, static_cast<int>(i));
            }
            for (int k = 0; k < q.windows && k < 2; ++k)
            {
                if (!Place(c, p, q.window[k], &rect) || !(rect == Rect{ strip[k].x0, strip[k].y0, strip[k].width, strip[k].rows }) ||
                    q.windowUnits[k] != EdgeUnits(p, strip[k].width, strip[k].rows))
                {
                    Fail("step window", c.index, static_cast<int>(i));
                }
                rects.push_back(rect);
            }
        }
        else
        {
            if (q.interior.width != 0 || q.interiorUnits != 0 || q.windows != 1 || !Place(c, p, q.window[0], &rect) ||
                !(rect == Rect{ 0, 0, p.width, p.rowCount }) || q.windowUnits[0] != EdgeUnits(p, p.width, p.rowCount))
            {
                Fail("step: an image without an interior is not one whole-image window", c.index, static_cast<int>(i));
            }
            rects.push_back(rect);
        }
        if (q.windows < 2 && q.windowUnits[1] != 0)
        {
            Fail("step: a missing window has units", c.index, static_cast<int>(i));
        }
        if (!CoveredOnce(rects, p.width, p.rowCount))
        {
            Fail("step: pixel not covered exactly once", c.index, static_cast<int>(i));
        }
    }
    return plans;
}

// The records of `plans` at the exclusive prefix sums of their units, as the plan kernel lays them out (interiors; windows,
// image i owning 2i and 2i + 1), and FindRecord against a linear walk for every unit: from the owner of the previous
// unit, from record 0 and from a random earlier record.  Returns the interior units.
inline int64_t CheckLayoutAndSearch(std::mt19937_64& rng, const std::vector<BatchImagePlan>& plans, int description)
{
    const size_t n = plans.size();
    std::vector<int64_t> interiorFirst(n), interiorUnits(n), windowFirst(2 * n), windowUnits(2 * n);
    int64_t interiorTotal = 0, windowTotal = 0;
    for (size_t i = 0; i < n; ++i)
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
        int owner = 0, record = 0;
        for (int64_t u = 0; u < total; ++u)
        {
            while (u >= first[owner] + units[owner])
            {
                ++owner;
            }
            record = FindRecord(first.data(), count, record, u);
            const int earlier = static_cast<int>(rng() % (owner + 1));
            if (record != owner || FindRecord(first.data(), count, 0, u) != owner || FindRecord(first.data(), count, earlier, u) != owner)
            {
                Fail("FindRecord", description, owner);
                return;
            }
        }
    };
    check(interiorFirst, interiorUnits, interiorTotal);
    check(windowFirst, windowUnits, windowTotal);
    return interiorTotal;
}

// The host-described plan of the accepted images: chunks of at most kBatchChunkImages images in increasing order, as many
// as the batched images need; interiors the route's, first units the running sums of the family's units; a second launch
// exactly when some image of the chunk has a strip; direct calls in increasing order and never batched; every pixel
// covered exactly once, and an image batched exactly when the route gives it an interior.
template <typename Params>
void CheckHostPlan(const Case<Params>& c, const std::vector<FakeImage<Params>>& images, int batch)
{
    std::vector<avifgpu_batch_image> records;
    std::vector<const Params*> own;
    for (const FakeImage<Params>& im : images)
    {
        if (!im.rejected)
        {
            records.push_back(im.record);
            own.push_back(&im.p);
        }
    }
    const int n = static_cast<int>(records.size());
    BatchPlan plan;
    PlanBatch(c.shared, c.hostDepth, c.planeMask, records, &plan);
    std::vector<std::vector<Rect>> rects(n);
    std::vector<int> route(n, 0); // 1: batched, 2: a direct call
    int last = -1, batched = 0;
    Rect rect{ 0, 0, 0, 0 };
    for (const BatchChunk& chunk : plan.chunks)
    {
        if (chunk.images < 1 || chunk.images > kBatchChunkImages)
        {
            Fail("chunk size", c.index, batch);
            return;
        }
        int64_t units = 0;
        bool strips = false;
        for (int j = 0; j < chunk.images; ++j)
        {
            const int i = chunk.imageIndex[j];
            if (i <= last || i >= n)
            {
                Fail("image order", c.index, batch);
                return;
            }
            last = i;
            route[i] = 1;
            ++batched;
            const Params& p = *own[i];
            const Interior inner = RouteInterior(p, c.hostDepth);
            if (!Place(c, p, chunk.interior[j], &rect) || !(rect == Rect{ 0, 0, inner.width, inner.rows }) || chunk.interior[j].firstUnit != units)
            {
                Fail("chunk interior", c.index, batch);
            }
            rects[i].push_back(rect);
            units += BatchInteriorUnits(inner.width, inner.rows, p.ys, UnitPixels(p, c.hostDepth));
            strips = strips || inner.width < p.width || inner.rows < p.rowCount;
        }
        if (units != chunk.interiorUnits)
        {
            Fail("chunk interior units", c.index, batch);
        }
        units = 0;
        for (int j = 0; j < chunk.windows; ++j)
        {
            const int i = chunk.windowImage[j];
            if (i < chunk.imageIndex[0] || i > last || route[i] != 1)
            {
                Fail("a window of an image outside its chunk", c.index, batch);
                return;
            }
            const BatchRecord& w = chunk.window[j];
            if (!Place(c, *own[i], w, &rect) || w.firstUnit != units)
            {
                Fail("chunk window units", c.index, batch);
            }
            rects[i].push_back(rect);
            units += EdgeUnits(*own[i], w.width, w.rowCount);
        }
        if (units != chunk.windowUnits)
        {
            Fail("chunk window units", c.index, batch);
        }
        if (BatchChunkLaunches(chunk) != (strips ? 2 : 1))
        {
            Fail("chunk launches", c.index, batch);
        }
    }
    if (static_cast<int>(plan.chunks.size()) != (batched + kBatchChunkImages - 1) / kBatchChunkImages)
    {
        Fail("chunk count", c.index, batch);
    }
    last = -1;
    for (const int32_t i : plan.fallback)
    {
        if (i <= last || i >= n || route[i] != 0)
        {
            Fail("direct calls out of order or batched", c.index, batch);
            return;
        }
        last = i;
        route[i] = 2;
        rects[i].push_back(Rect{ 0, 0, own[i]->width, own[i]->rowCount });
    }
    for (int i = 0; i < n; ++i)
    {
        const Params& p = *own[i];
        const bool empty = p.width == 0 || p.rowCount == 0;
        if (route[i] != (empty ? 0 : RouteInterior(p, c.hostDepth).width > 0 ? 1 : 2))
        {
            Fail("image routing", c.index, batch);
        }
        if (!CoveredOnce(rects[i], p.width, p.rowCount))
        {
            Fail("host plan: pixel not covered exactly once", c.index, batch);
        }
    }
}

struct Counts
{
    int descriptions = 0;
    long long images = 0, units = 0;
};

// One seeded batch of 1 to `maxImages` images of the description `d` through all three checks; the images, for the
// slice's own statements about them.
template <typename Desc, typename Params>
std::vector<FakeImage<Params>> CheckBatch(std::mt19937_64& rng, const Desc& d, const Case<Params>& c, int maxImages, int batch, Counts& counts)
{
    const std::vector<FakeImage<Params>> images = MakeBatch(rng, d, c, 1 + static_cast<int>(rng() % maxImages));
    const std::vector<BatchImagePlan> plans = CheckImageStep(c, images);
    counts.units += CheckLayoutAndSearch(rng, plans, c.index);
    CheckHostPlan(c, images, batch);
    counts.images += static_cast<long long>(images.size());
    return images;
}

// The first `bytes` of `object` copied so that they end where an inaccessible page begins: any read past them faults.
// nullptr when the pages cannot be mapped; they stay mapped until the process exits.
template <typename T>
T* EndingAtGuardPage(const T& object, size_t bytes)
{
    const long page = sysconf(_SC_PAGESIZE);
    void* pages = mmap(nullptr, 2 * page, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
    if (pages == MAP_FAILED || mprotect(static_cast<uint8_t*>(pages) + page, page, PROT_NONE) != 0)
    {
        return nullptr;
    }
    uint8_t* at = static_cast<uint8_t*>(pages) + page - bytes;
    std::memcpy(at, &object, bytes);
    return reinterpret_cast<T*>(at);
}

} // namespace avifgpu

#endif
