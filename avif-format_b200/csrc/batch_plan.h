// batch_plan.h -- the per-image planning step of both batch APIs, and the workspace of the device-described one.
//
// Host-described batches (avifgpu_encode_batch_device / avifgpu_decode_batch_device): PlanEncodeBatch / PlanDecodeBatch
// run the per-image step below on the host and pack its records into chunks that travel in a kernel parameter.
// Device-described batches (avifgpu_encode_batch_indirect / avifgpu_decode_batch_indirect): the image records, their
// count and the workspace live in device memory and are read when the work runs, so one call (or one captured graph of
// it) converts whatever the buffers hold at that moment.  A call is three launches:
//   1. the plan kernel (one CTA) routes every image with the same per-image step and writes, per image, one interior
//      record and up to two window records, the exclusive prefix sums of their units and the two totals into the workspace;
//   2. the interior kernel walks the interior units with the tuned integer (float, for 32-bit decode hosts; planar-RGB,
//      for planar-RGB decodes) kernel's per-unit code;
//   3. the edge kernel walks the window units with the generic kernel's per-site / per-pixel code.
// Both run the batched kernels of kernels_batch.cu.  Plain C++ (AVIFGPU_HD): host_params.cpp and the checks under
// tests/native compile the per-image step with the host compiler.
#ifndef AVIF_BATCH_PLAN_H
#define AVIF_BATCH_PLAN_H

#include <stddef.h>
#include <stdint.h>

#include "../../include/avifgpu.h"
#include "kernel_params.h"

namespace avifgpu
{

constexpr int kIndirectMaxImages = 4096;

// The workspace of a call of at most maxCount images: a header, then the first units of the interiors (maxCount) and
// of the windows (2 * maxCount, image i owning 2i and 2i + 1), then the records in the same order.  A record that owns
// no unit (an empty or rejected image, a missing strip) has the first unit of the next, so the last record whose first
// unit is at most u owns unit u.
struct IndirectHeader
{
    int64_t interiorUnits;
    int64_t windowUnits;
    int32_t count; // images planned: *device_count, or 0 when it was out of range
    int32_t reserved;
};

struct IndirectLayout
{
    size_t interiorFirst, windowFirst, interior, window, bytes; // byte offsets, and the total
};

AVIFGPU_HD inline size_t IndirectAlign(size_t bytes) { return (bytes + 255) / 256 * 256; }

AVIFGPU_HD inline IndirectLayout IndirectWorkspaceLayout(int maxCount)
{
    const size_t n = static_cast<size_t>(maxCount);
    IndirectLayout l;
    l.interiorFirst = IndirectAlign(sizeof(IndirectHeader));
    l.windowFirst = l.interiorFirst + IndirectAlign(sizeof(int64_t) * n);
    l.interior = l.windowFirst + IndirectAlign(sizeof(int64_t) * 2 * n);
    l.window = l.interior + IndirectAlign(sizeof(BatchRecord) * n);
    l.bytes = l.window + IndirectAlign(sizeof(BatchRecord) * 2 * n);
    return l;
}

// The last of `count` records whose first unit is at most `unit` -- the record that owns it -- searching from `record`,
// whose first unit is at most `unit` already (a worker passes the record of its previous unit: units only increase).
AVIFGPU_HD inline int FindRecord(const int64_t* first, int count, int record, long long unit)
{
    if (record + 1 >= count || unit < first[record + 1])
    {
        return record;
    }
    int lo = record + 1, hi = count - 1;
    while (lo < hi)
    {
        const int mid = (lo + hi + 1) >> 1;
        if (first[mid] <= unit)
        {
            lo = mid;
        }
        else
        {
            hi = mid - 1;
        }
    }
    return lo;
}

// One image's part of the plan: its status, its interior record (width 0: none) and its windows, with their units.
struct BatchImagePlan
{
    int32_t status;
    int32_t windows;
    BatchRecord interior;
    int64_t interiorUnits;
    BatchRecord window[2];
    int64_t windowUnits[2];
};

// Puts the record's size, rows and the planes of `planeMask` (bit k: the description has plane k) into `p`, with the
// host-described calls' checks: AVIFGPU_ERR_BAD_PARAM for a negative size, or for a non-empty image with NULL rows or a
// NULL plane the description has.
template <typename Params>
AVIFGPU_HD inline int AdoptBatchImage(Params& p, int planeMask, const avifgpu_batch_image& image)
{
    if (image.width < 0 || image.height < 0)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    p.width = image.width;
    p.rowCount = image.height;
    if (image.width == 0 || image.height == 0)
    {
        return AVIFGPU_OK;
    }
    if (image.rows == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    p.rows = image.rows;
    p.rowStride = image.row_stride_bytes;
    for (int k = 0; k < 4; ++k)
    {
        p.plane[k] = nullptr;
        p.planeStride[k] = 0;
        if ((planeMask >> k) & 1)
        {
            if (image.planes.data[k] == nullptr)
            {
                return AVIFGPU_ERR_BAD_PARAM;
            }
            p.plane[k] = image.planes.data[k];
            p.planeStride[k] = image.planes.stride[k];
        }
    }
    return AVIFGPU_OK;
}

// The per-image step of both plans.  `shared` is the description's block (FillEncodeParams), `family` the family its
// interiors take (EncodeBatchFamilyOf: RgbInt or Generic).  An image the tuned kernel takes in a direct call gets its
// interior and the strips CompleteEncode would hand to the generic kernel; any other non-empty image becomes one
// whole-image window, which is what the generic kernel converts in a direct call (the device-described batch runs that
// window; the host-described one makes the direct call).  Interior units are `unitPixels` wide: kBatchUnitPixels for
// EncodeBatchFamilyOf's family, kLightBatchUnitPixels for EncodeLightBatchFamilyOf's.
AVIFGPU_HD inline BatchImagePlan PlanBatchEncodeImage(const EncodeParams& shared, int hostDepth, EncodeFamily family, int planeMask,
                                                       const avifgpu_batch_image& image, int unitPixels)
{
    BatchImagePlan plan{};
    EncodeParams p = shared;
    plan.status = AdoptBatchImage(p, planeMask, image);
    if (plan.status != AVIFGPU_OK || p.width == 0 || p.rowCount == 0)
    {
        return plan;
    }
    const Interior inner = EncodeBlockInterior(family, p, hostDepth);
    if (inner.width == 0)
    {
        plan.window[0] = RecordOf(EncodeWindow(p, hostDepth, 0, 0, p.width, p.rowCount));
        plan.windowUnits[0] = BatchEdgeUnits(p.width, p.rowCount, p.xs, p.ys);
        plan.windows = 1;
        return plan;
    }
    plan.interior = RecordOf(EncodeWindow(p, hostDepth, 0, 0, inner.width, inner.rows));
    plan.interiorUnits = BatchInteriorUnits(inner.width, inner.rows, p.ys, unitPixels);
    Strip strip[2];
    plan.windows = InteriorStrips(p.width, p.rowCount, inner, strip);
    for (int k = 0; k < plan.windows; ++k)
    {
        plan.window[k] = RecordOf(EncodeWindow(p, hostDepth, strip[k].x0, strip[k].y0, strip[k].width, strip[k].rows));
        plan.windowUnits[k] = BatchEdgeUnits(strip[k].width, strip[k].rows, p.xs, p.ys);
    }
    return plan;
}
AVIFGPU_HD inline BatchImagePlan PlanBatchEncodeImage(const EncodeParams& shared, int hostDepth, EncodeFamily family, int planeMask,
                                                       const avifgpu_batch_image& image)
{
    return PlanBatchEncodeImage(shared, hostDepth, family, planeMask, image, kBatchUnitPixels);
}

// The same for decodes (`family` = DecodeBatchFamilyOf; interior units of DecodeBatchUnitPixels); edge units are runs of
// pixels of one row.
AVIFGPU_HD inline BatchImagePlan PlanBatchDecodeImage(const DecodeParams& shared, DecodeFamily family, int planeMask, const avifgpu_batch_image& image)
{
    BatchImagePlan plan{};
    DecodeParams p = shared;
    plan.status = AdoptBatchImage(p, planeMask, image);
    if (plan.status != AVIFGPU_OK || p.width == 0 || p.rowCount == 0)
    {
        return plan;
    }
    p.yPhase = 0;
    const Interior inner = DecodeBlockInterior(family, p);
    if (inner.width == 0)
    {
        plan.window[0] = RecordOf(DecodeWindow(p, 0, 0, p.width, p.rowCount));
        plan.windowUnits[0] = BatchEdgeUnits(p.width, p.rowCount, 0, 0);
        plan.windows = 1;
        return plan;
    }
    plan.interior = RecordOf(DecodeWindow(p, 0, 0, inner.width, inner.rows));
    plan.interiorUnits = BatchInteriorUnits(inner.width, inner.rows, p.ys, DecodeBatchUnitPixels(family));
    Strip strip[2];
    plan.windows = InteriorStrips(p.width, p.rowCount, inner, strip);
    for (int k = 0; k < plan.windows; ++k)
    {
        plan.window[k] = RecordOf(DecodeWindow(p, strip[k].x0, strip[k].y0, strip[k].width, strip[k].rows));
        plan.windowUnits[k] = BatchEdgeUnits(strip[k].width, strip[k].rows, 0, 0);
    }
    return plan;
}

// Splits a host-described batch into chunks of the images whose plan has an interior, in order, and direct calls for the
// other non-empty images; empty images are skipped.  `shared` is the description's block with the context's first-use
// state, `planeMask` its planes (bit k: plane k); every image has passed AdoptBatchImage's checks.
void PlanEncodeBatch(const EncodeParams& shared, int hostDepth, int planeMask, const avifgpu_batch_image* images, int32_t count, BatchPlan* plan);
void PlanDecodeBatch(const DecodeParams& shared, int planeMask, const avifgpu_batch_image* images, int32_t count, BatchPlan* plan);
// The same for a light-level batch of float images: EncodeLightBatchFamilyOf's family, kLightBatchUnitPixels units.
void PlanEncodeLightBatch(const EncodeParams& shared, int planeMask, const avifgpu_batch_image* images, int32_t count, BatchPlan* plan);

// The launchers (kernels_batch.cu): the plan, interior and edge kernels of one call on `stream`.  `shared` is the
// description's block with the context's first-use state; `family` the family its interiors take (EncodeBatchFamilyOf /
// DecodeBatchFamilyOf).  Return 3 (the launches) or a negative status.
int LaunchEncodeIndirect(const EncodeParams& shared, int hostDepth, EncodeFamily family, int planeMask, const avifgpu_batch_image* images,
                         const int32_t* count, int maxCount, void* workspace, int32_t* status, void* stream);
// The light-level one (float hosts, EncodeLightBatchFamilyOf): image i adds its content light level into light.acc[i].
int LaunchEncodeLightIndirect(const EncodeParams& shared, int planeMask, const avifgpu_batch_image* images, const int32_t* count, int maxCount,
                              void* workspace, int32_t* status, const LightSink& light, void* stream);
int LaunchDecodeIndirect(const DecodeParams& shared, DecodeFamily family, int planeMask, const avifgpu_batch_image* images, const int32_t* count,
                         int maxCount, void* workspace, int32_t* status, void* stream);

} // namespace avifgpu

#endif
