// tests/native/light_batch_plan_check.cpp -- the planning of the light-level batches (avifgpu_encode_batch_device_light_level,
// avifgpu_encode_batch_indirect_light_level) on the CPU: EncodeLightBatchFamilyOf, the per-image step with its unit width
// (PlanBatchEncodeImage, kLightBatchUnitPixels) and PlanEncodeLightBatch.  Every float-host PQ description runs seeded
// batches through plan_harness.h's three checks; on top, each restated independently of the library:
//   - which descriptions the light-level family takes, and which family;
//   - the unit width (128 pixels of a row, or of a 4:2:0 row pair);
//   - every interior against EncodeLightF32BatchKernel's loads and stores: 16-byte rows, 8-byte luma and alpha stores,
//     4- or 8-byte planar chroma stores, twice that for interleaved chroma; width a multiple of 4, rows of 1 << ys;
//   - that a record's image follows from its position: interior i and windows 2i, 2i + 1 of the step are image i's, and a
//     host chunk's imageIndex / windowImage name the image whose buffers the record points into;
//   - that a chunk's kernel parameters fit the 32764-byte limit.
// Prints "light descriptions=N images=K units=U tuned=T"; exit code 1 on any failure.
#include "plan_harness.h"

#include <cstdio>
#include <random>
#include <vector>

namespace avifgpu
{

// The description block of a light-level batch: plan_harness.h's checks then take the light-level family and unit.
struct LightParams : EncodeParams
{
};

inline LightParams Window(const LightParams& p, int hostDepth, int x0, int y0, int width, int rows)
{
    LightParams w;
    static_cast<EncodeParams&>(w) = EncodeWindow(p, hostDepth, x0, y0, width, rows);
    return w;
}
inline Interior RouteInterior(const LightParams& p, int hostDepth) { return EncodeBlockInterior(EncodeLightBatchFamilyOf(p, hostDepth), p, hostDepth); }
inline BatchImagePlan PlanImage(const LightParams& shared, int hostDepth, int planeMask, const avifgpu_batch_image& image)
{
    return PlanBatchEncodeImage(shared, hostDepth, EncodeLightBatchFamilyOf(shared, hostDepth), planeMask, image, kLightBatchUnitPixels);
}
inline void PlanBatch(const LightParams& shared, int, int planeMask, const std::vector<avifgpu_batch_image>& images, BatchPlan* plan)
{
    PlanEncodeLightBatch(shared, planeMask, images.data(), static_cast<int32_t>(images.size()), plan);
}
inline int UnitPixels(const LightParams&, int) { return kLightBatchUnitPixels; }

} // namespace avifgpu

using namespace avifgpu;

namespace
{

// The light-level chunks as kernels_batch.cu lays them out: the description, the count, the unit total, the records, their
// images and the sink.  The interior chunk carries the float kernels' parameters, a subset of EncodeParams' fields.
static_assert(kLightBatchUnitPixels == 128, "a unit is the single-image float kernels' 128-pixel tile");
static_assert(sizeof(EncodeParams) + 16 + 2 * kBatchChunkImages * (sizeof(BatchRecord) + sizeof(int32_t)) + sizeof(LightSink) <= 32764,
              "a light-level edge chunk fits one kernel parameter block");

// A table the size of the real ones (12-bit PQ: ~67 KB) or one too big for the batched kernel's shared memory.
CurveTableView FakeTable(uint32_t imageBytes)
{
    static const uint32_t words[4] = {};
    static const uint2 octaves[1] = {};
    CurveTableView t{};
    t.octaves = octaves;
    t.buckets = words;
    t.bandBits = words;
    t.compact = words;
    t.firstBits = words;
    t.compactImageBytes = imageBytes;
    return t;
}

// Which family the light-level batches take, restated: float planar RGB (no alpha) or RGBA (with alpha) into 10/12-bit
// planar YCbCr, PQ, no row matrix, through a compact table that fits both the single-image light route
// (FlatFixedBytes for RGB, RgbaFixedBytes for RGBA) and the batched kernel (LightBatchFixedBytes).
EncodeFamily Expected(const avifgpu_encode_desc& d, bool rowMatrix, uint32_t tableBytes)
{
    const bool rgb = d.host_channels == 3 && d.alpha_state == AVIFGPU_ALPHA_NONE;
    const bool rgba = d.host_channels == 4 && d.alpha_state != AVIFGPU_ALPHA_NONE;
    const size_t fixed = rgb ? FlatFixedBytes() : RgbaFixedBytes();
    const bool fits = tableBytes > 0 && fixed + tableBytes <= 227 * 1024 && LightBatchFixedBytes() + tableBytes <= 227 * 1024;
    if (d.host_depth != 32 || d.transfer != AVIFGPU_TRANSFER_PQ || d.layout != AVIFGPU_LAYOUT_PLANAR_YCBCR || d.image_bit_depth < 10 || rowMatrix ||
        !(rgb || rgba) || !fits)
    {
        return EncodeFamily::Generic;
    }
    return rgb ? EncodeFamily::RgbF32Flat : EncodeFamily::RgbaF32Flat;
}

// The interior against the kernel's accesses, restated from EncodeLightF32BatchKernel.
bool InteriorFitsTheKernel(const EncodeParams& p, Interior inner)
{
    const auto aligned = [](const void* q, int64_t stride, int a) { return reinterpret_cast<uintptr_t>(q) % a == 0 && stride % a == 0; };
    const int chromaStore = p.xs ? 4 : 8; // two or four 16-bit codes
    const bool chroma = SourceInterleaved(p.destLayout) ? aligned(p.plane[1], p.planeStride[1], 2 * chromaStore)
                                                        : aligned(p.plane[1], p.planeStride[1], chromaStore) && aligned(p.plane[2], p.planeStride[2], chromaStore);
    return inner.width % 4 == 0 && inner.rows % (1 << p.ys) == 0 && inner.width <= p.width && inner.rows <= p.rowCount && aligned(p.rows, p.rowStride, 16) &&
           aligned(p.plane[0], p.planeStride[0], 8) && chroma && (p.channels != 4 || aligned(p.plane[3], p.planeStride[3], 8));
}

// The image a record points into: MakeBatch puts image i's buffers at (i + 1) << 36.
int ImageOfPointer(const void* rows) { return static_cast<int>((reinterpret_cast<uintptr_t>(rows) >> 36) - 1); }

} // namespace

int main()
{
    std::mt19937_64 rng(4321);
    Counts n;
    int batch = 0, tuned = 0;
    const uint32_t tables[] = { 0u, 68u * 1024u, 180u * 1024u }; // none, a 12-bit-sized compact table, one too big
    for (int channels = 1; channels <= 4; ++channels)
        for (int alpha : { 0, 1, 2 })
            for (int depth : { 10, 12 })
                for (int layout : { 0, 1 })
                    for (int chroma : { 1, 2, 3 })
                        for (int dest = 0; dest < 4; ++dest)
                            for (int transfer : { AVIFGPU_TRANSFER_PQ, AVIFGPU_TRANSFER_SMPTE428 })
                                for (uint32_t tableBytes : tables)
                                    for (int rowMatrix : { 0, 1 })
                                    {
                                        avifgpu_encode_desc d{};
                                        d.struct_size = sizeof(d);
                                        d.width = 16;
                                        d.height = 16;
                                        d.host_depth = 32;
                                        d.host_channels = channels;
                                        d.alpha_state = alpha;
                                        d.image_bit_depth = depth;
                                        d.transfer = transfer;
                                        d.pq_peak_nits = 1000;
                                        d.layout = layout;
                                        d.chroma = layout == 1 ? chroma : 3;
                                        d.nclx = avifgpu_nclx{ 1, 9, 16, 9, 1 };
                                        d.dest_layout = layout == 1 ? dest : 0;
                                        d.row_matrix_enabled = rowMatrix;
                                        d.row_matrix[0] = d.row_matrix[4] = d.row_matrix[8] = 1.0f;
                                        if ((layout == 0 && (chroma != 3 || dest != 0)) || ValidateEncodeDesc(&d, nullptr) != AVIFGPU_OK)
                                        {
                                            continue;
                                        }
                                        ++n.descriptions;
                                        static CurveTableView table;
                                        table = FakeTable(tableBytes);
                                        LightParams shared;
                                        FillEncodeParams(d, &shared);
                                        shared.curveTable = tableBytes ? &table : nullptr;
                                        const EncodeFamily family = EncodeLightBatchFamilyOf(shared, 32);
                                        if (family != Expected(d, rowMatrix != 0, tableBytes))
                                        {
                                            Fail("light-level family", n.descriptions, -1);
                                        }
                                        tuned += family != EncodeFamily::Generic;
                                        const Case<LightParams> c = CaseOf(d, shared, n.descriptions);
                                        for (int trial = 0; trial < 2; ++trial)
                                        {
                                            const std::vector<FakeImage<LightParams>> images = CheckBatch(rng, d, c, trial == 1 ? 200 : 20, batch++, n);
                                            std::vector<avifgpu_batch_image> accepted;
                                            for (size_t i = 0; i < images.size(); ++i)
                                            {
                                                const FakeImage<LightParams>& im = images[i];
                                                const BatchImagePlan q = PlanImage(shared, 32, c.planeMask, im.record);
                                                if (!im.rejected)
                                                {
                                                    accepted.push_back(im.record);
                                                }
                                                if (q.interior.width > 0 &&
                                                    (!InteriorFitsTheKernel(im.p, Interior{ q.interior.width, q.interior.rowCount }) ||
                                                     q.interiorUnits != static_cast<int64_t>((q.interior.width + 127) / 128) * (q.interior.rowCount >> im.p.ys) ||
                                                     ImageOfPointer(q.interior.rows) != static_cast<int>(i)))
                                                {
                                                    Fail("interior against the kernel, its units or its image", n.descriptions, static_cast<int>(i));
                                                }
                                                for (int k = 0; k < q.windows; ++k)
                                                {
                                                    if (ImageOfPointer(q.window[k].rows) != static_cast<int>(i))
                                                    {
                                                        Fail("window of another image", n.descriptions, static_cast<int>(i));
                                                    }
                                                }
                                            }
                                            BatchPlan plan;
                                            PlanEncodeLightBatch(shared, c.planeMask, accepted.data(), static_cast<int32_t>(accepted.size()), &plan);
                                            for (const BatchChunk& chunk : plan.chunks)
                                            {
                                                for (int j = 0; j < chunk.images; ++j)
                                                {
                                                    if (ImageOfPointer(chunk.interior[j].rows) != ImageOfPointer(accepted[chunk.imageIndex[j]].rows))
                                                    {
                                                        Fail("chunk interior's image", n.descriptions, batch);
                                                    }
                                                }
                                                for (int j = 0; j < chunk.windows; ++j)
                                                {
                                                    if (ImageOfPointer(chunk.window[j].rows) != ImageOfPointer(accepted[chunk.windowImage[j]].rows))
                                                    {
                                                        Fail("chunk window's image", n.descriptions, batch);
                                                    }
                                                }
                                            }
                                        }
                                    }
    std::printf("light descriptions=%d images=%lld units=%lld tuned=%d\n", n.descriptions, n.images, n.units, tuned);
    return g_failures == 0 ? 0 : 1;
}
