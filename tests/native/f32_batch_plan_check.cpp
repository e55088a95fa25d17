// tests/native/f32_batch_plan_check.cpp -- host-side check of the float-host decode planning (csrc/batch_plan.h,
// csrc/host_params.cpp): PlanDecodeBatch behind avifgpu_decode_batch_device, and the per-image step PlanBatchDecodeImage
// that the plan kernel of avifgpu_decode_batch_indirect runs.  For every valid YCbCr description into 32-bit hosts (bit
// depths 8/10/12/16, alpha none / straight / premultiplied, 4:4:4 / 4:2:2 / 4:2:0, PQ, HLG with and without the OOTF,
// SMPTE 428, the context's verified divisions off and on) and seeded random batches of 1 to 300 images of mixed sizes --
// widths below 4, one-row images, some with misaligned rows or Y planes, some with unequal Cb / Cr strides -- on fake
// padded planes:
//   host plans     every pixel of every image is covered exactly once by an interior, a window or a direct call; an
//                  image is batched exactly when DecodeBlockInterior of DecodeBatchFamilyOf takes it, with that interior; chunks keep image
//                  order and hold at most kBatchChunkImages images; first units are running sums of 128-pixel units; a
//                  chunk has a second launch exactly when one of its images has a strip outside its interior;
//   per-image step every pixel covered exactly once by the interior and windows; every record's planes where DecodeWindow
//                  puts them; interior units counted with the 128-pixel unit, window units as BatchEdgeUnits; FindRecord
//                  over the concatenated interior units finds the record that owns each unit.
// Prints "f32 descriptions=N images=K units=U"; exit code 1 on any failure.
#include "batch_plan.h"
#include "host_params.h"

#include <cstdio>
#include <random>
#include <vector>

using namespace avifgpu;

namespace
{

long long g_failures = 0;

void Fail(const char* what, int description, int batch)
{
    if (++g_failures <= 20)
    {
        std::printf("FAIL %s: description %d, batch %d\n", what, description, batch);
    }
}

avifgpu_batch_image BatchImageOf(const DecodeParams& p)
{
    avifgpu_batch_image image{};
    image.width = p.width;
    image.height = p.rowCount;
    image.rows = p.rows;
    image.row_stride_bytes = p.rowStride;
    for (int k = 0; k < 4; ++k)
    {
        image.planes.data[k] = const_cast<void*>(p.plane[k]);
        image.planes.stride[k] = p.planeStride[k];
    }
    return image;
}

// The window of `p` a record's rows pointer starts, or false when it is not inside the image.
bool Origin(const DecodeParams& p, const BatchRecord& r, int colBytes, int& x0, int& y0)
{
    const int64_t offset = static_cast<int64_t>(reinterpret_cast<uintptr_t>(r.rows) - reinterpret_cast<uintptr_t>(p.rows));
    if (offset < 0)
    {
        return false;
    }
    y0 = static_cast<int>(offset / p.rowStride);
    x0 = static_cast<int>(offset % p.rowStride) / colBytes;
    return r.width > 0 && r.rowCount > 0 && x0 + r.width <= p.width && y0 + r.rowCount <= p.rowCount && (y0 & p.ys) == 0;
}

void Cover(std::vector<int>& count, const DecodeParams& p, const BatchRecord& r, int colBytes, int description, int batch)
{
    int x0, y0;
    if (!Origin(p, r, colBytes, x0, y0))
    {
        Fail("record outside its image or off a row pair", description, batch);
        return;
    }
    const DecodeParams w = DecodeWindow(p, x0, y0, r.width, r.rowCount);
    for (int k = 0; k < 4; ++k)
    {
        if (r.plane[k] != w.plane[k] || r.planeStride[k] != p.planeStride[k])
        {
            Fail("record plane not where DecodeWindow puts it", description, batch);
        }
    }
    for (int y = y0; y < y0 + r.rowCount; ++y)
    {
        for (int x = x0; x < x0 + r.width; ++x)
        {
            ++count[static_cast<size_t>(y) * p.width + x];
        }
    }
}

bool CoveredOnce(const std::vector<int>& count)
{
    for (int v : count)
    {
        if (v != 1)
        {
            return false;
        }
    }
    return true;
}

} // namespace

int main()
{
    std::mt19937_64 rng(20261016);
    int descriptions = 0;
    long long images = 0, units = 0;
    struct Curve
    {
        int transferCharacteristics, ootf;
    };
    for (int bitDepth : { 8, 10, 12, 16 })
        for (int alpha : { 0, 1, 2 })
            for (int chroma : { 1, 2, 3 })
                for (Curve curve : { Curve{ 16, 0 }, Curve{ 18, 1 }, Curve{ 18, 0 }, Curve{ 17, 0 } })
                    for (int verified : { 0, 1 })
                    {
                        avifgpu_decode_desc d{};
                        d.struct_size = sizeof(d);
                        d.colorspace = AVIFGPU_COLORSPACE_YCBCR;
                        d.chroma = chroma;
                        d.bit_depth = bitDepth;
                        d.alpha_state = alpha;
                        d.host_depth = 32;
                        d.nclx = avifgpu_nclx{ 1, 9, curve.transferCharacteristics, descriptions % 2 ? 9 : 1, (descriptions / 2) % 2 };
                        d.hlg_apply_ootf = curve.ootf;
                        d.hlg_display_gamma = 1.2f;
                        d.hlg_peak_nits = 1000;
                        d.pq_peak_nits = 1000;
                        int32_t transfer = 0;
                        DecodeParams probe{};
                        if (ValidateDecodeDesc(&d, &transfer, nullptr) != AVIFGPU_OK || !FillDecodeParams(d, transfer, &probe, nullptr))
                        {
                            continue;
                        }
                        probe.verifiedHlgDivisions = verified;
                        probe.verifiedGreenDivision = verified;
                        probe.verifiedPqRatio = verified;
                        const DecodeFamily family = DecodeBatchFamilyOf(probe);
                        const bool tuned = family != DecodeFamily::Generic;
                        if (tuned != (DecodeFamilyOf(probe) == DecodeFamily::YccF32))
                        {
                            Fail("DecodeBatchFamilyOf is not the float family for 32-bit hosts", descriptions, -1);
                        }
                        const bool expectTuned = bitDepth >= 10 && bitDepth <= 12 && alpha != 2 && (curve.transferCharacteristics != 18 || verified);
                        if (tuned != expectTuned)
                        {
                            Fail("description routing", descriptions, -1);
                        }
                        ++descriptions;
                        int planeMask = 0;
                        for (int k = 0; k < 4; ++k)
                        {
                            planeMask |= DecodePlaneGeometry(d, k).present ? 1 << k : 0;
                        }
                        const int colBytes = DecodeHostColBytes(d);
                        for (int trial = 0; trial < 3; ++trial)
                        {
                            const int n = 1 + static_cast<int>(rng() % (trial == 2 ? 300 : 24));
                            std::vector<DecodeParams> params(n);
                            for (int i = 0; i < n; ++i)
                            {
                                avifgpu_decode_desc di = d;
                                const int shape = static_cast<int>(rng() % 8);
                                di.width = shape == 0 ? 1 + static_cast<int>(rng() % 4) : 1 + static_cast<int>(rng() % 300);
                                di.height = shape == 1 ? 1 : 1 + static_cast<int>(rng() % 9);
                                DecodeParams& p = params[i];
                                FillDecodeParams(di, transfer, &p, nullptr);
                                p.verifiedHlgDivisions = verified;
                                p.verifiedGreenDivision = verified;
                                p.verifiedPqRatio = verified;
                                const uintptr_t base = static_cast<uintptr_t>(i + 1) << 36;
                                p.rows = reinterpret_cast<void*>(base + (shape == 2 ? 4 : 0));
                                p.rowStride = (static_cast<int64_t>(di.width) * colBytes + 63) / 64 * 64 + 64;
                                p.rowCount = di.height;
                                for (int k = 0; k < 4; ++k)
                                {
                                    const PlaneGeometry g = DecodePlaneGeometry(di, k);
                                    if (g.present)
                                    {
                                        p.plane[k] = reinterpret_cast<const void*>(base + (static_cast<uintptr_t>(k + 1) << 30) + (shape == 3 && k == 0 ? 2 : 0));
                                        p.planeStride[k] = (static_cast<int64_t>(g.widthSamples) * g.bytesPerSample + 63) / 64 * 64 + 128;
                                    }
                                }
                                if (shape == 4 && p.plane[2] != nullptr)
                                {
                                    p.planeStride[2] += 64;
                                }
                            }
                            std::vector<avifgpu_batch_image> batch(n);
                            for (int i = 0; i < n; ++i)
                            {
                                batch[i] = BatchImageOf(params[i]);
                            }
                            images += n;

                            // ---- the host plan ----
                            BatchPlan plan;
                            PlanDecodeBatch(probe, planeMask, batch.data(), n, &plan);
                            std::vector<std::vector<int>> count(n);
                            std::vector<int> batched(n, 0);
                            for (int i = 0; i < n; ++i)
                            {
                                count[i].assign(static_cast<size_t>(params[i].width) * params[i].rowCount, 0);
                            }
                            int last = -1;
                            for (const BatchChunk& c : plan.chunks)
                            {
                                if (c.images < 1 || c.images > kBatchChunkImages)
                                {
                                    Fail("chunk size", descriptions, trial);
                                }
                                bool edges = false;
                                int64_t first = 0;
                                for (int j = 0; j < c.images; ++j)
                                {
                                    const int i = c.imageIndex[j];
                                    if (i <= last)
                                    {
                                        Fail("image order", descriptions, trial);
                                    }
                                    last = i;
                                    batched[i] = 1;
                                    const Interior inner = DecodeBlockInterior(DecodeBatchFamilyOf(params[i]), params[i]);
                                    if (c.interior[j].width != inner.width || c.interior[j].rowCount != inner.rows || c.interior[j].firstUnit != first)
                                    {
                                        Fail("chunk interior", descriptions, trial);
                                    }
                                    first += BatchInteriorUnits(inner.width, inner.rows, params[i].ys, 128);
                                    edges = edges || inner.width < params[i].width || inner.rows < params[i].rowCount;
                                    Cover(count[i], params[i], c.interior[j], colBytes, descriptions, trial);
                                }
                                if (first != c.interiorUnits)
                                {
                                    Fail("chunk unit total", descriptions, trial);
                                }
                                for (int j = 0; j < c.windows; ++j)
                                {
                                    Cover(count[c.windowImage[j]], params[c.windowImage[j]], c.window[j], colBytes, descriptions, trial);
                                }
                                if (BatchChunkLaunches(c) != (edges ? 2 : 1))
                                {
                                    Fail("chunk launches", descriptions, trial);
                                }
                            }
                            for (const int32_t i : plan.fallback)
                            {
                                batched[i] = 2;
                                for (int& v : count[i])
                                {
                                    ++v;
                                }
                            }
                            for (int i = 0; i < n; ++i)
                            {
                                if ((DecodeBlockInterior(DecodeBatchFamilyOf(params[i]), params[i]).width > 0) != (batched[i] == 1))
                                {
                                    Fail("image routing", descriptions, trial);
                                }
                                if (!CoveredOnce(count[i]))
                                {
                                    Fail("host plan: pixel not covered exactly once", descriptions, trial);
                                }
                            }

                            // ---- the per-image step, as the plan kernel runs it ----
                            std::vector<int64_t> interiorFirst(n);
                            std::vector<int64_t> interiorUnits(n);
                            int64_t total = 0;
                            for (int i = 0; i < n; ++i)
                            {
                                const BatchImagePlan step = PlanBatchDecodeImage(probe, family, planeMask, batch[i]);
                                std::vector<int> covered(static_cast<size_t>(params[i].width) * params[i].rowCount, 0);
                                const Interior inner = DecodeBlockInterior(DecodeBatchFamilyOf(params[i]), params[i]);
                                if (step.status != AVIFGPU_OK || step.interior.width != inner.width || (inner.width > 0 && step.interior.rowCount != inner.rows))
                                {
                                    Fail("step interior", descriptions, trial);
                                }
                                if (step.interior.width > 0)
                                {
                                    Cover(covered, params[i], step.interior, colBytes, descriptions, trial);
                                    const int64_t expected = static_cast<int64_t>((inner.width + 127) / 128) * (inner.rows >> params[i].ys);
                                    if (step.interiorUnits != expected)
                                    {
                                        Fail("step interior units", descriptions, trial);
                                    }
                                }
                                for (int k = 0; k < step.windows; ++k)
                                {
                                    Cover(covered, params[i], step.window[k], colBytes, descriptions, trial);
                                    if (step.windowUnits[k] != BatchEdgeUnits(step.window[k].width, step.window[k].rowCount, 0, 0))
                                    {
                                        Fail("step window units", descriptions, trial);
                                    }
                                }
                                if (!CoveredOnce(covered))
                                {
                                    Fail("step: pixel not covered exactly once", descriptions, trial);
                                }
                                interiorFirst[i] = total;
                                interiorUnits[i] = step.interiorUnits;
                                total += step.interiorUnits;
                            }
                            // every unit's owner, by a forward walk from unit 0 with the owner of the previous unit
                            int record = 0;
                            for (int64_t u = 0; u < total; ++u)
                            {
                                record = FindRecord(interiorFirst.data(), n, record, u);
                                if (u < interiorFirst[record] || u >= interiorFirst[record] + interiorUnits[record])
                                {
                                    Fail("FindRecord", descriptions, trial);
                                    break;
                                }
                                // and from the first record, as a worker's first unit is searched
                                const int fresh = FindRecord(interiorFirst.data(), n, 0, u);
                                if (fresh != record)
                                {
                                    Fail("FindRecord from record 0", descriptions, trial);
                                    break;
                                }
                            }
                            units += total;
                        }
                    }
    std::printf("f32 descriptions=%d images=%lld units=%lld\n", descriptions, images, units);
    return g_failures == 0 ? 0 : 1;
}
