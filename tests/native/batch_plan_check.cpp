// tests/native/batch_plan_check.cpp -- host-side check of PlanEncodeBatch (csrc/host_params.cpp, csrc/batch_plan.h), the
// planner behind avifgpu_encode_batch_device.  For every valid encode description and seeded random batches of 1 to 300 images of mixed
// sizes (1 x 1, widths below 8, odd widths and heights) on fake planes, some of them misaligned:
//   - every pixel and every chroma site of every image is covered exactly once, by an interior, an edge window or a
//     direct call, read back from the records' rows and plane pointers;
//   - an image is batched exactly when EncodeBlockInterior of EncodeBatchFamilyOf takes it, and its interior is that rectangle;
//   - chunks hold at most kBatchChunkImages images in increasing order, records' first units are the running sums of
//     their unit counts, and a chunk has a second launch exactly when one of its images has a strip outside its interior;
//   - a chunk's kernel parameters fit the 32764-byte limit.
// Decode batches (PlanDecodeBatch) get the pixel coverage, routing and launch checks too.
// Prints "encode descriptions=N batches=M images=K" and "decode descriptions=N images=K"; exit code 1 on any failure.
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

struct FakeImage
{
    EncodeParams p;
    uintptr_t rowsBase;
    uintptr_t planeBase[4];
    int colBytes;
    PlaneGeometry g[4];
};

// The batch record of an image's own block.
template <typename Params>
avifgpu_batch_image BatchImageOf(const Params& p)
{
    avifgpu_batch_image image{};
    image.width = p.width;
    image.height = p.rowCount;
    image.rows = const_cast<void*>(static_cast<const void*>(p.rows));
    image.row_stride_bytes = p.rowStride;
    for (int k = 0; k < 4; ++k)
    {
        image.planes.data[k] = const_cast<void*>(static_cast<const void*>(p.plane[k]));
        image.planes.stride[k] = p.planeStride[k];
    }
    return image;
}

// Marks the pixels of the record [x, x + width) x [y, y + rows) of `image`, from its rows pointer.
void Cover(std::vector<int>& count, const FakeImage& im, const BatchRecord& r, int description, int batch)
{
    const int64_t offset = static_cast<int64_t>(reinterpret_cast<uintptr_t>(r.rows) - im.rowsBase);
    const int y0 = static_cast<int>(offset / im.p.rowStride);
    const int x0 = static_cast<int>(offset % im.p.rowStride) / im.colBytes;
    if (r.width <= 0 || r.rowCount <= 0 || x0 + r.width > im.p.width || y0 + r.rowCount > im.p.rowCount)
    {
        Fail("record outside its image", description, batch);
        return;
    }
    // chroma plane 1 must sit at the window's first site, as EncodeWindow places it
    if (im.g[1].present)
    {
        const uintptr_t expected = im.planeBase[1] + static_cast<uintptr_t>((y0 >> im.g[1].ys) * im.p.planeStride[1]) +
                                   static_cast<uintptr_t>((x0 >> im.g[1].xs) * im.g[1].bytesPerSample);
        if (reinterpret_cast<uintptr_t>(r.plane[1]) != expected || (x0 & ((1 << im.g[1].xs) - 1)) || (y0 & ((1 << im.g[1].ys) - 1)))
        {
            Fail("chroma plane of a record", description, batch);
        }
    }
    for (int y = y0; y < y0 + r.rowCount; ++y)
    {
        for (int x = x0; x < x0 + r.width; ++x)
        {
            ++count[static_cast<size_t>(y) * im.p.width + x];
        }
    }
}

} // namespace

int main()
{
    std::mt19937 rng(1234);
    int descriptions = 0;
    long long batches = 0, images = 0;
    static_assert(sizeof(EncodeParams) + 16 + 2 * kBatchChunkImages * sizeof(BatchRecord) <= 32764, "edge parameters");
    for (int hostDepth : { 8, 16, 32 })
        for (int channels = 1; channels <= 4; ++channels)
            for (int alpha : { 0, 1, 2 })
                for (int depth : { 8, 10, 12 })
                    for (int layout : { 0, 1 })
                        for (int chroma : { 1, 2, 3 })
                            for (int matrix : { 1, 0, 9 })
                            {
                                avifgpu_encode_desc d{};
                                d.struct_size = sizeof(d);
                                d.width = 16;
                                d.height = 16;
                                d.host_depth = hostDepth;
                                d.host_channels = channels;
                                d.alpha_state = alpha;
                                d.image_bit_depth = depth;
                                d.transfer = AVIFGPU_TRANSFER_CLIP;
                                d.pq_peak_nits = 80;
                                d.layout = layout;
                                d.chroma = chroma;
                                d.nclx = avifgpu_nclx{ 1, 1, 13, matrix, 1 };
                                if ((layout == 0 && (chroma != 3 || matrix != 1)) || ValidateEncodeDesc(&d, nullptr) != AVIFGPU_OK)
                                {
                                    continue;
                                }
                                ++descriptions;
                                int planeMask = 0;
                                for (int k = 0; k < 4; ++k)
                                {
                                    planeMask |= EncodePlaneGeometry(d, k).present ? 1 << k : 0;
                                }
                                for (int verified : { 0, 1 })
                                {
                                    EncodeParams shared;
                                    FillEncodeParams(d, &shared);
                                    shared.verifiedPremultiply = verified;
                                    for (int trial = 0; trial < 3; ++trial)
                                    {
                                        const int n = 1 + static_cast<int>(rng() % (trial == 2 ? 300 : 20));
                                        std::vector<FakeImage> fake(n);
                                        std::vector<avifgpu_batch_image> batch(n);
                                        for (int i = 0; i < n; ++i)
                                        {
                                            avifgpu_encode_desc di = d;
                                            const int kind = static_cast<int>(rng() % 5);
                                            di.width = kind == 0 ? 1 + static_cast<int>(rng() % 9) : 1 + static_cast<int>(rng() % 70);
                                            di.height = kind == 1 ? 1 : 1 + static_cast<int>(rng() % 9);
                                            FakeImage& im = fake[i];
                                            FillEncodeParams(di, &im.p);
                                            im.colBytes = EncodeHostColBytes(di);
                                            const bool misaligned = rng() % 6 == 0;
                                            im.rowsBase = (static_cast<uintptr_t>(i + 1) << 36) + (misaligned ? 2 : 0);
                                            im.p.rows = reinterpret_cast<const void*>(im.rowsBase);
                                            im.p.rowStride = (static_cast<int64_t>(di.width) * im.colBytes + 63) / 64 * 64 + 64;
                                            im.p.rowCount = di.height;
                                            im.p.verifiedPremultiply = verified;
                                            for (int k = 0; k < 4; ++k)
                                            {
                                                im.g[k] = EncodePlaneGeometry(di, k);
                                                im.planeBase[k] = 0;
                                                if (!im.g[k].present)
                                                {
                                                    continue;
                                                }
                                                im.planeBase[k] = (static_cast<uintptr_t>(i + 1) << 36) + (static_cast<uintptr_t>(k + 1) << 30);
                                                im.p.plane[k] = reinterpret_cast<void*>(im.planeBase[k]);
                                                im.p.planeStride[k] = static_cast<int64_t>(im.g[k].widthSamples) * im.g[k].bytesPerSample + 128;
                                            }
                                            batch[i] = BatchImageOf(im.p);
                                        }
                                        BatchPlan plan;
                                        PlanEncodeBatch(shared, hostDepth, planeMask, batch.data(), n, &plan);
                                        ++batches;
                                        images += n;
                                        std::vector<std::vector<int>> count(n);
                                        std::vector<int> batched(n, 0);
                                        for (int i = 0; i < n; ++i)
                                        {
                                            count[i].assign(static_cast<size_t>(fake[i].p.width) * fake[i].p.rowCount, 0);
                                        }
                                        int previous = -1;
                                        for (const BatchChunk& c : plan.chunks)
                                        {
                                            if (c.images < 1 || c.images > kBatchChunkImages) Fail("chunk size", descriptions, static_cast<int>(batches));
                                            int64_t units = 0;
                                            for (int j = 0; j < c.images; ++j)
                                            {
                                                const int i = c.imageIndex[j];
                                                if (i <= previous) Fail("image order", descriptions, static_cast<int>(batches));
                                                previous = i;
                                                batched[i] = 1;
                                                const Interior inner = EncodeBlockInterior(EncodeBatchFamilyOf(fake[i].p, hostDepth), fake[i].p, hostDepth);
                                                const BatchRecord& r = c.interior[j];
                                                if (r.firstUnit != units || r.width != inner.width || r.rowCount != inner.rows || r.rows != fake[i].p.rows)
                                                {
                                                    Fail("interior record", descriptions, static_cast<int>(batches));
                                                }
                                                units += BatchInteriorUnits(r.width, r.rowCount, fake[i].p.ys);
                                                Cover(count[i], fake[i], r, descriptions, static_cast<int>(batches));
                                            }
                                            if (units != c.interiorUnits) Fail("interior units", descriptions, static_cast<int>(batches));
                                            units = 0;
                                            for (int j = 0; j < c.windows; ++j)
                                            {
                                                const int i = c.windowImage[j];
                                                const BatchRecord& r = c.window[j];
                                                if (r.firstUnit != units) Fail("window units", descriptions, static_cast<int>(batches));
                                                units += BatchEdgeUnits(r.width, r.rowCount, fake[i].p.xs, fake[i].p.ys);
                                                Cover(count[i], fake[i], r, descriptions, static_cast<int>(batches));
                                            }
                                            if (units != c.windowUnits) Fail("window units", descriptions, static_cast<int>(batches));
                                            // a second launch exactly when some image of the chunk has a strip outside its interior
                                            bool edges = false;
                                            for (int j = 0; j < c.images; ++j)
                                            {
                                                const EncodeParams& q = fake[c.imageIndex[j]].p;
                                                const Interior inner = EncodeBlockInterior(EncodeBatchFamilyOf(q, hostDepth), q, hostDepth);
                                                edges = edges || inner.width < q.width || inner.rows < q.rowCount;
                                            }
                                            if (BatchChunkLaunches(c) != (edges ? 2 : 1)) Fail("launches", descriptions, static_cast<int>(batches));
                                        }
                                        int lastFallback = -1;
                                        for (const int32_t i : plan.fallback)
                                        {
                                            if (i <= lastFallback || batched[i]) Fail("fallback order", descriptions, static_cast<int>(batches));
                                            lastFallback = i;
                                            batched[i] = 2;
                                            for (int& v : count[i]) ++v;
                                        }
                                        for (int i = 0; i < n; ++i)
                                        {
                                            const bool eligible = EncodeBlockInterior(EncodeBatchFamilyOf(fake[i].p, hostDepth), fake[i].p, hostDepth).width > 0;
                                            if (eligible != (batched[i] == 1) || batched[i] == 0)
                                            {
                                                Fail("eligible / fallback against the predicate", descriptions, static_cast<int>(batches));
                                            }
                                            for (int v : count[i])
                                            {
                                                if (v != 1)
                                                {
                                                    Fail("pixel not covered exactly once", descriptions, static_cast<int>(batches));
                                                    break;
                                                }
                                            }
                                        }
                                    }
                                }
                            }
    std::printf("encode descriptions=%d batches=%lld images=%lld\n", descriptions, batches, images);

    // decode: every YCbCr integer-host description; coverage of every pixel from the rows pointers, routing against
    // DecodeBlockInterior of DecodeBatchFamilyOf, launches against the strips
    int decodeDescriptions = 0;
    long long decodeImages = 0;
    for (int hostDepth : { 8, 16 })
        for (int bitDepth : { 8, 10, 12 })
            for (int alpha : { 0, 1, 2 })
                for (int chroma : { 1, 2, 3 })
                {
                    avifgpu_decode_desc d{};
                    d.struct_size = sizeof(d);
                    d.width = 16;
                    d.height = 16;
                    d.colorspace = AVIFGPU_COLORSPACE_YCBCR;
                    d.chroma = chroma;
                    d.bit_depth = bitDepth;
                    d.alpha_state = alpha;
                    d.host_depth = hostDepth;
                    d.nclx = avifgpu_nclx{ 1, 1, 13, 1, 1 };
                    d.pq_peak_nits = 80;
                    int32_t transfer = 0;
                    DecodeParams probe{};
                    if (ValidateDecodeDesc(&d, &transfer, nullptr) != AVIFGPU_OK || !FillDecodeParams(d, transfer, &probe, nullptr))
                    {
                        continue;
                    }
                    ++decodeDescriptions;
                    int planeMask = 0;
                    for (int k = 0; k < 4; ++k)
                    {
                        planeMask |= DecodePlaneGeometry(d, k).present ? 1 << k : 0;
                    }
                    for (int trial = 0; trial < 3; ++trial)
                    {
                        const int n = 1 + static_cast<int>(rng() % (trial == 2 ? 300 : 20));
                        std::vector<DecodeParams> params(n);
                        std::vector<uintptr_t> rowsBase(n);
                        const int colBytes = DecodeHostColBytes(d);
                        for (int i = 0; i < n; ++i)
                        {
                            avifgpu_decode_desc di = d;
                            di.width = rng() % 5 == 0 ? 1 + static_cast<int>(rng() % 9) : 1 + static_cast<int>(rng() % 70);
                            di.height = 1 + static_cast<int>(rng() % 9);
                            DecodeParams& p = params[i];
                            FillDecodeParams(di, transfer, &p, nullptr);
                            rowsBase[i] = (static_cast<uintptr_t>(i + 1) << 36) + (rng() % 6 == 0 ? 2 : 0);
                            p.rows = reinterpret_cast<void*>(rowsBase[i]);
                            p.rowStride = (static_cast<int64_t>(di.width) * colBytes + 63) / 64 * 64 + 64;
                            p.rowCount = di.height;
                            for (int k = 0; k < 4; ++k)
                            {
                                const PlaneGeometry g = DecodePlaneGeometry(di, k);
                                if (g.present)
                                {
                                    p.plane[k] = reinterpret_cast<const void*>((static_cast<uintptr_t>(i + 1) << 36) + (static_cast<uintptr_t>(k + 1) << 30));
                                    p.planeStride[k] = static_cast<int64_t>(g.widthSamples) * g.bytesPerSample + 128;
                                }
                            }
                        }
                        std::vector<avifgpu_batch_image> batch(n);
                        for (int i = 0; i < n; ++i)
                        {
                            batch[i] = BatchImageOf(params[i]);
                        }
                        BatchPlan plan;
                        PlanDecodeBatch(probe, planeMask, batch.data(), n, &plan);
                        decodeImages += n;
                        std::vector<std::vector<int>> count(n);
                        std::vector<int> batched(n, 0);
                        for (int i = 0; i < n; ++i)
                        {
                            count[i].assign(static_cast<size_t>(params[i].width) * params[i].rowCount, 0);
                        }
                        const auto cover = [&](int i, const BatchRecord& r)
                        {
                            const int64_t offset = static_cast<int64_t>(reinterpret_cast<uintptr_t>(r.rows) - rowsBase[i]);
                            const int y0 = static_cast<int>(offset / params[i].rowStride), x0 = static_cast<int>(offset % params[i].rowStride) / colBytes;
                            if (x0 + r.width > params[i].width || y0 + r.rowCount > params[i].rowCount || (y0 & params[i].ys))
                            {
                                Fail("decode record outside its image or off a row pair", decodeDescriptions, trial);
                                return;
                            }
                            for (int y = y0; y < y0 + r.rowCount; ++y)
                                for (int x = x0; x < x0 + r.width; ++x) ++count[i][static_cast<size_t>(y) * params[i].width + x];
                        };
                        for (const BatchChunk& c : plan.chunks)
                        {
                            bool edges = false;
                            for (int j = 0; j < c.images; ++j)
                            {
                                const int i = c.imageIndex[j];
                                batched[i] = 1;
                                const Interior inner = DecodeBlockInterior(DecodeBatchFamilyOf(params[i]), params[i]);
                                edges = edges || inner.width < params[i].width || inner.rows < params[i].rowCount;
                                cover(i, c.interior[j]);
                            }
                            for (int j = 0; j < c.windows; ++j) cover(c.windowImage[j], c.window[j]);
                            if (BatchChunkLaunches(c) != (edges ? 2 : 1)) Fail("decode launches", decodeDescriptions, trial);
                        }
                        for (const int32_t i : plan.fallback)
                        {
                            batched[i] = 2;
                            for (int& v : count[i]) ++v;
                        }
                        for (int i = 0; i < n; ++i)
                        {
                            if ((DecodeBlockInterior(DecodeBatchFamilyOf(params[i]), params[i]).width > 0) != (batched[i] == 1)) Fail("decode routing", decodeDescriptions, trial);
                            for (int v : count[i])
                                if (v != 1) { Fail("decode pixel not covered exactly once", decodeDescriptions, trial); break; }
                        }
                    }
                }
    std::printf("decode descriptions=%d images=%lld\n", decodeDescriptions, decodeImages);
    return g_failures == 0 ? 0 : 1;
}
