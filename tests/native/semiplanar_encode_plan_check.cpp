// tests/native/semiplanar_encode_plan_check.cpp -- host-side check of the semi-planar and MSB-aligned encode destinations
// (avifgpu_encode_desc.dest_layout) in csrc/host_params.cpp, csrc/kernel_params.h and csrc/batch_plan.h:
//   validation   every layout bit set x host depth x channel count x layout kind x image depth: the description's own
//                checks first, then unknown bits BAD_PARAM, non-zero layouts for planar YCbCr only (UNSUPPORTED otherwise),
//                MSB-aligned for 10/12-bit images only (BAD_PARAM);
//   API-10 size  a description that ends where API version 10's did, placed against an inaccessible page: validation,
//                widening, geometry, host column bytes and the parameter block read nothing past it, and it means planar;
//   geometry     interleaved chroma is one plane 1 of 2 * ((width + xs) >> xs) samples and no plane 2; EncodeWindow moves
//                it by two samples per site;
//   block halves EncodeRgbIntBlockInterior and EncodeRgbF32BlockInterior against a restatement of the stores' alignment
//                (interleaved: twice the planar chroma's, at most 16 bytes; plane 2 not read) on random buffers;
//   batches      for every 8/16-bit RGB(A) description in each layout, seeded batches of mixed sizes (odd widths, one-row
//                images, misaligned rows, Y and interleaved chroma planes): every pixel covered exactly once; an image
//                batched exactly when the block half takes it; records' planes where EncodeWindow puts them; interior units
//                of 256 pixels, edge units of 256 sites; one or two launches per chunk.
// Prints "semiplanar_encode validations=V descriptions=N images=K units=U"; exit code 1 on any failure.
#include "batch_plan.h"
#include "host_params.h"

#include <sys/mman.h>
#include <unistd.h>

#include <cstddef>
#include <cstdio>
#include <cstring>
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

avifgpu_encode_desc Desc(int hostDepth, int channels, int alphaState, int imageDepth, int layout, int chroma, int dest)
{
    avifgpu_encode_desc d{};
    d.struct_size = sizeof(d);
    d.width = 64;
    d.height = 8;
    d.host_depth = hostDepth;
    d.host_channels = channels;
    d.alpha_state = alphaState;
    d.image_bit_depth = imageDepth;
    d.transfer = AVIFGPU_TRANSFER_PQ;
    d.pq_peak_nits = 10000;
    d.layout = layout;
    d.chroma = chroma;
    d.nclx = avifgpu_nclx{ 1, 9, 16, 9, 1 };
    d.hlg_display_gamma = 1.2f;
    d.hlg_peak_nits = 1000;
    d.dest_layout = dest;
    return d;
}

int AlphaFor(int channels) { return (channels == 2 || channels == 4) ? AVIFGPU_ALPHA_STRAIGHT : AVIFGPU_ALPHA_NONE; }

avifgpu_batch_image BatchImageOf(const EncodeParams& p)
{
    avifgpu_batch_image image{};
    image.width = p.width;
    image.height = p.rowCount;
    image.rows = const_cast<void*>(p.rows);
    image.row_stride_bytes = p.rowStride;
    for (int k = 0; k < 4; ++k)
    {
        image.planes.data[k] = p.plane[k];
        image.planes.stride[k] = p.planeStride[k];
    }
    return image;
}

// The alignment the tuned stores need of interleaved plane 1, restated from the stores: twice the planar chroma's bytes
// per thread (integer: 4 or 8 sites of 1 or 2 bytes; float: 2 or 4 sites of 2 bytes), at most 16 (16-bit 4:4:4 is two
// 128-bit stores).
int InterleavedAlignment(const EncodeParams& p, bool floatHost)
{
    const int planar = floatHost ? (p.xs ? 4 : 8) : (p.xs ? 4 : 8) * (p.imageDepth > 8 ? 2 : 1);
    return 2 * planar > 16 ? 16 : 2 * planar;
}

void Cover(std::vector<int>& count, const EncodeParams& p, int hostDepth, const BatchRecord& r, int colBytes, int description, int batch)
{
    const int64_t offset = static_cast<int64_t>(reinterpret_cast<uintptr_t>(r.rows) - reinterpret_cast<uintptr_t>(p.rows));
    const int y0 = static_cast<int>(offset / p.rowStride);
    const int x0 = static_cast<int>(offset % p.rowStride) / colBytes;
    if (offset < 0 || r.width <= 0 || r.rowCount <= 0 || x0 + r.width > p.width || y0 + r.rowCount > p.rowCount || (y0 & p.ys) != 0 || (x0 & p.xs) != 0)
    {
        Fail("record outside its image or off a chroma site", description, batch);
        return;
    }
    const EncodeParams w = EncodeWindow(p, hostDepth, x0, y0, r.width, r.rowCount);
    for (int k = 0; k < 4; ++k)
    {
        if (r.plane[k] != w.plane[k] || r.planeStride[k] != p.planeStride[k])
        {
            Fail("record plane not where EncodeWindow puts it", description, batch);
        }
    }
    if (SourceInterleaved(p.destLayout))
    {
        const int64_t expected = static_cast<int64_t>(y0 >> p.ys) * p.planeStride[1] + static_cast<int64_t>(x0 >> p.xs) * 2 * (p.imageDepth > 8 ? 2 : 1);
        if (static_cast<const uint8_t*>(r.plane[1]) - static_cast<const uint8_t*>(p.plane[1]) != expected || r.plane[2] != nullptr)
        {
            Fail("interleaved chroma window offset", description, batch);
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

int Validations()
{
    int checked = 0;
    for (int dest : { 0, 1, 2, 3, 4, 5, 8, -1 })
        for (int hostDepth : { 8, 16, 32 })
            for (int channels : { 1, 2, 3, 4 })
                for (int layout : { AVIFGPU_LAYOUT_REFERENCE, AVIFGPU_LAYOUT_PLANAR_YCBCR })
                    for (int imageDepth : { 8, 10, 12 })
                    {
                        avifgpu_encode_desc d = Desc(hostDepth, channels, AlphaFor(channels), imageDepth, layout, AVIFGPU_CHROMA_420, 0);
                        const int base = ValidateEncodeDesc(&d, nullptr);
                        d.dest_layout = dest;
                        const int status = ValidateEncodeDesc(&d, nullptr);
                        int expected = base;
                        if (base == AVIFGPU_OK && dest != 0)
                        {
                            if (dest & ~3)
                            {
                                expected = AVIFGPU_ERR_BAD_PARAM;
                            }
                            else if (layout != AVIFGPU_LAYOUT_PLANAR_YCBCR)
                            {
                                expected = AVIFGPU_ERR_UNSUPPORTED;
                            }
                            else if ((dest & AVIFGPU_SOURCE_MSB_ALIGNED) && imageDepth == 8)
                            {
                                expected = AVIFGPU_ERR_BAD_PARAM;
                            }
                        }
                        if (status != expected)
                        {
                            std::printf("FAIL validation dest %d host %d channels %d layout %d depth %d: %d, expected %d\n", dest, hostDepth, channels, layout,
                                        imageDepth, status, expected);
                            ++g_failures;
                        }
                        ++checked;
                    }

    // An API-10-sized description as the last bytes before an inaccessible page: whatever would lie past it cannot be read.
    const long page = sysconf(_SC_PAGESIZE);
    uint8_t* pages = static_cast<uint8_t*>(mmap(nullptr, 2 * page, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0));
    if (pages == MAP_FAILED || mprotect(pages + page, page, PROT_NONE) != 0)
    {
        std::printf("FAIL guard page\n");
        ++g_failures;
        return checked;
    }
    const avifgpu_encode_desc current = Desc(16, 4, AVIFGPU_ALPHA_STRAIGHT, 10, AVIFGPU_LAYOUT_PLANAR_YCBCR, AVIFGPU_CHROMA_420, 3);
    auto* old = reinterpret_cast<avifgpu_encode_desc*>(pages + page - AVIFGPU_ENCODE_DESC_V10_SIZE);
    std::memcpy(old, &current, AVIFGPU_ENCODE_DESC_V10_SIZE);
    old->struct_size = AVIFGPU_ENCODE_DESC_V10_SIZE;
    avifgpu_encode_desc full;
    const avifgpu_encode_desc* widened = WidenEncodeDesc(old, &full);
    EncodeParams fromOld;
    FillEncodeParams(*widened, &fromOld);
    const PlaneGeometry g1 = EncodePlaneGeometry(*widened, 1), g2 = EncodePlaneGeometry(*widened, 2);
    if (AVIFGPU_ENCODE_DESC_V10_SIZE != 124 || sizeof(avifgpu_encode_desc) != 128 || ValidateEncodeDesc(old, nullptr) != AVIFGPU_OK ||
        DestLayoutOf(*old) != 0 || widened != &full || full.struct_size != sizeof(avifgpu_encode_desc) || full.dest_layout != 0 ||
        ValidateEncodeDesc(widened, nullptr) != AVIFGPU_OK || full.image_bit_depth != 10 || full.pq_peak_nits != 10000 ||
        std::memcmp(full.row_matrix, current.row_matrix, sizeof(full.row_matrix)) != 0 || EncodeHostColBytes(*widened) != 8 ||
        fromOld.destLayout != 0 || !g1.present || g1.widthSamples != 32 || !g2.present)
    {
        std::printf("FAIL API-10-sized description\n");
        ++g_failures;
    }
    munmap(pages, 2 * page);
    if (WidenEncodeDesc(&current, &full) != &current || DestLayoutOf(current) != 3)
    {
        std::printf("FAIL current-sized description\n");
        ++g_failures;
    }
    avifgpu_encode_desc odd = current;
    for (uint32_t size : { 0u, 40u, 120u, 126u, 132u })
    {
        odd.struct_size = size;
        if (ValidateEncodeDesc(&odd, nullptr) != AVIFGPU_ERR_BAD_PARAM || WidenEncodeDesc(&odd, &full) != &odd)
        {
            std::printf("FAIL description size %u\n", size);
            ++g_failures;
        }
    }
    checked += 3;

    // geometry: 7 x 5 -> 4 x 3 sites (4:2:0), 4 x 5 (4:2:2), 7 x 5 (4:4:4); and EncodeWindow's move of plane 1
    for (int chroma : { AVIFGPU_CHROMA_420, AVIFGPU_CHROMA_422, AVIFGPU_CHROMA_444 })
        for (int dest : { 0, 1, 2, 3 })
        {
            avifgpu_encode_desc d = Desc(16, 4, AVIFGPU_ALPHA_STRAIGHT, 12, AVIFGPU_LAYOUT_PLANAR_YCBCR, chroma, dest);
            d.width = 7;
            d.height = 5;
            const int xs = chroma == AVIFGPU_CHROMA_444 ? 0 : 1, ys = chroma == AVIFGPU_CHROMA_420 ? 1 : 0;
            const int sites = (7 + xs) >> xs, chromaRows = (5 + ys) >> ys;
            const bool interleaved = dest & 1;
            const PlaneGeometry g0 = EncodePlaneGeometry(d, 0), c1 = EncodePlaneGeometry(d, 1), c2 = EncodePlaneGeometry(d, 2), g3 = EncodePlaneGeometry(d, 3);
            if (!g0.present || g0.widthSamples != 7 || !g3.present || g3.widthSamples != 7 || !c1.present || c1.height != chromaRows ||
                c1.bytesPerSample != 2 || c1.widthSamples != (interleaved ? 2 * sites : sites) || c2.present == interleaved ||
                (!interleaved && (c2.widthSamples != sites || c2.height != chromaRows)) || (interleaved && c2.bytesPerSample != 0))
            {
                std::printf("FAIL geometry chroma %d dest %d\n", chroma, dest);
                ++g_failures;
            }
            EncodeParams p;
            FillEncodeParams(d, &p);
            for (int k = 0; k < 4; ++k)
            {
                p.plane[k] = (k == 2 && interleaved) ? nullptr : reinterpret_cast<void*>(static_cast<uintptr_t>(k + 1) << 32);
                p.planeStride[k] = 1024 * (k + 1);
            }
            p.rows = reinterpret_cast<const void*>(static_cast<uintptr_t>(1) << 40);
            p.rowStride = 4096;
            p.width = 7;
            p.rowCount = 5;
            const int x0 = 4, y0 = 2;
            const EncodeParams w = EncodeWindow(p, 16, x0, y0, 3, 3);
            const int64_t expected1 = static_cast<int64_t>(y0 >> ys) * p.planeStride[1] + static_cast<int64_t>(x0 >> xs) * (interleaved ? 2 : 1) * 2;
            const int64_t expected0 = static_cast<int64_t>(y0) * p.planeStride[0] + x0 * 2;
            if (static_cast<uint8_t*>(w.plane[1]) - static_cast<uint8_t*>(p.plane[1]) != expected1 ||
                static_cast<uint8_t*>(w.plane[0]) - static_cast<uint8_t*>(p.plane[0]) != expected0 || (interleaved && w.plane[2] != nullptr) ||
                static_cast<uint8_t*>(w.plane[3]) - static_cast<uint8_t*>(p.plane[3]) != static_cast<int64_t>(y0) * p.planeStride[3] + x0 * 2)
            {
                std::printf("FAIL EncodeWindow chroma %d dest %d\n", chroma, dest);
                ++g_failures;
            }
            ++checked;
        }
    return checked;
}

// The block halves against the restated alignment rule on random buffers, both kernel families, every layout.
void BlockHalves(std::mt19937_64& rng)
{
    for (int hostDepth : { 8, 16, 32 })
        for (int imageDepth : { 8, 10, 12 })
            for (int chroma : { 1, 2, 3 })
                for (int dest : { 0, 1, 2, 3 })
                    for (int channels : { 3, 4 })
                    {
                        const avifgpu_encode_desc d = Desc(hostDepth, channels, AlphaFor(channels), imageDepth, AVIFGPU_LAYOUT_PLANAR_YCBCR, chroma, dest);
                        if (ValidateEncodeDesc(&d, nullptr) != AVIFGPU_OK)
                        {
                            continue;
                        }
                        EncodeParams p;
                        FillEncodeParams(d, &p);
                        const bool floatHost = hostDepth == 32;
                        const int planeBytes = imageDepth > 8 ? 2 : 1;
                        for (int trial = 0; trial < 200; ++trial)
                        {
                            const auto pointer = [&](int k) { return reinterpret_cast<void*>((static_cast<uintptr_t>(k + 1) << 32) + 2 * (rng() % 16)); };
                            p.rows = pointer(4);
                            p.rowStride = 4096 + 4 * static_cast<int64_t>(rng() % 8);
                            for (int k = 0; k < 4; ++k)
                            {
                                p.plane[k] = (k == 2 && (dest & 1)) || (k == 3 && channels == 3) ? nullptr : pointer(k);
                                p.planeStride[k] = 2048 + 2 * static_cast<int64_t>(rng() % 16);
                            }
                            p.width = 1 + static_cast<int>(rng() % 40);
                            p.rowCount = 1 + static_cast<int>(rng() % 5);
                            const bool chromaOk = (dest & 1) ? Aligned(p.plane[1], p.planeStride[1], InterleavedAlignment(p, floatHost))
                                                             : Aligned(p.plane[1], p.planeStride[1], floatHost ? (p.xs ? 4 : 8) : (p.xs ? 4 : 8) * planeBytes) &&
                                                                   Aligned(p.plane[2], p.planeStride[2], floatHost ? (p.xs ? 4 : 8) : (p.xs ? 4 : 8) * planeBytes);
                            const int evenRows = p.ys ? (p.rowCount & ~1) : p.rowCount;
                            Interior expected{ 0, 0 }, got;
                            if (floatHost)
                            {
                                const bool ok = chromaOk && Aligned(p.rows, p.rowStride, 16) && Aligned(p.plane[0], p.planeStride[0], 8) &&
                                                (channels == 3 || Aligned(p.plane[3], p.planeStride[3], 8)) && p.width >= 4 && evenRows >= 1;
                                expected = ok ? Interior{ p.width & ~3, evenRows } : Interior{ 0, 0 };
                                got = EncodeRgbF32BlockInterior(p);
                            }
                            else
                            {
                                const int rowAlign = (8 * channels * hostDepth / 8) % 16 == 0 ? 16 : 8;
                                const bool ok = chromaOk && Aligned(p.rows, p.rowStride, rowAlign) && Aligned(p.plane[0], p.planeStride[0], 8 * planeBytes) &&
                                                (channels == 3 || Aligned(p.plane[3], p.planeStride[3], 8 * planeBytes)) && p.width >= 8 && evenRows >= 1;
                                expected = ok ? Interior{ p.width & ~7, evenRows } : Interior{ 0, 0 };
                                got = EncodeRgbIntBlockInterior(p, hostDepth);
                            }
                            if (got.width != expected.width || got.rows != expected.rows)
                            {
                                Fail("block half against the restated alignment rule", hostDepth * 1000 + imageDepth * 10 + dest, trial);
                            }
                        }
                    }
}

} // namespace

int main()
{
    const int validations = Validations();
    std::mt19937_64 rng(20261018);
    BlockHalves(rng);
    int descriptions = 0;
    long long images = 0, units = 0;
    for (int hostDepth : { 8, 16 })
        for (int imageDepth : { 8, 10, 12 })
            for (int alphaCase : { 0, 1, 2 })
                for (int chroma : { 1, 2, 3 })
                    for (int dest : { 0, 1, 2, 3 })
                    {
                        const int channels = alphaCase == 0 ? 3 : 4;
                        const int alphaState = alphaCase == 0 ? AVIFGPU_ALPHA_NONE : alphaCase == 1 ? AVIFGPU_ALPHA_STRAIGHT : AVIFGPU_ALPHA_PREMULTIPLIED;
                        const avifgpu_encode_desc d = Desc(hostDepth, channels, alphaState, imageDepth, AVIFGPU_LAYOUT_PLANAR_YCBCR, chroma, dest);
                        if (ValidateEncodeDesc(&d, nullptr) != AVIFGPU_OK)
                        {
                            continue;
                        }
                        EncodeParams probe;
                        FillEncodeParams(d, &probe);
                        probe.verifiedPremultiply = 1;
                        if (probe.destLayout != dest)
                        {
                            Fail("FillEncodeParams does not carry the layout", descriptions, -1);
                        }
                        const EncodeFamily family = EncodeBatchFamilyOf(probe, hostDepth);
                        const bool tuned = family == EncodeFamily::RgbInt;
                        EncodeParams planarProbe = probe;
                        planarProbe.destLayout = 0;
                        if (!tuned || (EncodeBatchFamilyOf(planarProbe, hostDepth) == EncodeFamily::RgbInt) != tuned)
                        {
                            Fail("description routing depends on the layout", descriptions, -1);
                        }
                        ++descriptions;
                        int planeMask = 0;
                        for (int k = 0; k < 4; ++k)
                        {
                            planeMask |= EncodePlaneGeometry(d, k).present ? 1 << k : 0;
                        }
                        if (((planeMask >> 2) & 1) == (dest & 1) || (planeMask & 3) != 3 || ((planeMask >> 3) & 1) != (channels == 4 ? 1 : 0))
                        {
                            Fail("plane mask", descriptions, -1);
                        }
                        const int colBytes = EncodeHostColBytes(d);
                        for (int trial = 0; trial < 3; ++trial)
                        {
                            const int n = 1 + static_cast<int>(rng() % (trial == 2 ? 200 : 24));
                            std::vector<EncodeParams> params(n);
                            std::vector<int> shapes(n);
                            for (int i = 0; i < n; ++i)
                            {
                                avifgpu_encode_desc di = d;
                                const int shape = shapes[i] = static_cast<int>(rng() % 8);
                                di.width = shape == 0 ? 1 + static_cast<int>(rng() % 9) : 1 + static_cast<int>(rng() % 600);
                                di.height = shape == 1 ? 1 : 1 + static_cast<int>(rng() % 9);
                                EncodeParams& p = params[i];
                                FillEncodeParams(di, &p);
                                p.verifiedPremultiply = 1;
                                const uintptr_t base = static_cast<uintptr_t>(i + 1) << 36;
                                p.rows = reinterpret_cast<const void*>(base + (shape == 2 ? 4 : 0));
                                p.rowStride = (static_cast<int64_t>(di.width) * colBytes + 63) / 64 * 64 + 64;
                                p.rowCount = di.height;
                                for (int k = 0; k < 4; ++k)
                                {
                                    const PlaneGeometry g = EncodePlaneGeometry(di, k);
                                    if (g.present)
                                    {
                                        p.plane[k] = reinterpret_cast<void*>(base + (static_cast<uintptr_t>(k + 1) << 30) + (shape == 3 && k == 0 ? 2 : 0));
                                        p.planeStride[k] = (static_cast<int64_t>(g.widthSamples) * g.bytesPerSample + 63) / 64 * 64 + 128;
                                    }
                                }
                                // misalign plane 1 by half the interleaved store (shape 4) or just its stride (shape 5)
                                if ((shape == 4 || shape == 5) && (dest & 1))
                                {
                                    const int half = InterleavedAlignment(p, false) / 2;
                                    if (shape == 4)
                                    {
                                        p.plane[1] = static_cast<uint8_t*>(p.plane[1]) + half;
                                    }
                                    else
                                    {
                                        p.planeStride[1] += half;
                                    }
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
                            PlanEncodeBatch(probe, hostDepth, planeMask, batch.data(), n, &plan);
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
                                int64_t first = 0, windowFirst = 0;
                                for (int j = 0; j < c.images; ++j)
                                {
                                    const int i = c.imageIndex[j];
                                    if (i <= last)
                                    {
                                        Fail("image order", descriptions, trial);
                                    }
                                    last = i;
                                    batched[i] = 1;
                                    const Interior inner = EncodeBlockInterior(EncodeBatchFamilyOf(params[i], hostDepth), params[i], hostDepth);
                                    if (c.interior[j].width != inner.width || c.interior[j].rowCount != inner.rows || c.interior[j].firstUnit != first)
                                    {
                                        Fail("chunk interior", descriptions, trial);
                                    }
                                    first += BatchInteriorUnits(inner.width, inner.rows, params[i].ys);
                                    edges = edges || inner.width < params[i].width || inner.rows < params[i].rowCount;
                                    Cover(count[i], params[i], hostDepth, c.interior[j], colBytes, descriptions, trial);
                                }
                                if (first != c.interiorUnits)
                                {
                                    Fail("chunk unit total", descriptions, trial);
                                }
                                for (int j = 0; j < c.windows; ++j)
                                {
                                    const EncodeParams& p = params[c.windowImage[j]];
                                    if (c.window[j].firstUnit != windowFirst)
                                    {
                                        Fail("chunk window units", descriptions, trial);
                                    }
                                    windowFirst += BatchEdgeUnits(c.window[j].width, c.window[j].rowCount, p.xs, p.ys);
                                    Cover(count[c.windowImage[j]], p, hostDepth, c.window[j], colBytes, descriptions, trial);
                                }
                                if (windowFirst != c.windowUnits || BatchChunkLaunches(c) != (edges ? 2 : 1))
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
                                const EncodeParams& p = params[i];
                                const Interior inner = EncodeBlockInterior(EncodeBatchFamilyOf(p, hostDepth), p, hostDepth);
                                if ((inner.width > 0) != (batched[i] == 1))
                                {
                                    Fail("image routing", descriptions, trial);
                                }
                                if (!CoveredOnce(count[i]))
                                {
                                    Fail("host plan: pixel not covered exactly once", descriptions, trial);
                                }
                                if ((dest & 1) && inner.width > 0 && !Aligned(p.plane[1], p.planeStride[1], InterleavedAlignment(p, false)))
                                {
                                    Fail("a misaligned interleaved plane took the tuned route", descriptions, trial);
                                }
                                if ((dest & 1) && (shapes[i] == 4 || shapes[i] == 5) && inner.width > 0)
                                {
                                    Fail("a misaligned interleaved plane has an interior", descriptions, trial);
                                }
                                if ((dest & 1) && shapes[i] >= 6 && p.width >= 8 && p.rowCount >= 2 && inner.width == 0)
                                {
                                    Fail("an aligned interleaved image lost its interior", descriptions, trial);
                                }
                            }

                            // ---- the per-image step, as the plan kernel runs it ----
                            std::vector<int64_t> interiorFirst(n), interiorUnits(n);
                            int64_t total = 0;
                            for (int i = 0; i < n; ++i)
                            {
                                const BatchImagePlan step = PlanBatchEncodeImage(probe, hostDepth, family, planeMask, batch[i]);
                                std::vector<int> covered(static_cast<size_t>(params[i].width) * params[i].rowCount, 0);
                                const Interior inner = EncodeBlockInterior(EncodeBatchFamilyOf(params[i], hostDepth), params[i], hostDepth);
                                if (step.status != AVIFGPU_OK || step.interior.width != inner.width || (inner.width > 0 && step.interior.rowCount != inner.rows))
                                {
                                    Fail("step interior", descriptions, trial);
                                }
                                if (step.interior.width > 0)
                                {
                                    Cover(covered, params[i], hostDepth, step.interior, colBytes, descriptions, trial);
                                    const int64_t expected = static_cast<int64_t>((inner.width + kBatchUnitPixels - 1) / kBatchUnitPixels) * (inner.rows >> params[i].ys);
                                    if (step.interiorUnits != expected)
                                    {
                                        Fail("step interior units", descriptions, trial);
                                    }
                                }
                                for (int k = 0; k < step.windows; ++k)
                                {
                                    Cover(covered, params[i], hostDepth, step.window[k], colBytes, descriptions, trial);
                                    if (step.windowUnits[k] != BatchEdgeUnits(step.window[k].width, step.window[k].rowCount, params[i].xs, params[i].ys))
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
                            int record = 0;
                            for (int64_t u = 0; u < total; ++u)
                            {
                                record = FindRecord(interiorFirst.data(), n, record, u);
                                if (u < interiorFirst[record] || u >= interiorFirst[record] + interiorUnits[record])
                                {
                                    Fail("FindRecord", descriptions, trial);
                                    break;
                                }
                            }
                            units += total;
                        }
                    }
    std::printf("semiplanar_encode validations=%d descriptions=%d images=%lld units=%lld\n", validations, descriptions, images, units);
    return g_failures == 0 ? 0 : 1;
}
