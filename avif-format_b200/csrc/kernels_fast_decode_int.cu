// kernels_fast_decode_int.cu -- tuned decode kernels for the integer hosts: planar YCbCr (+ alpha) -> interleaved
// RGB(A) 8-bit (YuvDecode.cpp:281-399 driven by ReadHeifImage.cpp:83-184) and 16-bit (YuvDecode.cpp:401-519 driven by
// ReadHeifImage.cpp:186-288).  No transfer curve on these paths: table look-up, matrix, clamp, round -- HBM-bound work
// (4.5 B/px for 8-bit 4:2:0) if the instruction count per pixel stays near 25.
//
//   * a warp converts units of (2 rows for 4:2:0, else 1) x 256 pixels; a lane owns 8 adjacent pixels per row: one
//     64/128-bit load of Y per row, one 32/64-bit (sub-sampled) load of Cb and of Cr, 3-4 vector stores per row;
//   * the unorm -> float tables (YuvLookupTables.cpp:115-192) sit in shared memory; for 16-bit hosts the alpha output
//     (u16)(0.5f + a * 32768f) is tabulated whole;
//   * the chroma-dependent terms of YuvDecode.cpp:306-312 are evaluated once per chroma site and reused for every luma
//     sample the site covers (both rows of a 4:2:0 site); same float expressions, same association;
//   * premultiplied alpha, odd starting rows of a 4:2:0 block, depths above 12 bits and unaligned buffers stay with the
//     generic kernel.
#include "group_walk.cuh"
#include "int_units.cuh"
#include "kernel_params.h"
#include "launch_keys.h"
#include "packed_f32x2.cuh"
#include "pixel_math.cuh"
#include "stream_units.cuh"
#include "../../include/avifgpu.h"

#include <cuda_runtime.h>

namespace avifgpu
{

using namespace avifpix;

namespace
{

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

// SOURCE: the avifgpu_source_layout bits the kernel reads (LoadYccUnit); 0 is libheif's planar, low-bit layout.
template <typename SampleT, int XS, int YS, int ALPHA, int SOURCE>
__global__ void __launch_bounds__(kThreads, kYccBlocksPerSm) DecodeYccToRgbIntKernel(const IntDecodeParams p)
{
    constexpr int kRows = YS ? 2 : 1;
    extern __shared__ __align__(16) uint8_t sharedBytes[];
    const YccTables tables = StageYccTables<SampleT, ALPHA>(sharedBytes, p);
    __syncthreads();
    const YccFactors factors = MakeYccFactors<SampleT>(p.matrix);

    const int lane = threadIdx.x & 31;
    const int warpInBlock = threadIdx.x >> 5;
    const int unitsX = (p.width + kUnitPixels - 1) / kUnitPixels;
    const int unitRows = (p.rowCount + kRows - 1) / kRows;
    const long long unitCount = static_cast<long long>(unitsX) * unitRows;
    const int warpCount = static_cast<int>(gridDim.x) * kWarps;
    // unit coordinates advance incrementally (no division per unit)
    const long long firstUnit = static_cast<long long>(blockIdx.x) * kWarps + warpInBlock;
    const int stepRows = warpCount / unitsX;
    const int stepX = warpCount - stepRows * unitsX;
    int unitRow = static_cast<int>(firstUnit / unitsX);
    int unitX = static_cast<int>(firstUnit - static_cast<long long>(unitRow) * unitsX);

    // Software pipeline: the loads of unit i+1 are issued once unit i's samples have been expanded, so they are in flight
    // during its arithmetic and stores.
    Raw8<SampleT> rawY[kRows], rawA[kRows], rawCb, rawCr;
#pragma unroll
    for (int r = 0; r < kRows; ++r)
    {
        rawY[r] = {};
        rawA[r] = {};
    }
    rawCb = {};
    rawCr = {};
    LoadYccUnit<SampleT, XS, YS, ALPHA, SOURCE>(p, lane, unitRow, unitX, firstUnit < unitCount, rawY, rawA, rawCb, rawCr);

#pragma unroll 1
    for (long long unit = firstUnit; unit < unitCount; unit += warpCount)
    {
        const int x0 = unitX * kUnitPixels + lane * 8;
        const int y0 = unitRow * kRows;
        const bool laneActive = x0 < p.width;
        const bool secondRow = kRows == 2 && (y0 + 1) < p.rowCount;
        int nextRow = unitRow + stepRows;
        int nextX = unitX + stepX;
        if (nextX >= unitsX)
        {
            nextX -= unitsX;
            ++nextRow;
        }

        YccValues<XS, YS> values;
        ExpandYccUnit<SampleT, XS, YS, ALPHA>(p, tables, factors, rawY, rawA, rawCb, rawCr, values);

        LoadYccUnit<SampleT, XS, YS, ALPHA, SOURCE>(p, lane, nextRow, nextX, unit + warpCount < unitCount, rawY, rawA, rawCb, rawCr);
        unitRow = nextRow;
        unitX = nextX;
        if (!laneActive)
        {
            continue;
        }
        StoreYccUnit<SampleT, XS, YS, ALPHA>(p, factors, values, x0, y0, secondRow);
    }
}

template <typename SampleT, int XS, int YS, int ALPHA, int SOURCE>
cudaError_t LaunchOne(const IntDecodeParams& fp, int smCount, cudaStream_t stream)
{
    const size_t shared = YccTableBytes(fp.bitDepth, ALPHA && sizeof(SampleT) == 2);
    static std::atomic<uint64_t> configuredDevices{ 0 }; // per instantiation
    {
        const cudaError_t e = AllowDynamicShared(DecodeYccToRgbIntKernel<SampleT, XS, YS, ALPHA, SOURCE>, 64 * 1024, configuredDevices);
        if (e != cudaSuccess)
        {
            return e;
        }
    }
    constexpr int rowsPerUnit = YS ? 2 : 1;
    const long long units = static_cast<long long>((fp.width + kUnitPixels - 1) / kUnitPixels) * ((fp.rowCount + rowsPerUnit - 1) / rowsPerUnit);
    const unsigned grid = GridFor((units + kWarps - 1) / kWarps, static_cast<long long>(smCount) * kYccBlocksPerSm);
    DecodeYccToRgbIntKernel<SampleT, XS, YS, ALPHA, SOURCE><<<grid, kThreads, shared, stream>>>(fp);
    return cudaGetLastError();
}

// ---- monochrome and planar-RGB images: pure streaming ------------------------------------------------------------------
//
// Monochrome (ReadHeifImage.cpp:418-559 driving YuvDecode.cpp:55-203): out = round(table[Y]) -- no matrix, so the whole
// per-sample result is tabulated in shared memory; alpha is copied (8-bit) or tabulated (16-bit).
// Planar RGB: ConvertRgbGroup (stream_units.cuh).  A thread moves 8 pixels: one vector load per plane, CH * 8 samples
// stored as 64/128-bit words.
template <typename SampleT, int CHANNELS, bool MONO>
__global__ void __launch_bounds__(kStreamThreads) StreamDecodeKernel(const StreamDecodeParams p)
{
    constexpr bool kHost8 = sizeof(SampleT) == 1;
    extern __shared__ __align__(16) uint8_t sharedBytes[];
    uint16_t* lutY = reinterpret_cast<uint16_t*>(sharedBytes);
    uint16_t* lutA = lutY + (1u << p.bitDepth);
    if (MONO)
    {
        for (uint32_t i = threadIdx.x; i <= p.maxCode; i += blockDim.x)
        {
            const float y = UnormToFloatY(i, p.range); // YuvLookupTables.cpp:157-171
            lutY[i] = static_cast<uint16_t>(0.5f + (y * (kHost8 ? 255.0f : 32768.0f))); // YuvDecode.cpp:76, 150
            lutA[i] = static_cast<uint16_t>(0.5f + (UnormToFloatPlain(i, p.range.maxChannelFloat) * 32768.0f)); // YuvDecode.cpp:197
        }
        __syncthreads();
    }
    // An 8-bit full-range monochrome image read by an 8-bit host: the table maps every code to itself (checked, not
    // assumed) and the kernel is a strided copy -- eight shared-memory look-ups per 8 bytes otherwise bound it.
    bool identityLuma = false;
    if (MONO && kHost8)
    {
        bool mine = true;
        for (uint32_t i = threadIdx.x; i <= p.maxCode; i += blockDim.x)
        {
            mine = mine && lutY[i] == i;
        }
        identityLuma = __syncthreads_and(mine ? 1 : 0) != 0;
    }
    // A group is 8 samples per plane -- 8 bytes for an 8-bit image: there a thread keeps several groups' loads in flight
    // before it converts the first (ncu: 2048 threads x 8 bytes per SM in flight is too little; planar RGB8 +4 %).  With
    // 16-byte groups one at a time is better (two in flight cost registers and occupancy: planar RGB 10-bit -12 %).
    constexpr int kInFlight = kHost8 ? 4 : 1;
    // one group: 8 samples per plane -> 8 host pixels at `target`
    const auto convertGroup = [&](const Raw8<SampleT>(&raw)[CHANNELS], uint8_t* target)
    {
        if (!MONO)
        {
            ConvertRgbGroup<SampleT, CHANNELS>(raw, p.maxCode, target);
            return;
        }
        if (kHost8 && CHANNELS == 1)
        {
            if (identityLuma)
            {
                // the 8 bytes as they are: unpacking and repacking them made this path instruction-bound (76 % of the issue slots)
                __stcs(reinterpret_cast<uint2*>(target), make_uint2(raw[0].w[0], raw[0].w[1]));
                return;
            }
        }
        uint32_t samples[8 * CHANNELS];
#pragma unroll
        for (int i = 0; i < 8; ++i)
        {
#pragma unroll
            for (int c = 0; c < CHANNELS; ++c)
            {
                uint32_t v = Sample<SampleT>(raw[c], i);
                const bool isAlpha = CHANNELS == 2 && c == 1;
                if (!isAlpha)
                {
                    if (!(kHost8 && identityLuma))
                    {
                        v = lutY[kHost8 ? v : min(v, p.maxCode)];
                    }
                }
                else if (!kHost8)
                {
                    v = lutA[min(v, p.maxCode)];
                }
                samples[i * CHANNELS + c] = v;
            }
        }
        StoreStreamGroup<SampleT, CHANNELS>(samples, target);
    };
    const auto loadGroup = [&](Raw8<SampleT>(&raw)[CHANNELS], long long row, long long column) { LoadStreamGroup<SampleT, CHANNELS, MONO>(p, raw, row, column); };
    GroupWalk walk(static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x, static_cast<long long>(gridDim.x) * blockDim.x, p.groupsPerRow, p.rowCount);
    if (kInFlight == 1)
    {
        for (; walk.Inside(p.rowCount); walk.Advance(p.rowCount))
        {
            const long long row = walk.row;
            const long long column = static_cast<long long>(walk.column) * 8;
            Raw8<SampleT> raw[CHANNELS];
            loadGroup(raw, row, column);
            convertGroup(raw, p.rows + row * p.rowStride + column * static_cast<long long>(CHANNELS * sizeof(SampleT)));
        }
        return;
    }
    while (walk.Inside(p.rowCount))
    {
        Raw8<SampleT> rawAll[kInFlight][CHANNELS];
        long long targetOffset[kInFlight];
#pragma unroll
        for (int u = 0; u < kInFlight; ++u)
        {
            targetOffset[u] = -1;
            if (walk.Inside(p.rowCount))
            {
                const long long row = walk.row;
                const long long column = static_cast<long long>(walk.column) * 8;
                loadGroup(rawAll[u], row, column);
                targetOffset[u] = row * p.rowStride + column * static_cast<long long>(CHANNELS * sizeof(SampleT));
            }
            walk.Advance(p.rowCount);
        }
#pragma unroll
        for (int u = 0; u < kInFlight; ++u)
        {
            if (targetOffset[u] >= 0)
            {
                convertGroup(rawAll[u], p.rows + targetOffset[u]);
            }
        }
    }
}

template <typename SampleT, int CHANNELS, bool MONO>
cudaError_t LaunchStream(const StreamDecodeParams& sp, int smCount, cudaStream_t stream)
{
    const long long groups = static_cast<long long>(sp.groupsPerRow) * sp.rowCount;
    const unsigned grid = GridFor((groups + kStreamThreads - 1) / kStreamThreads, static_cast<long long>(smCount) * kStreamBlocksPerSm);
    const size_t shared = MONO ? 2 * sizeof(uint16_t) * (static_cast<size_t>(1) << sp.bitDepth) : 0;
    StreamDecodeKernel<SampleT, CHANNELS, MONO><<<grid, kStreamThreads, shared, stream>>>(sp);
    return cudaGetLastError();
}

} // namespace

// Monochrome and planar-RGB images for the integer hosts.
cudaError_t LaunchDecodeStream(const DecodeParams& p, Interior inner, void* streamHandle)
{
    cudaStream_t stream = static_cast<cudaStream_t>(streamHandle);
    const bool mono = p.colorspace == AVIFGPU_COLORSPACE_MONOCHROME;
    StreamDecodeParams sp = StreamDecodeDescription(p);
    for (int k = 0; k < 4; ++k)
    {
        sp.plane[k] = static_cast<const uint8_t*>(p.plane[k]);
        sp.planeStride[k] = p.planeStride[k];
    }
    sp.rows = static_cast<uint8_t*>(p.rows);
    sp.rowStride = p.rowStride;
    sp.groupsPerRow = inner.width / 8;
    sp.rowCount = inner.rows;
    const int smCount = SmCountOrDefault(p.smCount);
    return WithIntDecodeKey(p, [&](auto sample, auto alpha) {
        using SampleT = TypeOf<decltype(sample)>;
        return mono ? LaunchStream<SampleT, 1 + alpha(), true>(sp, smCount, stream) : LaunchStream<SampleT, 3 + alpha(), false>(sp, smCount, stream);
    });
}

cudaError_t LaunchDecodeYccInt(const DecodeParams& p, Interior inner, void* streamHandle)
{
    cudaStream_t stream = static_cast<cudaStream_t>(streamHandle);
    IntDecodeParams fp = IntDecodeShared(p);
    for (int k = 0; k < 4; ++k)
    {
        fp.plane[k] = static_cast<const uint8_t*>(p.plane[k]);
        fp.planeStride[k] = p.planeStride[k];
    }
    fp.rows = static_cast<uint8_t*>(p.rows);
    fp.rowStride = p.rowStride;
    fp.width = inner.width;
    fp.rowCount = inner.rows;
    const int smCount = SmCountOrDefault(p.smCount);
    return WithYccIntKey(p, [&](auto sample, auto alpha, auto xs, auto ys, auto source) {
        return LaunchOne<TypeOf<decltype(sample)>, xs(), ys(), alpha(), source()>(fp, smCount, stream);
    });
}

} // namespace avifgpu
