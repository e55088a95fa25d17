// kernels_fast_decode_table.cu -- float hosts reading images whose samples decode one plane at a time: planar RGB
// (ReadHeifImageRGBThirtyTwoBit's RGB branch, ReadHeifImage.cpp:949-1178) and monochrome
// (ReadHeifImageGrayThirtyTwoBit, ReadHeifImage.cpp:863-947 driving DecodeY16RowToGray32 / ...GrayAlpha32,
// YuvDecode.cpp:199-279), 10 / 12-bit.
//
// There the whole per-sample chain -- unorm -> float table, then PQToLinear / HLGToLinear / SMPTE428ToLinear -- is a
// function of ONE code, so every CTA evaluates it once per code with the exact (glibc-identical) device libm into a
// shared-memory table (2^depth floats: 4096 exact evaluations per CTA against ~200 000 pixels it then converts) and the
// pixel loop is loads, look-ups and stores: HBM-bound (6 + 12 bytes per pixel for RGB -> RGB32f) instead of
// 6 powf per pixel.  What cannot be tabulated stays per pixel and exact: the HLG OOTF (one powf of the pixel's luma,
// ColorTransfer.cpp:192-205) and the integer-domain un-premultiplication the reference applies BEFORE the table
// (ReadHeifImage.cpp:1049-1066, YuvDecode.cpp:247-260).
// A thread converts 8 adjacent pixels: one 128-bit load per plane, 128-bit stores.
#include "float_units.cuh"
#include "group_walk.cuh"
#include "kernel_params.h"
#include "launch_keys.h"
#include "../../include/avifgpu.h"

#include <cuda_runtime.h>

namespace avifgpu
{

using namespace avifpix;
using avifmath::LibmTables;

namespace
{

// COLOURS 3 (planar RGB) or 1 (monochrome); ALPHA adds the alpha plane as the last host channel.
template <int COLOURS, int ALPHA>
__global__ void __launch_bounds__(kTableThreads) TableDecodeF32Kernel(const TableDecodeParams p)
{
    extern __shared__ __align__(16) uint8_t sharedBytes[];
    const CodeTables tables = StageCodeTables<COLOURS, ALPHA>(sharedBytes, p);
    const float maxCodeFloat = static_cast<float>(p.maxCode);
    for (GroupWalk walk(static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x, static_cast<long long>(gridDim.x) * blockDim.x, p.groupsPerRow, p.rowCount);
         walk.Inside(p.rowCount); walk.Advance(p.rowCount))
    {
        TableDecodeGroup<COLOURS, ALPHA>(p, tables, maxCodeFloat, walk.row, static_cast<long long>(walk.column) * 8);
    }
}

template <int COLOURS, int ALPHA>
cudaError_t LaunchTable(const TableDecodeParams& tp, int smCount, cudaStream_t stream)
{
    const long long groups = static_cast<long long>(tp.groupsPerRow) * tp.rowCount;
    const size_t shared = CodeTableBytes(tp.bitDepth, ALPHA != 0);
    // each CTA pays for its own table: exactly as many as are resident at once (4 at 52 registers, 8 at 32), long-lived
    const long long cap = CodeTableGridCap(TableDecodeF32Kernel<COLOURS, ALPHA>, shared, smCount);
    TableDecodeF32Kernel<COLOURS, ALPHA><<<GridFor((groups + kTableThreads - 1) / kTableThreads, cap), kTableThreads, shared, stream>>>(tp);
    return cudaGetLastError();
}

} // namespace

// Monochrome and planar-RGB images for the float hosts.
cudaError_t LaunchDecodeTable(const DecodeParams& p, Interior inner, void* streamHandle)
{
    cudaStream_t stream = static_cast<cudaStream_t>(streamHandle);
    const bool mono = p.colorspace == AVIFGPU_COLORSPACE_MONOCHROME;
    TableDecodeParams tp = TableDecodeDescription(p);
    for (int k = 0; k < 4; ++k)
    {
        tp.plane[k] = static_cast<const uint8_t*>(p.plane[k]);
        tp.planeStride[k] = p.planeStride[k];
    }
    tp.rows = static_cast<uint8_t*>(p.rows);
    tp.rowStride = p.rowStride;
    tp.groupsPerRow = inner.width / 8;
    tp.rowCount = inner.rows;
    const int smCount = SmCountOrDefault(p.smCount);
    return WithTableF32Key(p, [&](auto alpha) {
        return mono ? LaunchTable<1, alpha()>(tp, smCount, stream) : LaunchTable<3, alpha()>(tp, smCount, stream);
    });
}

} // namespace avifgpu
