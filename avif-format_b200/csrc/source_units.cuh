// source_units.cuh -- the tuned YCbCr decode kernels' reads of the sources GPU video decoders write
// (avifgpu_decode_desc.source_layout): Cb, Cr pairs interleaved in one plane (NV12 / P010 / P016 order, Cb first), and
// 16-bit samples whose code sits in the top bits.  Both turn into the registers the planar, low-bit path loads, so the
// conversion after the loads is that path's own code.
#ifndef AVIFGPU_SOURCE_UNITS_CUH
#define AVIFGPU_SOURCE_UNITS_CUH

#include <stdint.h>

#include <cuda_runtime.h>

namespace avifgpu
{
namespace
{

// Two MSB-aligned 16-bit samples -> their two codes, for shift = 16 - depth: each half moves down, and the bits that would
// cross from the upper half into the lower one are masked off.  Whatever the low bits held is gone.
__device__ __forceinline__ uint32_t MsbPairToCodes(uint32_t pair, uint32_t shift) { return (pair >> shift) & ((0xffffu >> shift) * 0x10001u); }

// The even (Cb) and odd (Cr) bytes of two words of interleaved 8-bit pairs, four samples to a word.
__device__ __forceinline__ uint32_t EvenBytes(uint32_t a, uint32_t b) { return __byte_perm(a, b, 0x6420); }
__device__ __forceinline__ uint32_t OddBytes(uint32_t a, uint32_t b) { return __byte_perm(a, b, 0x7531); }

// The low (Cb) and high (Cr) halves of two words of interleaved 16-bit pairs, two samples to a word.
__device__ __forceinline__ uint32_t LowHalves(uint32_t a, uint32_t b) { return __byte_perm(a, b, 0x5410); }
__device__ __forceinline__ uint32_t HighHalves(uint32_t a, uint32_t b) { return __byte_perm(a, b, 0x7632); }

} // namespace
} // namespace avifgpu

#endif
