// source_units.cuh -- the tuned YCbCr decode kernels' reads of the sources GPU video decoders write
// (avifgpu_decode_desc.source_layout): Cb, Cr pairs interleaved in one plane (NV12 / P010 / P016 order, Cb first), and
// 16-bit samples whose code sits in the top bits.  Both turn into the registers the planar, low-bit path loads, so the
// conversion after the loads is that path's own code.  The tuned planar encodes write the same layouts
// (avifgpu_encode_desc.dest_layout) with the reverse operations, from the registers the planar stores take.
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

// The reverse, for the encodes' MSB-aligned planes: two codes below 2^depth -> their two samples, for shift = 16 - depth.
// Neither code crosses into the other's half, so one shift of the word moves both.
__device__ __forceinline__ uint32_t CodesToMsbPair(uint32_t pair, uint32_t shift) { return pair << shift; }

// The even (Cb) and odd (Cr) bytes of two words of interleaved 8-bit pairs, four samples to a word.
__device__ __forceinline__ uint32_t EvenBytes(uint32_t a, uint32_t b) { return __byte_perm(a, b, 0x6420); }
__device__ __forceinline__ uint32_t OddBytes(uint32_t a, uint32_t b) { return __byte_perm(a, b, 0x7531); }

// The low (Cb) and high (Cr) halves of two words of interleaved 16-bit pairs, two samples to a word.
__device__ __forceinline__ uint32_t LowHalves(uint32_t a, uint32_t b) { return __byte_perm(a, b, 0x5410); }
__device__ __forceinline__ uint32_t HighHalves(uint32_t a, uint32_t b) { return __byte_perm(a, b, 0x7632); }

// The reverse, for the encodes' interleaved chroma: a Cb word and a Cr word of four 8-bit codes -> the Cb, Cr pairs of
// codes 0-1 (LowPairs) and 2-3 (HighPairs); for words of two 16-bit codes, LowHalves / HighHalves above pair them.
__device__ __forceinline__ uint32_t LowPairs(uint32_t cb, uint32_t cr) { return __byte_perm(cb, cr, 0x5140); }
__device__ __forceinline__ uint32_t HighPairs(uint32_t cb, uint32_t cr) { return __byte_perm(cb, cr, 0x7362); }

} // namespace
} // namespace avifgpu

#endif
