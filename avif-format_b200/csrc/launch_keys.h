// launch_keys.h -- which instantiation of a tuned kernel a description takes, decided once per kernel family.
//
// A picker reads the description fields that make up its family's key, turns them into compile-time tags and calls `f`
// with them; it is the only code that reads those fields for that purpose.  The single-image launcher and the batched
// launcher of a family (kernels_batch.cu) both call the family's picker and differ only in what `f` launches: which
// kernel, with which grid, shared bytes and parameter object.  Host code only.
#ifndef AVIFGPU_LAUNCH_KEYS_H
#define AVIFGPU_LAUNCH_KEYS_H

#include <type_traits>

#include "kernel_params.h"

namespace avifgpu
{

// Tags: Int<V>{}() is V in a constant expression; TypeOf<decltype(tag)> is the T of a Type<T> tag.
template <int V>
using Int = std::integral_constant<int, V>;
template <typename T>
struct Type
{
    using type = T;
};
template <typename Tag>
using TypeOf = typename Tag::type;

// f(flag): Int<1> when `set`, else Int<0>.
template <typename F>
auto WithFlag(bool set, F&& f)
{
    return set ? f(Int<1>{}) : f(Int<0>{});
}

// f(XS, YS): the chroma shifts -- 4:2:0 (1, 1), 4:2:2 (1, 0), anything else 4:4:4 (0, 0).
template <typename F>
auto WithChroma(int xs, int ys, F&& f)
{
    if (xs == 1 && ys == 1) return f(Int<1>{}, Int<1>{});
    if (xs == 1) return f(Int<1>{}, Int<0>{});
    return f(Int<0>{}, Int<0>{});
}

// f(LAYOUT): avifgpu_source_layout bits -- the planes a YCbCr decode reads (SOURCE) or a planar encode writes (DEST):
// interleaved chroma (1), MSB-aligned samples (2), both (3) or libheif's planar, low-bit layout (0).
template <typename F>
auto WithLayout(int layout, F&& f)
{
    if (SourceInterleaved(layout) && SourceMsbAligned(layout)) return f(Int<AVIFGPU_SOURCE_CHROMA_INTERLEAVED | AVIFGPU_SOURCE_MSB_ALIGNED>{});
    if (SourceMsbAligned(layout)) return f(Int<AVIFGPU_SOURCE_MSB_ALIGNED>{});
    if (SourceInterleaved(layout)) return f(Int<AVIFGPU_SOURCE_CHROMA_INTERLEAVED>{});
    return f(Int<AVIFGPU_SOURCE_PLANAR>{});
}

// f(HostT): the sample type of an integer host -- uint16_t for 16 bits, uint8_t for anything else.
template <typename F>
auto WithIntHost(int hostDepth, F&& f)
{
    return hostDepth == 16 ? f(Type<uint16_t>{}) : f(Type<uint8_t>{});
}

// f(PlaneT, HostT): the generic kernels' plane and host sample types -- 8-bit hosts read and write 8-bit planes, 16-bit
// hosts 16-bit ones, and anything else is the 32-bit float host beside 16-bit planes.  The generic encode kernels take HostT.
template <typename F>
auto WithHostDepth(int hostDepth, F&& f)
{
    if (hostDepth == 8) return f(Type<uint8_t>{}, Type<uint8_t>{});
    if (hostDepth == 16) return f(Type<uint16_t>{}, Type<uint16_t>{});
    return f(Type<uint16_t>{}, Type<float>{});
}

// Integer planar encode (EncodeRgbIntPlanarKernel, EncodeRgbIntBatchKernel).
// f(HostT, PlaneT, CHANNELS, PREMULTIPLY, XS, YS, DEST): host depth x plane depth (16-bit planes above 8 bits) x channels /
// premultiply (3, 4 straight, 4 premultiplied) x chroma x destination layout.  8-bit planes are never MSB-aligned
// (ValidateEncodeDesc), so they take DEST 0 or 1 only.
template <typename F>
auto WithRgbIntKey(const EncodeParams& d, int hostDepth, F&& f)
{
    return WithIntHost(hostDepth, [&](auto host) {
        const auto withPlane = [&](auto plane) {
            const auto withChannels = [&](auto channels, auto premultiply) {
                return WithChroma(d.xs, d.ys, [&](auto xs, auto ys) {
                    const auto withDest = [&](auto dest) { return f(host, plane, channels, premultiply, xs, ys, dest); };
                    if constexpr (sizeof(TypeOf<decltype(plane)>) == 1)
                    {
                        return WithFlag(SourceInterleaved(d.destLayout), withDest);
                    }
                    else
                    {
                        return WithLayout(d.destLayout, withDest);
                    }
                });
            };
            if (d.channels == 4 && d.premultiply) return withChannels(Int<4>{}, Int<1>{});
            if (d.channels == 4) return withChannels(Int<4>{}, Int<0>{});
            return withChannels(Int<3>{}, Int<0>{});
        };
        return d.imageDepth > 8 ? withPlane(Type<uint16_t>{}) : withPlane(Type<uint8_t>{});
    });
}

// Light-level float encode interiors (EncodeLightF32BatchKernel).  f(CHANNELS, XS, YS, DEST): RGB (3) or RGBA (4; straight
// or premultiplied is a runtime value, as in the single-image RGBA kernel) x chroma x destination layout.
template <typename F>
auto WithLightF32Key(const EncodeParams& d, F&& f)
{
    const auto withChannels = [&](auto channels) {
        return WithChroma(d.xs, d.ys, [&](auto xs, auto ys) { return WithLayout(d.destLayout, [&](auto dest) { return f(channels, xs, ys, dest); }); });
    };
    return d.channels == 4 ? withChannels(Int<4>{}) : withChannels(Int<3>{});
}

// Decodes into 8/16-bit hosts.  f(SampleT, ALPHA): uint8_t for 8-bit hosts, uint16_t for anything else, x alpha.  The
// planar-RGB kernels (StreamDecodeKernel, DecodePlanarRgbIntBatchKernel) take 3 + ALPHA channels, the monochrome
// instantiations of StreamDecodeKernel 1 + ALPHA.
template <typename F>
auto WithIntDecodeKey(const DecodeParams& d, F&& f)
{
    const auto withSample = [&](auto sample) { return WithFlag(d.hasAlpha != 0, [&](auto alpha) { return f(sample, alpha); }); };
    return d.hostDepth == 8 ? withSample(Type<uint8_t>{}) : withSample(Type<uint16_t>{});
}

// Integer YCbCr decode (DecodeYccToRgbIntKernel, DecodeYccToRgbIntBatchKernel).  f(SampleT, ALPHA, XS, YS, SOURCE): 8-bit
// samples (8-bit hosts) are never MSB-aligned (ValidateDecodeDesc), so they take SOURCE 0 or 1 only.
template <typename F>
auto WithYccIntKey(const DecodeParams& d, F&& f)
{
    return WithIntDecodeKey(d, [&](auto sample, auto alpha) {
        return WithChroma(d.xs, d.ys, [&](auto xs, auto ys) {
            const auto withSource = [&](auto source) { return f(sample, alpha, xs, ys, source); };
            if constexpr (sizeof(TypeOf<decltype(sample)>) == 1)
            {
                return WithFlag(SourceInterleaved(d.sourceLayout), withSource);
            }
            else
            {
                return WithLayout(d.sourceLayout, withSource);
            }
        });
    });
}

// Float YCbCr decode (DecodeYccToRgbF32Kernel, DecodeYccToRgbF32BatchKernel).  f(TRANSFER, FASTDIV, ALPHA, XS, YS, SOURCE):
// PQ with (FASTDIV = 1) or without the context's verified division, HLG, and SMPTE 428 for anything else --
// DecodeFamilyOf leaves these three.
template <typename F>
auto WithYccF32Key(const DecodeParams& d, F&& f)
{
    const auto withTransfer = [&](auto transfer, auto fastDiv) {
        return WithFlag(d.hasAlpha != 0, [&](auto alpha) {
            return WithChroma(d.xs, d.ys, [&](auto xs, auto ys) {
                return WithLayout(d.sourceLayout, [&](auto source) { return f(transfer, fastDiv, alpha, xs, ys, source); });
            });
        });
    };
    if (d.transfer == AVIFGPU_TRANSFER_PQ && d.verifiedPqRatio) return withTransfer(Int<AVIFGPU_TRANSFER_PQ>{}, Int<1>{});
    if (d.transfer == AVIFGPU_TRANSFER_PQ) return withTransfer(Int<AVIFGPU_TRANSFER_PQ>{}, Int<0>{});
    if (d.transfer == AVIFGPU_TRANSFER_HLG) return withTransfer(Int<AVIFGPU_TRANSFER_HLG>{}, Int<0>{});
    return withTransfer(Int<AVIFGPU_TRANSFER_SMPTE428>{}, Int<0>{});
}

// Decodes of one plane at a time into 32-bit hosts (TableDecodeF32Kernel, TableDecodeF32BatchKernel).  f(ALPHA); transfer and
// OOTF are runtime values there.
template <typename F>
auto WithTableF32Key(const DecodeParams& d, F&& f)
{
    return WithFlag(d.hasAlpha != 0, f);
}

} // namespace avifgpu

#endif
