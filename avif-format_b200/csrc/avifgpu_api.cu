// avifgpu_api.cu -- the extern "C" surface declared in include/avifgpu.h: context, validation, PCIe staging for
// the host-pointer entry points, and dispatch to the kernels.  No CPU fallback anywhere: every entry point that
// converts pixels launches a CUDA kernel or fails.
#include "../../include/avifgpu.h"

#include "batch_plan.h"
#include "curve_tables.h"
#include "host_params.h"
#include "kernel_params.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <new>
#include <string>
#include <thread>
#include <vector>


namespace avifgpu
{
namespace
{
    thread_local int g_launchFailure = 0; // cudaError_t of the last failed launch on this thread, 0 = none
}

int ReportLaunchFailure(int cudaErrorCode)
{
    g_launchFailure = cudaErrorCode;
    return AVIFGPU_ERR_CUDA;
}

static int TakeLaunchFailure()
{
    const int code = g_launchFailure;
    g_launchFailure = 0;
    return code;
}

int LaunchEncode(const EncodeParams& params, int hostDepth, void* stream, const LightSink* light)
{
    EncodeFamily family = EncodeFamilyOf(params, hostDepth);
    if (light != nullptr && (family == EncodeFamily::RgbF32Interleaved || family == EncodeFamily::RgbF32Flat) && !FlatCompactFits(*params.curveTable))
    {
        family = EncodeFamily::Generic; // the light-level flat kernels have the compact table only, which every PQ table built so far has
    }
    const Interior inner = EncodeBlockInterior(family, params, hostDepth);
    if (inner.width == 0)
    {
        return LaunchEncodeGeneric(params, hostDepth, stream, light);
    }
    cudaError_t e;
    switch (family)
    {
    case EncodeFamily::RgbF32Interleaved: e = LaunchEncodeRgbF32Interleaved(params, inner, stream, light); break;
    case EncodeFamily::Gray16Lut: e = LaunchEncodeGray16Lut(params, inner, stream); break;
    case EncodeFamily::GrayInt: e = LaunchEncodeGrayInt(params, hostDepth, inner, stream); break;
    case EncodeFamily::RgbInt: e = LaunchEncodeRgbInt(params, hostDepth, inner, stream); break;
    case EncodeFamily::GrayF32: e = LaunchEncodeGrayF32(params, inner, stream, light); break;
    default: e = LaunchEncodeRgbF32Planar(family, params, inner, stream, light); break; // RgbF32Flat, RgbaF32Flat, RgbF32Clip
    }
    return CompleteEncode(e, params, hostDepth, inner.width, inner.rows, stream, light);
}

int LaunchDecode(const DecodeParams& params, void* stream)
{
    const DecodeFamily family = DecodeFamilyOf(params);
    const Interior inner = DecodeBlockInterior(family, params);
    if (inner.width == 0)
    {
        return LaunchDecodeGeneric(params, stream);
    }
    cudaError_t e;
    switch (family)
    {
    case DecodeFamily::YccF32: e = LaunchDecodeYccF32(params, inner, stream); break;
    case DecodeFamily::YccInt: e = LaunchDecodeYccInt(params, inner, stream); break;
    case DecodeFamily::MonoInt:
    case DecodeFamily::PlanarRgbInt: e = LaunchDecodeStream(params, inner, stream); break;
    default: e = LaunchDecodeTable(params, inner, stream); break; // MonoF32, PlanarRgbF32
    }
    return CompleteDecode(e, params, inner.width, inner.rows, stream);
}
} // namespace avifgpu

using namespace avifgpu;

namespace
{
    thread_local std::string g_creationError;

    // A host-pointer call is cut into row-block slices that rotate through this many pipeline slots (stream + staging
    // buffers each), so that the H2D copy of slice i+1, the kernel of slice i and the D2H copy of slice i-1 overlap.
    // Two slots keep both copy engines busy; the third lets the host thread fill / drain a pinned bounce buffer
    // (pageable caller memory) while the other two are on the wire.
    constexpr int kPipelineStreams = 3;
    // A slot stages each plane k in its buffers k and the host rows in buffer kRowsBuffer.
    constexpr int kRowsBuffer = AVIFGPU_MAX_PLANES;
    constexpr int kSlotBuffers = AVIFGPU_MAX_PLANES + 1;

    // `rows` rows of `payload` bytes from `source` to `target`.
    struct RowCopy
    {
        uint8_t* target;
        int64_t targetStride;
        const uint8_t* source;
        int64_t sourceStride;
        int64_t payload;
        int rows;
    };
}

struct avifgpu_context
{
    int device = -1;
    cudaEvent_t callRowsConsumed[2] = {};            // every H2D of an asynchronous encode call has finished (calls alternate between the two)
    int64_t asyncEncodeCalls = 0;
    bool previousCallRowsPending = false;            // callRowsConsumed[(asyncEncodeCalls - 1) & 1] guards caller memory still on the wire

    struct Buffer
    {
        void* ptr = nullptr;
        size_t bytes = 0;
    };
    // One pipeline slot of the host-pointer entry points.  Its staging buffers are grow-only.
    struct Slot
    {
        cudaStream_t stream = nullptr;
        cudaEvent_t sliceDone = nullptr;
        cudaEvent_t rowsConsumed = nullptr; // encode: the slot's H2D of caller rows has finished
        bool busy = false;
        int64_t ticket = 0;
        Buffer device[kSlotBuffers];
        Buffer pinned[kSlotBuffers]; // bounce buffers for pageable caller memory
        // What the slot still owes the caller once its stream has drained: owed[b] copies pinned[b] into pageable caller
        // memory (libheif's planes on the encode side, pageable host rows on the decode side); rows == 0 when nothing.
        RowCopy owed[kSlotBuffers] = {};
        // The light-level host encode's per-slice statistic: a device accumulator and its pinned mirror, allocated at the
        // first light-level slice.  owedLight is the caller's accumulator the mirror still has to be merged into (a debt
        // like owed[], paid once the slice is done), nullptr when nothing.
        avifgpu_light_level* lightDevice = nullptr;
        avifgpu_light_level* lightMirror = nullptr;
        avifgpu_light_level* owedLight = nullptr;
    };
    Slot slots[kPipelineStreams];
    int nextSlot = 0;
    int64_t lastTicket = 0;       // ticket of the most recent host-pointer call
    std::string lastError;
    int64_t launches = 0;
    int smCount = 0;

    Buffer transferScratch[2];
    std::vector<CurveTable*> curveTables; // exact step tables, built per (curve, param, depth): explicitly or once they pay off
    struct PendingTable
    {
        int curve, param, depth;
        int64_t pixels; // converted with the exact kernel so far
    };
    std::vector<PendingTable> pendingTables;
    int64_t tableAutoBuildPixels = AVIFGPU_TABLE_AUTOBUILD_DEFAULT;
    struct Gray16Lut
    {
        int depth = 0;
        int smpte428 = 0;
        uint16_t* device = nullptr;
    };
    std::vector<Gray16Lut> gray16Luts;
    uint32_t* lightLevels[3] = {}; // level(k) of every code (light_level.cuh) at image depth 8 / 10 / 12, made with the depth's first PQ step table
    int premultiplyState[3] = { -1, -1, -1 }; // image depth 8 / 10 / 12: -1 not checked yet, 0 keep the reference sequence, 1 fast form verified
    // The first-use helpers below take `capturing`: the call is being recorded into a CUDA graph, where nothing but kernel
    // launches on the caller's stream may happen.  What is not prepared yet then answers "not verified" / nullptr for
    // this call only -- the path that needs no preparation, with bit-identical outputs -- and nothing is cached.  (The
    // verify sweeps, LUT and table builds allocate and synchronise; BuildCurveTable's cudaGetDeviceProperties is only
    // reached from a build.)
    //
    // A captured graph holds the device pointers of the step tables and Gray16 LUTs it was recorded with: those are only
    // ever added to (never freed, moved or rebuilt) until avifgpu_destroy.

    // The tuned integer encode kernel premultiplies with a 6-instruction form, but only after it has been compared with
    // PremultiplyColor's own sequence for every (colour, alpha) code pair of the depth, on this device.
    int VerifiedPremultiply(const avifgpu_encode_desc& d, bool capturing)
    {
        if (d.alpha_state != AVIFGPU_ALPHA_PREMULTIPLIED || d.host_depth == 32 || d.host_channels != 4 || d.layout != AVIFGPU_LAYOUT_PLANAR_YCBCR)
        {
            return 0;
        }
        const int slot = d.image_bit_depth == 8 ? 0 : d.image_bit_depth == 10 ? 1 : 2;
        if (premultiplyState[slot] < 0)
        {
            if (capturing)
            {
                return 0;
            }
            premultiplyState[slot] = VerifyFastPremultiply((1u << d.image_bit_depth) - 1u, slots[0].stream) == 0 ? 1 : 0;
            launches += 1;
        }
        return premultiplyState[slot];
    }
    int hlgDivisionState = -1; // -1 not checked yet, 0 keep IEEE divisions, 1 fast divisions verified exact

    // HLG decode replaces two constant divisions by a 3-instruction form, but only after comparing it with the
    // IEEE division over every numerator the call sites can produce, on this device.
    int VerifiedHlgDivisions(bool capturing)
    {
        if (hlgDivisionState < 0)
        {
            if (capturing)
            {
                return 0;
            }
            const long long disagreements = VerifyHlgDivisions(slots[0].stream);
            hlgDivisionState = disagreements == 0 ? 1 : 0;
            launches += 1;
        }
        return hlgDivisionState;
    }

    // The quotient inside PQToLinear (ColorTransfer.cpp:110-112): the tuned float decode kernel uses a branch-free division
    // once it has been compared with the IEEE one for every value the quotient's operands can take, on this device.
    int pqRatioState = -1;
    int VerifiedPqRatio(bool capturing)
    {
        if (pqRatioState < 0)
        {
            if (capturing)
            {
                return 0;
            }
            const long long disagreements = VerifyPqRatio(slots[0].stream);
            pqRatioState = disagreements == 0 ? 1 : 0;
            launches += 1;
        }
        return pqRatioState;
    }

    // YuvDecode.cpp:308 divides by the per-image constant kg; the tuned decode kernels use a 3-instruction form after
    // it has been compared with the IEEE division for every (Cb, Cr) code pair of the configuration, on this device.
    struct GreenDivision
    {
        avifpix::InverseMatrix matrix;
        avifpix::RangeParams range;
        uint32_t maxCode;
        int state;
    };
    std::vector<GreenDivision> greenDivisions;
    int VerifiedGreenDivision(const DecodeParams& p, bool capturing)
    {
        if (p.colorspace != AVIFGPU_COLORSPACE_YCBCR || p.bitDepth > 12)
        {
            return 0;
        }
        for (const GreenDivision& g : greenDivisions)
        {
            if (std::memcmp(&g.matrix, &p.matrix, sizeof(g.matrix)) == 0 && std::memcmp(&g.range, &p.range, sizeof(g.range)) == 0 && g.maxCode == p.maxCode)
            {
                return g.state;
            }
        }
        if (capturing)
        {
            return 0;
        }
        GreenDivision g{};
        g.matrix = p.matrix;
        g.range = p.range;
        g.maxCode = p.maxCode;
        g.state = VerifyGreenDivision(p, slots[0].stream) == 0 ? 1 : 0;
        launches += 1;
        greenDivisions.push_back(g);
        return g.state;
    }

    // The 65536-entry code table of a Gray16 host configuration (built on the device on first use), or nullptr.
    const uint16_t* Gray16LutFor(const avifgpu_encode_desc& d, bool capturing)
    {
        if (d.host_depth != 16 || d.host_channels != 1 || d.layout != AVIFGPU_LAYOUT_REFERENCE || d.image_bit_depth <= 8)
        {
            return nullptr;
        }
        const int smpte428 = d.gray16_curve == AVIFGPU_GRAY16_SMPTE428 ? 1 : 0;
        for (const Gray16Lut& l : gray16Luts)
        {
            if (l.depth == d.image_bit_depth && l.smpte428 == smpte428)
            {
                return l.device;
            }
        }
        if (capturing)
        {
            return nullptr;
        }
        Gray16Lut lut;
        lut.depth = d.image_bit_depth;
        lut.smpte428 = smpte428;
        if (cudaMalloc(&lut.device, 65536 * sizeof(uint16_t)) != cudaSuccess)
        {
            cudaGetLastError();
            return nullptr;
        }
        if (BuildGray16Lut(lut.device, smpte428, (1u << d.image_bit_depth) - 1u, slots[0].stream) != cudaSuccess ||
            cudaStreamSynchronize(slots[0].stream) != cudaSuccess)
        {
            cudaGetLastError();
            cudaFree(lut.device);
            return nullptr;
        }
        launches += 1;
        gray16Luts.push_back(lut);
        return lut.device;
    }

    // The verified step table for a float-host encode description, or nullptr when the description does not use
    // one / the table could not be verified / building it has not paid off yet (then the generic exact kernel serves
    // the call).  `pixels` = the size of the call that asks; `force` = avifgpu_prepare_encode.  A capturing call neither
    // builds a table nor counts its pixels towards one.
    CurveTable* CurveTableFor(const avifgpu_encode_desc& d, int64_t pixels, bool force, bool capturing)
    {
        if (d.host_depth != 32 || d.image_bit_depth > 12)
        {
            return nullptr;
        }
        int curve;
        int param = 0;
        if (d.transfer == AVIFGPU_TRANSFER_PQ)
        {
            curve = kCurveLinearToPQ;
            param = d.pq_peak_nits;
        }
        else if (d.transfer == AVIFGPU_TRANSFER_SMPTE428)
        {
            curve = kCurveLinearToSMPTE428;
        }
        else if (d.transfer == AVIFGPU_TRANSFER_HLG)
        {
            curve = kCurveLinearToHLG;
        }
        else
        {
            return nullptr;
        }
        for (CurveTable* t : curveTables)
        {
            if (t->curve == curve && t->param == param && t->depth == d.image_bit_depth)
            {
                return t;
            }
        }
        if (capturing)
        {
            return nullptr;
        }
        if (!force)
        {
            // ~40 ms of sweeps buy a ~7x faster kernel: worth it once a configuration has seen enough pixels
            PendingTable* pending = nullptr;
            for (PendingTable& candidate : pendingTables)
            {
                if (candidate.curve == curve && candidate.param == param && candidate.depth == d.image_bit_depth)
                {
                    pending = &candidate;
                }
            }
            if (pending == nullptr)
            {
                pendingTables.push_back(PendingTable{ curve, param, d.image_bit_depth, 0 });
                pending = &pendingTables.back();
            }
            pending->pixels += pixels;
            if (tableAutoBuildPixels < 0 || pending->pixels <= tableAutoBuildPixels)
            {
                return nullptr;
            }
        }
        CurveTable* t = new (std::nothrow) CurveTable();
        if (t == nullptr)
        {
            return nullptr;
        }
        BuildCurveTable(curve, param, d.image_bit_depth, slots[0].stream, t);
        launches += t->stats.sweptInputs ? (t->stats.bandBitmapBytes ? 3 : 2) : 0; // sweep, (band bitmap,) verify
        curveTables.push_back(t);
        if (curve == kCurveLinearToPQ)
        {
            BuildLightLevels(d.image_bit_depth); // the light-level call's tuned kernels run wherever a PQ step table is
        }
        return t;
    }

    // The level table of an image depth (host arithmetic, one copy), once; a failure leaves it absent, and the light-level
    // call then takes the generic kernel.
    void BuildLightLevels(int depth)
    {
        uint32_t*& levels = lightLevels[depth == 8 ? 0 : depth == 10 ? 1 : 2];
        if (levels != nullptr)
        {
            return;
        }
        std::vector<uint32_t> host(static_cast<size_t>(1) << depth);
        const avifmath::LibmTables tables = avifmath::HostLibmTables();
        const float maxCodeFloat = static_cast<float>(host.size() - 1);
        for (size_t k = 0; k < host.size(); ++k)
        {
            host[k] = LightLevelOf(static_cast<uint32_t>(k), maxCodeFloat, tables);
        }
        uint32_t* device = nullptr;
        const size_t bytes = host.size() * sizeof(uint32_t);
        if (cudaMalloc(&device, bytes) != cudaSuccess)
        {
            cudaGetLastError();
            return;
        }
        if (cudaMemcpyAsync(device, host.data(), bytes, cudaMemcpyHostToDevice, slots[0].stream) != cudaSuccess ||
            cudaStreamSynchronize(slots[0].stream) != cudaSuccess)
        {
            cudaGetLastError();
            cudaFree(device);
            return;
        }
        levels = device;
    }

    // The first-use state an encode call reads: step table, Gray16 LUT, premultiply check.
    void FirstUseEncode(const avifgpu_encode_desc& d, int64_t pixels, bool capturing, EncodeParams* p)
    {
        if (CurveTable* table = CurveTableFor(d, pixels, false, capturing))
        {
            p->curveTable = table->valid ? &table->view : nullptr;
        }
        p->gray16Lut = Gray16LutFor(d, capturing);
        p->verifiedPremultiply = VerifiedPremultiply(d, capturing);
    }

    // The first-use state a decode call reads: the verified HLG, green-channel and PQ divisions.
    void FirstUseDecode(const avifgpu_decode_desc& d, int32_t transfer, bool capturing, DecodeParams* p)
    {
        p->verifiedHlgDivisions = (d.host_depth == 32 && transfer == AVIFGPU_TRANSFER_HLG) ? VerifiedHlgDivisions(capturing) : 0;
        p->verifiedGreenDivision = VerifiedGreenDivision(*p, capturing);
        p->verifiedPqRatio = (d.host_depth == 32 && transfer == AVIFGPU_TRANSFER_PQ && d.colorspace == AVIFGPU_COLORSPACE_YCBCR) ? VerifiedPqRatio(capturing) : 0;
    }

    int Fail(int status, const std::string& message)
    {
        lastError = message;
        return status;
    }

    // A launcher returned a negative status: report the CUDA error it recorded (it has already cleared CUDA's own
    // slot), after draining the pipeline streams so that no copy of an earlier slice is still writing into caller memory
    // when the entry point returns.  A capturing call synchronises nothing: ending the capture is the caller's business.
    int LaunchFailed(int status, const char* what, bool capturing = false)
    {
        const int code = TakeLaunchFailure();
        for (const Slot& slot : slots)
        {
            if (slot.stream && !capturing)
            {
                cudaStreamSynchronize(slot.stream);
            }
        }
        cudaGetLastError();
        lastError = std::string(what) + " failed: " + (code != 0 ? cudaGetErrorString(static_cast<cudaError_t>(code)) : avifgpu_status_string(status));
        return status;
    }

    int Cuda(cudaError_t e, const char* what)
    {
        if (e == cudaSuccess)
        {
            return AVIFGPU_OK;
        }
        lastError = std::string(what) + ": " + cudaGetErrorString(e);
        return (e == cudaErrorMemoryAllocation) ? AVIFGPU_ERR_OOM : AVIFGPU_ERR_CUDA;
    }

    int EnsureDevice(Buffer& b, size_t bytes)
    {
        if (b.bytes >= bytes)
        {
            return AVIFGPU_OK;
        }
        if (b.ptr)
        {
            cudaFree(b.ptr);
            b.ptr = nullptr;
            b.bytes = 0;
        }
        const size_t rounded = ((bytes + (1u << 20) - 1) >> 20) << 20;
        const int status = Cuda(cudaMalloc(&b.ptr, rounded), "cudaMalloc");
        if (status == AVIFGPU_OK)
        {
            b.bytes = rounded;
        }
        return status;
    }

    int EnsurePinned(Buffer& b, size_t bytes)
    {
        if (b.bytes >= bytes)
        {
            return AVIFGPU_OK;
        }
        if (b.ptr)
        {
            cudaFreeHost(b.ptr);
            b.ptr = nullptr;
            b.bytes = 0;
        }
        const size_t rounded = ((bytes + (1u << 20) - 1) >> 20) << 20;
        const int status = Cuda(cudaHostAlloc(&b.ptr, rounded, cudaHostAllocDefault), "cudaHostAlloc");
        if (status == AVIFGPU_OK)
        {
            b.bytes = rounded;
        }
        return status;
    }
};

static int RetireThrough(avifgpu_context* ctx, int64_t ticket);

namespace
{
    bool IsPinned(const void* p)
    {
        cudaPointerAttributes attr{};
        if (cudaPointerGetAttributes(&attr, p) != cudaSuccess)
        {
            cudaGetLastError();
            return false;
        }
        return attr.type == cudaMemoryTypeHost;
    }

    struct DeviceGuard
    {
        int previous = -1;
        explicit DeviceGuard(int device)
        {
            cudaGetDevice(&previous);
            if (previous != device)
            {
                cudaSetDevice(device);
            }
            else
            {
                previous = -1;
            }
        }
        ~DeviceGuard()
        {
            if (previous >= 0)
            {
                cudaSetDevice(previous);
            }
        }
    };

    // Whether work enqueued on `stream` is being recorded into a CUDA graph (in any capture mode).  The query itself
    // fails for the legacy NULL stream while a blocking stream of the device is being captured.
    int QueryCapture(avifgpu_context* ctx, void* stream, bool* capturing)
    {
        cudaStreamCaptureStatus status = cudaStreamCaptureStatusNone;
        const cudaError_t e = cudaStreamIsCapturing(static_cast<cudaStream_t>(stream), &status);
        *capturing = status != cudaStreamCaptureStatusNone;
        if (e != cudaSuccess)
        {
            cudaGetLastError();
            return ctx->Fail(AVIFGPU_ERR_CUDA, std::string("cudaStreamIsCapturing: ") + cudaGetErrorString(e));
        }
        return AVIFGPU_OK;
    }

    int CheckBlock(avifgpu_context* ctx, int height, int ys, int y0, int nrows)
    {
        if (y0 < 0 || nrows < 0 || y0 > height || nrows > height - y0)
        {
            return ctx->Fail(AVIFGPU_ERR_BAD_PARAM, "row block outside the image");
        }
        if (ys && (y0 & 1))
        {
            return ctx->Fail(AVIFGPU_ERR_BAD_PARAM, "4:2:0 row blocks must start on an even row");
        }
        if (ys && (nrows & 1) && y0 + nrows != height)
        {
            return ctx->Fail(AVIFGPU_ERR_BAD_PARAM, "4:2:0 row blocks must have an even height unless they end the image");
        }
        return AVIFGPU_OK;
    }
}

// ---- context ------------------------------------------------------------------------------------------------

extern "C" {

AVIFGPU_EXPORT int avifgpu_api_version(void) { return AVIFGPU_API_VERSION; }

AVIFGPU_EXPORT const char* avifgpu_status_string(int status)
{
    switch (status)
    {
    case AVIFGPU_OK: return "ok";
    case AVIFGPU_ERR_BAD_PARAM: return "bad parameter";
    case AVIFGPU_ERR_UNSUPPORTED: return "unsupported";
    case AVIFGPU_ERR_NO_DEVICE: return "no usable CUDA device";
    case AVIFGPU_ERR_CUDA: return "CUDA error";
    case AVIFGPU_ERR_OOM: return "out of memory";
    case AVIFGPU_ERR_CANCELED: return "canceled";
    default: return "unknown status";
    }
}

AVIFGPU_EXPORT int avifgpu_create(int device_ordinal, avifgpu_context** out_ctx)
{
    if (out_ctx == nullptr)
    {
        g_creationError = "out_ctx is NULL";
        return AVIFGPU_ERR_BAD_PARAM;
    }
    *out_ctx = nullptr;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count <= 0)
    {
        cudaGetLastError();
        g_creationError = std::string("no CUDA device: ") + (e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0") +
                          " (this library has no CPU fallback)";
        return AVIFGPU_ERR_NO_DEVICE;
    }
    if (device_ordinal < 0 || device_ordinal >= count)
    {
        g_creationError = "device ordinal out of range";
        return AVIFGPU_ERR_BAD_PARAM;
    }
    cudaDeviceProp prop{};
    e = cudaGetDeviceProperties(&prop, device_ordinal);
    if (e != cudaSuccess)
    {
        g_creationError = std::string("cudaGetDeviceProperties: ") + cudaGetErrorString(e);
        return AVIFGPU_ERR_NO_DEVICE;
    }
    if (prop.major != 9 || prop.minor != 0)
    {
        char text[160];
        std::snprintf(text, sizeof(text), "device %d is sm_%d%d; this library ships sm_90a code only", device_ordinal, prop.major, prop.minor);
        g_creationError = text;
        return AVIFGPU_ERR_NO_DEVICE;
    }
    avifgpu_context* ctx = new (std::nothrow) avifgpu_context();
    if (ctx == nullptr)
    {
        g_creationError = "out of host memory";
        return AVIFGPU_ERR_OOM;
    }
    ctx->device = device_ordinal;
    ctx->smCount = prop.multiProcessorCount;
    DeviceGuard guard(device_ordinal);
    for (int i = 0; i < kPipelineStreams; ++i)
    {
        avifgpu_context::Slot& slot = ctx->slots[i];
        if (cudaStreamCreateWithFlags(&slot.stream, cudaStreamNonBlocking) != cudaSuccess ||
            cudaEventCreateWithFlags(&slot.sliceDone, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&slot.rowsConsumed, cudaEventDisableTiming) != cudaSuccess ||
            (i < 2 && cudaEventCreateWithFlags(&ctx->callRowsConsumed[i], cudaEventDisableTiming) != cudaSuccess))
        {
            g_creationError = std::string("stream/event creation failed: ") + cudaGetErrorString(cudaGetLastError());
            avifgpu_destroy(ctx);
            return AVIFGPU_ERR_CUDA;
        }
    }
    *out_ctx = ctx;
    return AVIFGPU_OK;
}

AVIFGPU_EXPORT void avifgpu_destroy(avifgpu_context* ctx)
{
    if (ctx == nullptr)
    {
        return;
    }
    DeviceGuard guard(ctx->device);
    cudaDeviceSynchronize();
    for (int i = 0; i < kPipelineStreams; ++i)
    {
        const avifgpu_context::Slot& slot = ctx->slots[i];
        if (slot.stream) cudaStreamDestroy(slot.stream);
        if (slot.sliceDone) cudaEventDestroy(slot.sliceDone);
        if (slot.rowsConsumed) cudaEventDestroy(slot.rowsConsumed);
        if (i < 2 && ctx->callRowsConsumed[i]) cudaEventDestroy(ctx->callRowsConsumed[i]);
        for (int b = 0; b < kSlotBuffers; ++b)
        {
            if (slot.device[b].ptr) cudaFree(slot.device[b].ptr);
            if (slot.pinned[b].ptr) cudaFreeHost(slot.pinned[b].ptr);
        }
        if (slot.lightDevice) cudaFree(slot.lightDevice);
        if (slot.lightMirror) cudaFreeHost(slot.lightMirror);
    }
    for (auto& b : ctx->transferScratch)
    {
        if (b.ptr) cudaFree(b.ptr);
    }
    for (CurveTable* t : ctx->curveTables)
    {
        FreeCurveTable(t);
        delete t;
    }
    for (auto& l : ctx->gray16Luts)
    {
        cudaFree(l.device);
    }
    for (uint32_t* levels : ctx->lightLevels)
    {
        if (levels) cudaFree(levels);
    }
    delete ctx;
}

AVIFGPU_EXPORT const char* avifgpu_last_error(const avifgpu_context* ctx)
{
    return ctx ? ctx->lastError.c_str() : g_creationError.c_str();
}

AVIFGPU_EXPORT int64_t avifgpu_launch_count(const avifgpu_context* ctx) { return ctx ? ctx->launches : 0; }

AVIFGPU_EXPORT int avifgpu_synchronize(avifgpu_context* ctx)
{
    if (ctx == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    DeviceGuard guard(ctx->device);
    const int status = ctx->Cuda(cudaDeviceSynchronize(), "cudaDeviceSynchronize");
    const int retired = RetireThrough(ctx, ctx->lastTicket); // pays the bounce copies asynchronous calls still owe
    ctx->previousCallRowsPending = false;
    return status != AVIFGPU_OK ? status : retired;
}

AVIFGPU_EXPORT int avifgpu_host_alloc(avifgpu_context* ctx, size_t bytes, void** out_ptr)
{
    if (ctx == nullptr || out_ptr == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    DeviceGuard guard(ctx->device);
    *out_ptr = nullptr;
    return ctx->Cuda(cudaHostAlloc(out_ptr, bytes ? bytes : 1, cudaHostAllocDefault), "cudaHostAlloc");
}

AVIFGPU_EXPORT int avifgpu_host_free(avifgpu_context* ctx, void* ptr)
{
    if (ctx == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    DeviceGuard guard(ctx->device);
    return ctx->Cuda(cudaFreeHost(ptr), "cudaFreeHost");
}

// ---- geometry and parameter derivation (no device needed) -----------------------------------------------------

AVIFGPU_EXPORT int avifgpu_encode_host_col_bytes(const avifgpu_encode_desc* desc)
{
    avifgpu_encode_desc full;
    desc = WidenEncodeDesc(desc, &full);
    return ValidateEncodeDesc(desc, nullptr) == AVIFGPU_OK ? EncodeHostColBytes(*desc) : AVIFGPU_ERR_BAD_PARAM;
}

AVIFGPU_EXPORT int avifgpu_decode_host_col_bytes(const avifgpu_decode_desc* desc)
{
    avifgpu_decode_desc full;
    desc = WidenDecodeDesc(desc, &full);
    int32_t transfer;
    return ValidateDecodeDesc(desc, &transfer, nullptr) == AVIFGPU_OK ? DecodeHostColBytes(*desc) : AVIFGPU_ERR_BAD_PARAM;
}

static int ReportGeometry(const PlaneGeometry& g, int32_t* w, int32_t* h, int32_t* b)
{
    if (w) *w = g.present ? g.widthSamples : 0;
    if (h) *h = g.present ? g.height : 0;
    if (b) *b = g.present ? g.bytesPerSample : 0;
    return g.present ? 1 : 0;
}

AVIFGPU_EXPORT int avifgpu_encode_plane_geometry(const avifgpu_encode_desc* desc, int index, int32_t* w, int32_t* h, int32_t* b)
{
    avifgpu_encode_desc full;
    desc = WidenEncodeDesc(desc, &full);
    const int status = ValidateEncodeDesc(desc, nullptr);
    if (status != AVIFGPU_OK || index < 0 || index >= AVIFGPU_MAX_PLANES)
    {
        ReportGeometry(PlaneGeometry(), w, h, b);
        return status != AVIFGPU_OK ? status : AVIFGPU_ERR_BAD_PARAM;
    }
    return ReportGeometry(EncodePlaneGeometry(*desc, index), w, h, b);
}

AVIFGPU_EXPORT int avifgpu_decode_plane_geometry(const avifgpu_decode_desc* desc, int index, int32_t* w, int32_t* h, int32_t* b)
{
    avifgpu_decode_desc full;
    desc = WidenDecodeDesc(desc, &full);
    int32_t transfer;
    const int status = ValidateDecodeDesc(desc, &transfer, nullptr);
    if (status != AVIFGPU_OK || index < 0 || index >= AVIFGPU_MAX_PLANES)
    {
        ReportGeometry(PlaneGeometry(), w, h, b);
        return status != AVIFGPU_OK ? status : AVIFGPU_ERR_BAD_PARAM;
    }
    return ReportGeometry(DecodePlaneGeometry(*desc, index), w, h, b);
}

AVIFGPU_EXPORT int avifgpu_get_yuv_coefficients(const avifgpu_nclx* nclx, float* out)
{
    if (out == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    GetYuvCoefficients(nclx, out);
    return AVIFGPU_OK;
}

AVIFGPU_EXPORT int avifgpu_get_hlg_luma_coefficients(int32_t color_primaries, float* out)
{
    if (out == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    return GetHlgLumaCoefficients(color_primaries, out) ? AVIFGPU_OK : AVIFGPU_ERR_UNSUPPORTED;
}

AVIFGPU_EXPORT int avifgpu_build_yuv_tables(const avifgpu_nclx* nclx, int32_t bit_depth, int32_t monochrome, float* out_y,
                                            float* out_uv, float* out_alpha)
{
    if (bit_depth != 8 && bit_depth != 10 && bit_depth != 12 && bit_depth != 16)
    {
        return AVIFGPU_ERR_UNSUPPORTED;
    }
    const avifpix::RangeParams range = MakeRangeParams(nclx, bit_depth, monochrome != 0);
    const uint32_t count = 1u << bit_depth;
    for (uint32_t i = 0; i < count; ++i)
    {
        if (out_y) out_y[i] = avifpix::UnormToFloatY(i, range);
        if (out_uv && !monochrome) out_uv[i] = avifpix::UnormToFloatUV(i, range);
        if (out_alpha) out_alpha[i] = avifpix::UnormToFloatPlain(i, range.maxChannelFloat);
    }
    return AVIFGPU_OK;
}

// ---- device-pointer entry points -------------------------------------------------------------------------------

// The level table of the description's image depth, or nullptr when the context has none yet.
static const uint32_t* LightLevelsFor(const avifgpu_context* ctx, const avifgpu_encode_desc& d)
{
    return ctx->lightLevels[d.image_bit_depth == 8 ? 0 : d.image_bit_depth == 10 ? 1 : 2];
}

// The light-level calls' own checks, after the description's: float-host PQ encodes only, and an accumulator.
static int CheckLightLevelCall(avifgpu_context* ctx, const avifgpu_encode_desc& d, const avifgpu_light_level* acc)
{
    if (d.host_depth != 32 || d.transfer != AVIFGPU_TRANSFER_PQ)
    {
        return ctx->Fail(AVIFGPU_ERR_UNSUPPORTED, "the content light level is measured on float-host PQ encodes only");
    }
    if (acc == nullptr)
    {
        return ctx->Fail(AVIFGPU_ERR_BAD_PARAM, "NULL light-level accumulator");
    }
    return AVIFGPU_OK;
}

// The device-pointer encode; `acc` != nullptr: the light-level call, whose description the caller has checked.
static int EncodeRowsDevice(avifgpu_context* ctx, const avifgpu_encode_desc* desc, const void* device_rows, int64_t row_stride_bytes, int32_t y0,
                            int32_t nrows, const avifgpu_planes* device_dst, avifgpu_light_level* acc, void* cuda_stream)
{
    int status;
    if (device_dst == nullptr || (device_rows == nullptr && nrows > 0 && desc->width > 0))
    {
        return ctx->Fail(AVIFGPU_ERR_BAD_PARAM, "NULL buffer");
    }
    EncodeParams p;
    FillEncodeParams(*desc, &p);
    status = CheckBlock(ctx, desc->height, p.ys, y0, nrows);
    if (status != AVIFGPU_OK)
    {
        return status;
    }
    if (nrows == 0 || desc->width == 0)
    {
        return AVIFGPU_OK;
    }
    p.rows = device_rows;
    p.rowStride = row_stride_bytes;
    p.rowCount = nrows;
    for (int k = 0; k < AVIFGPU_MAX_PLANES; ++k)
    {
        const PlaneGeometry g = EncodePlaneGeometry(*desc, k);
        if (!g.present)
        {
            continue;
        }
        if (device_dst->data[k] == nullptr)
        {
            return ctx->Fail(AVIFGPU_ERR_BAD_PARAM, "missing destination plane");
        }
        p.plane[k] = static_cast<uint8_t*>(device_dst->data[k]) + static_cast<int64_t>(y0 >> g.ys) * device_dst->stride[k];
        p.planeStride[k] = device_dst->stride[k];
    }
    DeviceGuard guard(ctx->device);
    bool capturing;
    if ((status = QueryCapture(ctx, cuda_stream, &capturing)) != AVIFGPU_OK)
    {
        return status;
    }
    p.smCount = ctx->smCount;
    ctx->FirstUseEncode(*desc, static_cast<int64_t>(desc->width) * nrows, capturing, &p);
    const LightSink light = { acc, LightLevelsFor(ctx, *desc) };
    if (acc != nullptr && light.levels == nullptr)
    {
        p.curveTable = nullptr; // no level table (not built yet, or its allocation failed): the generic kernel evaluates the levels
    }
    const int launched = LaunchEncode(p, desc->host_depth, cuda_stream, acc != nullptr ? &light : nullptr);
    if (launched < 0)
    {
        return ctx->LaunchFailed(launched, "encode kernel launch", capturing);
    }
    ctx->launches += launched;
    return AVIFGPU_OK;
}

AVIFGPU_EXPORT int avifgpu_encode_rows_device(avifgpu_context* ctx, const avifgpu_encode_desc* desc, const void* device_rows,
                                              int64_t row_stride_bytes, int32_t y0, int32_t nrows,
                                              const avifgpu_planes* device_dst, void* cuda_stream)
{
    if (ctx == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    avifgpu_encode_desc full;
    desc = WidenEncodeDesc(desc, &full);
    std::string error;
    const int status = ValidateEncodeDesc(desc, &error);
    if (status != AVIFGPU_OK)
    {
        return ctx->Fail(status, error);
    }
    return EncodeRowsDevice(ctx, desc, device_rows, row_stride_bytes, y0, nrows, device_dst, nullptr, cuda_stream);
}

AVIFGPU_EXPORT int avifgpu_encode_rows_device_light_level(avifgpu_context* ctx, const avifgpu_encode_desc* desc, const void* device_rows,
                                                          int64_t row_stride_bytes, int32_t y0, int32_t nrows,
                                                          const avifgpu_planes* device_dst, avifgpu_light_level* device_acc,
                                                          void* cuda_stream)
{
    if (ctx == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    avifgpu_encode_desc full;
    desc = WidenEncodeDesc(desc, &full);
    std::string error;
    int status = ValidateEncodeDesc(desc, &error);
    if (status != AVIFGPU_OK)
    {
        return ctx->Fail(status, error);
    }
    if ((status = CheckLightLevelCall(ctx, *desc, device_acc)) != AVIFGPU_OK)
    {
        return status;
    }
    return EncodeRowsDevice(ctx, desc, device_rows, row_stride_bytes, y0, nrows, device_dst, device_acc, cuda_stream);
}

AVIFGPU_EXPORT int avifgpu_content_light_level(const avifgpu_light_level* acc, int32_t image_bit_depth, uint16_t* out_max_cll,
                                               uint16_t* out_max_fall)
{
    if (acc == nullptr || out_max_cll == nullptr || out_max_fall == nullptr ||
        (image_bit_depth != 8 && image_bit_depth != 10 && image_bit_depth != 12))
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    const uint32_t maxCode = (1u << image_bit_depth) - 1u;
    using Wide = unsigned __int128;
    const Wide unit = static_cast<Wide>(acc->pixels) << 22; // 2^22 x pixels: the level sum of that many pixels at 10000 cd/m2
    if (acc->max_code > maxCode || static_cast<Wide>(acc->level_sum) > unit)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    if (acc->pixels == 0)
    {
        *out_max_cll = 0;
        *out_max_fall = 0;
        return AVIFGPU_OK;
    }
    const uint64_t peak = LightLevelOf(acc->max_code, static_cast<float>(maxCode), avifmath::HostLibmTables());
    *out_max_cll = static_cast<uint16_t>((10000u * peak + (1u << 22) - 1u) >> 22);
    *out_max_fall = static_cast<uint16_t>((static_cast<Wide>(acc->level_sum) * 10000u + unit - 1u) / unit);
    return AVIFGPU_OK;
}

AVIFGPU_EXPORT int avifgpu_decode_rows_device(avifgpu_context* ctx, const avifgpu_decode_desc* desc,
                                              const avifgpu_planes* device_src, int32_t y0, int32_t nrows, void* device_rows,
                                              int64_t row_stride_bytes, void* cuda_stream)
{
    if (ctx == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    avifgpu_decode_desc full;
    desc = WidenDecodeDesc(desc, &full);
    std::string error;
    int32_t transfer;
    int status = ValidateDecodeDesc(desc, &transfer, &error);
    if (status != AVIFGPU_OK)
    {
        return ctx->Fail(status, error);
    }
    if (device_src == nullptr || (device_rows == nullptr && nrows > 0 && desc->width > 0))
    {
        return ctx->Fail(AVIFGPU_ERR_BAD_PARAM, "NULL buffer");
    }
    DecodeParams p;
    if (!FillDecodeParams(*desc, transfer, &p, &error))
    {
        return ctx->Fail(AVIFGPU_ERR_UNSUPPORTED, error);
    }
    if (y0 < 0 || nrows < 0 || y0 > desc->height || nrows > desc->height - y0)
    {
        return ctx->Fail(AVIFGPU_ERR_BAD_PARAM, "row block outside the image");
    }
    if (nrows == 0 || desc->width == 0)
    {
        return AVIFGPU_OK;
    }
    p.rows = device_rows;
    p.rowStride = row_stride_bytes;
    p.rowCount = nrows;
    p.yPhase = y0 & p.ys;
    p.smCount = ctx->smCount;
    DeviceGuard guard(ctx->device);
    bool capturing;
    if ((status = QueryCapture(ctx, cuda_stream, &capturing)) != AVIFGPU_OK)
    {
        return status;
    }
    ctx->FirstUseDecode(*desc, transfer, capturing, &p);
    for (int k = 0; k < AVIFGPU_MAX_PLANES; ++k)
    {
        const PlaneGeometry g = DecodePlaneGeometry(*desc, k);
        if (!g.present)
        {
            continue;
        }
        if (device_src->data[k] == nullptr)
        {
            return ctx->Fail(AVIFGPU_ERR_BAD_PARAM, "missing source plane");
        }
        p.plane[k] = static_cast<const uint8_t*>(device_src->data[k]) + static_cast<int64_t>(y0 >> g.ys) * device_src->stride[k];
        p.planeStride[k] = device_src->stride[k];
    }
    const int launched = LaunchDecode(p, cuda_stream);
    if (launched < 0)
    {
        return ctx->LaunchFailed(launched, "decode kernel launch", capturing);
    }
    ctx->launches += launched;
    return AVIFGPU_OK;
}

} // extern "C"

// The host-described batch encode; `acc` != nullptr: the light-level call, image i adding into acc[i] through the
// light-level family's batched kernels and, for the other images, the direct light-level route.
static int EncodeBatchDevice(avifgpu_context* ctx, const avifgpu_encode_desc* desc, const avifgpu_batch_image* images, int32_t count,
                             avifgpu_light_level* acc, void* cuda_stream)
{
    if (ctx == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    if (desc == nullptr || count < 0 || (count > 0 && images == nullptr))
    {
        return ctx->Fail(AVIFGPU_ERR_BAD_PARAM, "NULL description or image array");
    }
    avifgpu_encode_desc full;
    desc = WidenEncodeDesc(desc, &full);
    // every image is validated before anything is enqueued: the description at the image's size, then its buffers
    avifgpu_encode_desc d = *desc;
    EncodeParams shared;
    int planeMask = 0;
    int64_t pixels = 0;
    for (int32_t i = 0; i < count; ++i)
    {
        const avifgpu_batch_image& image = images[i];
        d.width = image.width;
        d.height = image.height;
        std::string error;
        const int status = ValidateEncodeDesc(&d, &error);
        if (status != AVIFGPU_OK)
        {
            return ctx->Fail(status, "image " + std::to_string(i) + ": " + error);
        }
        if (i == 0)
        {
            FillEncodeParams(d, &shared);
            for (int k = 0; k < AVIFGPU_MAX_PLANES; ++k)
            {
                planeMask |= EncodePlaneGeometry(d, k).present ? 1 << k : 0;
            }
        }
        EncodeParams p = shared;
        if (AdoptBatchImage(p, planeMask, image) != AVIFGPU_OK)
        {
            return ctx->Fail(AVIFGPU_ERR_BAD_PARAM, "image " + std::to_string(i) + (image.rows == nullptr ? ": NULL rows" : ": missing destination plane"));
        }
        pixels += static_cast<int64_t>(image.width) * image.height;
    }
    if (pixels == 0)
    {
        return AVIFGPU_OK;
    }
    DeviceGuard guard(ctx->device);
    bool capturing;
    int status = QueryCapture(ctx, cuda_stream, &capturing);
    if (status != AVIFGPU_OK)
    {
        return status;
    }
    shared.smCount = ctx->smCount;
    ctx->FirstUseEncode(*desc, pixels, capturing, &shared);
    const LightSink light = { acc, LightLevelsFor(ctx, *desc) };
    if (acc != nullptr && light.levels == nullptr)
    {
        shared.curveTable = nullptr; // no level table: every image takes the generic kernel, as a direct light-level call does
    }
    BatchPlan plan;
    if (acc != nullptr)
    {
        PlanEncodeLightBatch(shared, planeMask, images, count, &plan);
    }
    else
    {
        PlanEncodeBatch(shared, desc->host_depth, planeMask, images, count, &plan);
    }
    for (const BatchChunk& chunk : plan.chunks)
    {
        const int launched = acc != nullptr ? LaunchEncodeLightBatchChunk(shared, chunk, light, cuda_stream)
                                            : LaunchEncodeBatchChunk(shared, desc->host_depth, chunk, cuda_stream);
        if (launched < 0)
        {
            return ctx->LaunchFailed(launched, "batched encode kernel launch", capturing);
        }
        ctx->launches += launched;
    }
    for (const int32_t i : plan.fallback)
    {
        EncodeParams p = shared;
        AdoptBatchImage(p, planeMask, images[i]);
        const LightSink own = { acc + i, light.levels };
        const int launched = LaunchEncode(p, desc->host_depth, cuda_stream, acc != nullptr ? &own : nullptr);
        if (launched < 0)
        {
            return ctx->LaunchFailed(launched, "encode kernel launch", capturing);
        }
        ctx->launches += launched;
    }
    return AVIFGPU_OK;
}

extern "C" {

AVIFGPU_EXPORT int avifgpu_encode_batch_device(avifgpu_context* ctx, const avifgpu_encode_desc* desc, const avifgpu_batch_image* images,
                                               int32_t count, void* cuda_stream)
{
    return EncodeBatchDevice(ctx, desc, images, count, nullptr, cuda_stream);
}

// The description is checked at size 0 (the images carry the sizes) for the light-level refusals, which come before the
// images' own checks.
AVIFGPU_EXPORT int avifgpu_encode_batch_device_light_level(avifgpu_context* ctx, const avifgpu_encode_desc* desc, const avifgpu_batch_image* images,
                                                           int32_t count, avifgpu_light_level* device_acc, void* cuda_stream)
{
    if (ctx == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    if (desc == nullptr)
    {
        return ctx->Fail(AVIFGPU_ERR_BAD_PARAM, "NULL description");
    }
    avifgpu_encode_desc full;
    avifgpu_encode_desc d = *WidenEncodeDesc(desc, &full);
    d.width = 0;
    d.height = 0;
    std::string error;
    int status = ValidateEncodeDesc(&d, &error);
    if (status != AVIFGPU_OK)
    {
        return ctx->Fail(status, error);
    }
    if ((status = CheckLightLevelCall(ctx, d, device_acc)) != AVIFGPU_OK)
    {
        return status;
    }
    return EncodeBatchDevice(ctx, desc, images, count, device_acc, cuda_stream);
}

AVIFGPU_EXPORT int avifgpu_decode_batch_device(avifgpu_context* ctx, const avifgpu_decode_desc* desc, const avifgpu_batch_image* images,
                                               int32_t count, void* cuda_stream)
{
    if (ctx == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    if (desc == nullptr || count < 0 || (count > 0 && images == nullptr))
    {
        return ctx->Fail(AVIFGPU_ERR_BAD_PARAM, "NULL description or image array");
    }
    avifgpu_decode_desc full;
    desc = WidenDecodeDesc(desc, &full);
    // every image is validated before anything is enqueued: the description at the image's size, then its buffers
    avifgpu_decode_desc d = *desc;
    DecodeParams shared;
    int32_t transfer = 0;
    int planeMask = 0;
    int64_t pixels = 0;
    for (int32_t i = 0; i < count; ++i)
    {
        const avifgpu_batch_image& image = images[i];
        d.width = image.width;
        d.height = image.height;
        std::string error;
        const int status = ValidateDecodeDesc(&d, &transfer, &error);
        if (status != AVIFGPU_OK)
        {
            return ctx->Fail(status, "image " + std::to_string(i) + ": " + error);
        }
        if (i == 0)
        {
            if (!FillDecodeParams(d, transfer, &shared, &error))
            {
                return ctx->Fail(AVIFGPU_ERR_UNSUPPORTED, "image 0: " + error);
            }
            for (int k = 0; k < AVIFGPU_MAX_PLANES; ++k)
            {
                planeMask |= DecodePlaneGeometry(d, k).present ? 1 << k : 0;
            }
        }
        DecodeParams p = shared;
        if (AdoptBatchImage(p, planeMask, image) != AVIFGPU_OK)
        {
            return ctx->Fail(AVIFGPU_ERR_BAD_PARAM, "image " + std::to_string(i) + (image.rows == nullptr ? ": NULL rows" : ": missing source plane"));
        }
        pixels += static_cast<int64_t>(image.width) * image.height;
    }
    if (pixels == 0)
    {
        return AVIFGPU_OK;
    }
    DeviceGuard guard(ctx->device);
    bool capturing;
    int status = QueryCapture(ctx, cuda_stream, &capturing);
    if (status != AVIFGPU_OK)
    {
        return status;
    }
    shared.smCount = ctx->smCount;
    ctx->FirstUseDecode(*desc, transfer, capturing, &shared);
    BatchPlan plan;
    PlanDecodeBatch(shared, planeMask, images, count, &plan);
    for (const BatchChunk& chunk : plan.chunks)
    {
        const int launched = LaunchDecodeBatchChunk(shared, chunk, cuda_stream);
        if (launched < 0)
        {
            return ctx->LaunchFailed(launched, "batched decode kernel launch", capturing);
        }
        ctx->launches += launched;
    }
    for (const int32_t i : plan.fallback)
    {
        DecodeParams p = shared;
        AdoptBatchImage(p, planeMask, images[i]);
        const int launched = LaunchDecode(p, cuda_stream);
        if (launched < 0)
        {
            return ctx->LaunchFailed(launched, "decode kernel launch", capturing);
        }
        ctx->launches += launched;
    }
    return AVIFGPU_OK;
}

AVIFGPU_EXPORT int avifgpu_batch_workspace_bytes(int32_t max_count, size_t* out_bytes)
{
    if (out_bytes == nullptr || max_count < 1 || max_count > kIndirectMaxImages)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    *out_bytes = IndirectWorkspaceLayout(max_count).bytes;
    return AVIFGPU_OK;
}

} // extern "C"

namespace
{
    // The host checks both device-described calls make before anything is launched.
    int CheckIndirect(avifgpu_context* ctx, const void* images, const int32_t* count, int32_t maxCount, const void* workspace, size_t workspaceBytes)
    {
        if (images == nullptr || count == nullptr || workspace == nullptr)
        {
            return ctx->Fail(AVIFGPU_ERR_BAD_PARAM, "NULL device image array, count or workspace");
        }
        if (maxCount < 1 || maxCount > kIndirectMaxImages)
        {
            return ctx->Fail(AVIFGPU_ERR_BAD_PARAM, "max_count must be 1..4096");
        }
        if (workspaceBytes < IndirectWorkspaceLayout(maxCount).bytes)
        {
            return ctx->Fail(AVIFGPU_ERR_BAD_PARAM, "workspace smaller than avifgpu_batch_workspace_bytes(max_count)");
        }
        return AVIFGPU_OK;
    }
} // namespace

// The device-described batch encode; `acc` != nullptr: the light-level call (float hosts through the light-level family's
// batched kernels), image i adding into acc[i].
static int EncodeBatchIndirect(avifgpu_context* ctx, const avifgpu_encode_desc* desc, const avifgpu_batch_image* device_images,
                               const int32_t* device_count, int32_t max_count, void* device_workspace, size_t workspace_bytes,
                               int32_t* device_status, avifgpu_light_level* acc, bool light, void* cuda_stream)
{
    if (ctx == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    if (desc == nullptr)
    {
        return ctx->Fail(AVIFGPU_ERR_BAD_PARAM, "NULL description");
    }
    avifgpu_encode_desc full;
    desc = WidenEncodeDesc(desc, &full);
    avifgpu_encode_desc d = *desc; // the images carry the sizes
    d.width = 0;
    d.height = 0;
    std::string error;
    int status = ValidateEncodeDesc(&d, &error);
    if (status != AVIFGPU_OK)
    {
        return ctx->Fail(status, error);
    }
    if (light && (status = CheckLightLevelCall(ctx, d, acc)) != AVIFGPU_OK)
    {
        return status;
    }
    if ((status = CheckIndirect(ctx, device_images, device_count, max_count, device_workspace, workspace_bytes)) != AVIFGPU_OK)
    {
        return status;
    }
    if (light && (d.layout != AVIFGPU_LAYOUT_PLANAR_YCBCR || d.host_channels < 3))
    {
        return ctx->Fail(AVIFGPU_ERR_UNSUPPORTED, "device-described light-level batches encode RGB(A)32f hosts into planar YCbCr");
    }
    if (!light && ((d.host_depth != 8 && d.host_depth != 16) || d.layout != AVIFGPU_LAYOUT_PLANAR_YCBCR))
    {
        return ctx->Fail(AVIFGPU_ERR_UNSUPPORTED, "device-described batches encode 8- or 16-bit RGB(A) hosts into planar YCbCr");
    }
    EncodeParams shared;
    FillEncodeParams(d, &shared);
    int planeMask = 0;
    for (int k = 0; k < AVIFGPU_MAX_PLANES; ++k)
    {
        planeMask |= EncodePlaneGeometry(d, k).present ? 1 << k : 0;
    }
    DeviceGuard guard(ctx->device);
    bool capturing;
    if ((status = QueryCapture(ctx, cuda_stream, &capturing)) != AVIFGPU_OK)
    {
        return status;
    }
    shared.smCount = ctx->smCount;
    ctx->FirstUseEncode(d, 0, capturing, &shared);
    int launched;
    if (light)
    {
        const LightSink sink = { acc, LightLevelsFor(ctx, d) };
        if (sink.levels == nullptr)
        {
            shared.curveTable = nullptr; // no level table: every image through the edge kernel, which evaluates the levels
        }
        launched = LaunchEncodeLightIndirect(shared, planeMask, device_images, device_count, max_count, device_workspace, device_status, sink, cuda_stream);
    }
    else
    {
        launched = LaunchEncodeIndirect(shared, d.host_depth, EncodeBatchFamilyOf(shared, d.host_depth), planeMask, device_images, device_count, max_count,
                                        device_workspace, device_status, cuda_stream);
    }
    if (launched < 0)
    {
        return ctx->LaunchFailed(launched, "device-described batch encode launch", capturing);
    }
    ctx->launches += launched;
    return AVIFGPU_OK;
}

extern "C" {

AVIFGPU_EXPORT int avifgpu_encode_batch_indirect(avifgpu_context* ctx, const avifgpu_encode_desc* desc, const avifgpu_batch_image* device_images,
                                                 const int32_t* device_count, int32_t max_count, void* device_workspace, size_t workspace_bytes,
                                                 int32_t* device_status, void* cuda_stream)
{
    return EncodeBatchIndirect(ctx, desc, device_images, device_count, max_count, device_workspace, workspace_bytes, device_status, nullptr, false,
                               cuda_stream);
}

AVIFGPU_EXPORT int avifgpu_encode_batch_indirect_light_level(avifgpu_context* ctx, const avifgpu_encode_desc* desc,
                                                             const avifgpu_batch_image* device_images, const int32_t* device_count,
                                                             int32_t max_count, void* device_workspace, size_t workspace_bytes,
                                                             int32_t* device_status, avifgpu_light_level* device_acc, void* cuda_stream)
{
    return EncodeBatchIndirect(ctx, desc, device_images, device_count, max_count, device_workspace, workspace_bytes, device_status, device_acc, true,
                               cuda_stream);
}

AVIFGPU_EXPORT int avifgpu_decode_batch_indirect(avifgpu_context* ctx, const avifgpu_decode_desc* desc, const avifgpu_batch_image* device_images,
                                                 const int32_t* device_count, int32_t max_count, void* device_workspace, size_t workspace_bytes,
                                                 int32_t* device_status, void* cuda_stream)
{
    if (ctx == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    if (desc == nullptr)
    {
        return ctx->Fail(AVIFGPU_ERR_BAD_PARAM, "NULL description");
    }
    avifgpu_decode_desc full;
    desc = WidenDecodeDesc(desc, &full);
    avifgpu_decode_desc d = *desc;
    d.width = 0;
    d.height = 0;
    std::string error;
    int32_t transfer = 0;
    int status = ValidateDecodeDesc(&d, &transfer, &error);
    if (status != AVIFGPU_OK)
    {
        return ctx->Fail(status, error);
    }
    if ((status = CheckIndirect(ctx, device_images, device_count, max_count, device_workspace, workspace_bytes)) != AVIFGPU_OK)
    {
        return status;
    }
    if (d.colorspace == AVIFGPU_COLORSPACE_MONOCHROME || d.alpha_state == AVIFGPU_ALPHA_PREMULTIPLIED)
    {
        return ctx->Fail(AVIFGPU_ERR_UNSUPPORTED, "device-described batches decode YCbCr or planar RGB with no or straight alpha");
    }
    DecodeParams shared;
    if (!FillDecodeParams(d, transfer, &shared, &error))
    {
        return ctx->Fail(AVIFGPU_ERR_UNSUPPORTED, error);
    }
    int planeMask = 0;
    for (int k = 0; k < AVIFGPU_MAX_PLANES; ++k)
    {
        planeMask |= DecodePlaneGeometry(d, k).present ? 1 << k : 0;
    }
    DeviceGuard guard(ctx->device);
    bool capturing;
    if ((status = QueryCapture(ctx, cuda_stream, &capturing)) != AVIFGPU_OK)
    {
        return status;
    }
    shared.smCount = ctx->smCount;
    ctx->FirstUseDecode(d, transfer, capturing, &shared);
    const int launched = LaunchDecodeIndirect(shared, DecodeBatchFamilyOf(shared), planeMask, device_images, device_count, max_count, device_workspace,
                                              device_status, cuda_stream);
    if (launched < 0)
    {
        return ctx->LaunchFailed(launched, "device-described batch decode launch", capturing);
    }
    ctx->launches += launched;
    return AVIFGPU_OK;
}

} // extern "C"

// ---- host-pointer entry points (PCIe inside) ---------------------------------------------------------------------
//
// A call is cut into row-block slices; slice i uses pipeline slot i mod kPipelineStreams (a stream, device staging,
// pinned bounce buffers).  Caller memory that is not page-locked is bounced through the slot's pinned buffers on BOTH
// sides -- a copy to or from pageable memory would make the driver stage it synchronously and serialise the pipeline.
// The bounce -> pageable copies of a slot's last slice, and a light-level encode's merge of the slice's statistic into the
// caller's accumulator, stay owed (its debts) until the slot's next slice or a retire pays them.  Slots retire in issue
// order, so "everything up to ticket t" is a prefix.
//
// Both directions run a slice through the same steps: AcquireSlot, StageIn, the kernel launch, StageOut, CloseSlice.
// Every pinned buffer those steps write into or regrow comes from TakePinned, which first pays the debts that read it.

// Rows per pipeline slice: big enough to amortise launch + copy latency, small enough that the slots overlap.
static int SliceRows(int nrows, int64_t bytesPerRow)
{
    const int64_t target = 32ll << 20; // ~32 MiB of host rows per slice
    int64_t rows = bytesPerRow > 0 ? target / bytesPerRow : nrows;
    rows = std::max<int64_t>(rows, 2);
    rows &= ~1ll; // keep 4:2:0 row pairs together
    return static_cast<int>(std::min<int64_t>(rows, nrows));
}

static void CopyRowsSerial(uint8_t* target, int64_t targetStride, const uint8_t* source, int64_t sourceStride, int64_t payload, int rows)
{
    if (targetStride == payload && sourceStride == payload)
    {
        std::memcpy(target, source, static_cast<size_t>(payload) * rows);
        return;
    }
    for (int r = 0; r < rows; ++r)
    {
        std::memcpy(target + static_cast<int64_t>(r) * targetStride, source + static_cast<int64_t>(r) * sourceStride, static_cast<size_t>(payload));
    }
}

// Bounce copies between pageable caller memory and the pinned slot buffers.  One core moves ~10 GB/s, a fifth of what
// the PCIe link next to it carries, and an 8K frame owes 100 MB of plane copies: a small pool of parked threads (created
// at the first bounce, process-wide, joined at exit) shares every batch of copies above a megabyte, cut into chunks of
// rows that the threads -- and the caller -- pull from a common counter.
namespace
{
    class CopyPool
    {
    public:
        static CopyPool& Instance()
        {
            static CopyPool pool;
            return pool;
        }

        void Copy(const RowCopy* copies, int count)
        {
            int64_t bytes = 0;
            for (int i = 0; i < count; ++i)
            {
                bytes += copies[i].payload * copies[i].rows;
            }
            if (bytes < (1ll << 20) || workers.empty())
            {
                for (int i = 0; i < count; ++i)
                {
                    CopyRowsSerial(copies[i].target, copies[i].targetStride, copies[i].source, copies[i].sourceStride, copies[i].payload, copies[i].rows);
                }
                return;
            }
            std::unique_lock<std::mutex> callers(callerMutex); // one batch at a time (contexts on several threads share the pool)
            {
                std::lock_guard<std::mutex> lock(mutex);
                chunks.clear();
                for (int i = 0; i < count; ++i)
                {
                    const RowCopy& c = copies[i];
                    const int rowsPerChunk = static_cast<int>(std::max<int64_t>((256ll << 10) / std::max<int64_t>(c.payload, 1), 1));
                    for (int begin = 0; begin < c.rows; begin += rowsPerChunk)
                    {
                        chunks.push_back(RowCopy{ c.target + static_cast<int64_t>(begin) * c.targetStride, c.targetStride,
                                                  c.source + static_cast<int64_t>(begin) * c.sourceStride, c.sourceStride, c.payload,
                                                  std::min(rowsPerChunk, c.rows - begin) });
                    }
                }
                next.store(0, std::memory_order_relaxed);
                remaining = static_cast<int>(chunks.size());
                ++generation;
            }
            wake.notify_all();
            Drain();
            std::unique_lock<std::mutex> lock(mutex);
            done.wait(lock, [&] { return remaining == 0; });
        }

    private:
        CopyPool()
        {
            const unsigned cores = std::thread::hardware_concurrency();
            // 8 copying threads with the caller.  More copy threads disturb the DMA they run beside, while fewer than 4
            // cannot keep up with config 4's 1.6 GB of planes or with first-touch page faults.
            const int count = static_cast<int>(std::min<unsigned>(cores > 1 ? cores - 1 : 0, 7));
            for (int i = 0; i < count; ++i)
            {
                workers.emplace_back([this] { Run(); });
            }
        }

        ~CopyPool()
        {
            {
                std::lock_guard<std::mutex> lock(mutex);
                stopping = true;
            }
            wake.notify_all();
            for (std::thread& t : workers)
            {
                t.join();
            }
        }

        // Pulls chunks until none is left; returns how many this thread copied.
        void Drain()
        {
            int copied = 0;
            const int total = static_cast<int>(chunks.size());
            for (;;)
            {
                const int i = next.fetch_add(1, std::memory_order_relaxed);
                if (i >= total)
                {
                    break;
                }
                const RowCopy& c = chunks[i];
                CopyRowsSerial(c.target, c.targetStride, c.source, c.sourceStride, c.payload, c.rows);
                ++copied;
            }
            if (copied)
            {
                std::lock_guard<std::mutex> lock(mutex);
                remaining -= copied;
                if (remaining == 0)
                {
                    done.notify_all();
                }
            }
        }

        void Run()
        {
            uint64_t seen = 0;
            for (;;)
            {
                {
                    std::unique_lock<std::mutex> lock(mutex);
                    wake.wait(lock, [&] { return stopping || generation != seen; });
                    if (stopping)
                    {
                        return;
                    }
                    seen = generation;
                }
                Drain(); // `chunks` is stable until the caller has seen remaining == 0, which needs every pulled chunk finished
            }
        }

        std::vector<std::thread> workers;
        std::mutex mutex, callerMutex;
        std::condition_variable wake, done;
        std::vector<RowCopy> chunks;
        std::atomic<int> next{ 0 };
        int remaining = 0;
        uint64_t generation = 0;
        bool stopping = false;
    };
}

using Slot = avifgpu_context::Slot;

// Waits for the slot's stream work (its device buffers are free again after this); what it owes the caller stays owed.
static int WaitSlot(avifgpu_context* ctx, Slot& slot)
{
    if (!slot.busy)
    {
        return AVIFGPU_OK;
    }
    const int status = ctx->Cuda(cudaEventSynchronize(slot.sliceDone), "cudaEventSynchronize");
    if (status != AVIFGPU_OK)
    {
        for (RowCopy& c : slot.owed) c.rows = 0;
        slot.owedLight = nullptr;
    }
    slot.busy = false;
    return status;
}

// Adds a partial statistic into a host accumulator (the statistic does not depend on the order of its parts);
// `reserved` is never written.
static void AddLightLevel(avifgpu_light_level& acc, const avifgpu_light_level& part)
{
    acc.max_code = std::max(acc.max_code, part.max_code);
    acc.level_sum += part.level_sum;
    acc.pixels += part.pixels;
}

// Merges the light-level mirror of a waited-for slot into the caller's accumulator it is owed to, on the caller's thread.
static void PayLightDebt(Slot& slot)
{
    if (slot.owedLight != nullptr)
    {
        AddLightLevel(*slot.owedLight, *slot.lightMirror);
        slot.owedLight = nullptr;
    }
}

// Pays, in one batch for the copy pool, what a waited-for slot owes out of the pinned buffers marked in `buffers` (out
// of all of them, and the light-level merge, when nullptr: whoever takes or retires the slot then finds it owing nothing,
// so every debt stays with the ticket of the slice that made it).  Separate batches would cost a wake-up and a wait each.
static void PayDebts(Slot& slot, const bool* buffers = nullptr)
{
    RowCopy batch[kSlotBuffers];
    int count = 0;
    for (int b = 0; b < kSlotBuffers; ++b)
    {
        if (slot.owed[b].rows > 0 && (buffers == nullptr || buffers[b]))
        {
            batch[count++] = slot.owed[b];
            slot.owed[b].rows = 0;
        }
    }
    if (count > 0) CopyPool::Instance().Copy(batch, count); // the pool's threads start at the first copy
    if (buffers == nullptr) PayLightDebt(slot);
}

// Retires, oldest first, every slot issued by a call with ticket <= `ticket`.
static int RetireThrough(avifgpu_context* ctx, int64_t ticket)
{
    int result = AVIFGPU_OK;
    for (int i = 0; i < kPipelineStreams; ++i)
    {
        Slot& slot = ctx->slots[(ctx->nextSlot + i) % kPipelineStreams]; // nextSlot is the oldest
        bool owes = slot.owedLight != nullptr;
        for (const RowCopy& c : slot.owed) owes = owes || c.rows > 0;
        if ((slot.busy || owes) && slot.ticket <= ticket)
        {
            const int status = WaitSlot(ctx, slot);
            if (status == AVIFGPU_OK) PayDebts(slot);
            else if (result == AVIFGPU_OK) result = status;
        }
    }
    return result;
}

// Every host-pointer call that returns AVIFGPU_OK hands the rows of the previous asynchronous encode call back to the
// caller (avifgpu.h).  A call takes that release before it queues its own copies and waits for those rows' H2Ds just
// before it returns (FinishCall), so the link never idles at a call boundary.  Returns the callRowsConsumed event to
// wait for, or -1.
static int TakeRowsRelease(avifgpu_context* ctx)
{
    const int event = ctx->previousCallRowsPending ? static_cast<int>((ctx->asyncEncodeCalls - 1) & 1) : -1;
    ctx->previousCallRowsPending = false;
    return event;
}

// A failure in the middle of a call: nothing of this context may still be writing into caller memory on return.
static int AbandonCall(avifgpu_context* ctx, int status)
{
    for (Slot& slot : ctx->slots)
    {
        cudaStreamSynchronize(slot.stream);
        for (RowCopy& c : slot.owed) c.rows = 0;
        slot.owedLight = nullptr;
        slot.busy = false;
    }
    cudaGetLastError();
    return status;
}

// The end of a call that has queued all its slices, or had none: release the previous asynchronous encode's rows, then
// retire the call's slots if the call waits.
static int FinishCall(avifgpu_context* ctx, int previousRows, int64_t ticket, bool wait)
{
    int status = previousRows < 0 ? AVIFGPU_OK : ctx->Cuda(cudaEventSynchronize(ctx->callRowsConsumed[previousRows]), "cudaEventSynchronize");
    if (status == AVIFGPU_OK && wait)
    {
        status = RetireThrough(ctx, ticket);
    }
    return status == AVIFGPU_OK ? AVIFGPU_OK : AbandonCall(ctx, status);
}

// One host <-> device copy of a slice, between caller memory and the slot's buffers number `buffer`.
struct SliceCopy
{
    int buffer;          // a plane index, or kRowsBuffer
    uint8_t* host;       // the slice's first row in caller memory
    int64_t hostStride;
    bool hostPinned;     // false: the copy bounces through the slot's pinned buffer
    int64_t payload;     // bytes per row
    int64_t deviceStride;
    int rows;
};

// Fills `windows` with the rows of each present whole-image plane that the slice of image rows [yFirst, yFirst + rows)
// covers, and returns how many planes there are.
static int PlaneWindows(const avifgpu_planes* planes, const PlaneGeometry* geometry, const bool* pinned, int yFirst, int rows, SliceCopy* windows)
{
    int count = 0;
    for (int k = 0; k < AVIFGPU_MAX_PLANES; ++k)
    {
        const PlaneGeometry& g = geometry[k];
        if (g.present)
        {
            const int firstRow = yFirst >> g.ys;
            const int64_t payload = static_cast<int64_t>(g.widthSamples) * g.bytesPerSample;
            windows[count++] = SliceCopy{ k, static_cast<uint8_t*>(planes->data[k]) + static_cast<int64_t>(firstRow) * planes->stride[k], planes->stride[k],
                                          pinned[k], payload, (payload + 255) & ~255ll, ((yFirst + rows - 1) >> g.ys) - firstRow + 1 };
        }
    }
    return count;
}

static int EnsureDeviceStaging(avifgpu_context* ctx, Slot& slot, const SliceCopy* copies, int count)
{
    for (int i = 0; i < count; ++i)
    {
        const int status = ctx->EnsureDevice(slot.device[copies[i].buffer], static_cast<size_t>(copies[i].deviceStride) * copies[i].rows);
        if (status != AVIFGPU_OK) return status;
    }
    return AVIFGPU_OK;
}

// Hands out, grown to fit, the slot's pinned buffers that the pageable sides of `copies` bounce through: the only way
// to a pinned buffer that the host or the device is about to write.  It first pays, in one batch, the debts that read
// those buffers, so no pinned buffer is written or regrown while the slot owes copies out of it.
static int TakePinned(avifgpu_context* ctx, Slot& slot, const SliceCopy* copies, int count, uint8_t* pinned[kSlotBuffers])
{
    bool taken[kSlotBuffers] = {};
    for (int i = 0; i < count; ++i)
    {
        taken[copies[i].buffer] = !copies[i].hostPinned;
    }
    PayDebts(slot, taken);
    for (int i = 0; i < count; ++i)
    {
        const SliceCopy& c = copies[i];
        if (!c.hostPinned)
        {
            const int status = ctx->EnsurePinned(slot.pinned[c.buffer], static_cast<size_t>(c.payload) * c.rows);
            if (status != AVIFGPU_OK) return status;
            pinned[c.buffer] = static_cast<uint8_t*>(slot.pinned[c.buffer].ptr);
        }
    }
    return AVIFGPU_OK;
}

// Waits for the next slot in rotation and takes it for a slice; what the slot owes is paid by StageIn and StageOut.
static int AcquireSlot(avifgpu_context* ctx, int* slot)
{
    *slot = ctx->nextSlot;
    const int status = WaitSlot(ctx, ctx->slots[*slot]);
    if (status == AVIFGPU_OK)
    {
        ctx->nextSlot = (*slot + 1) % kPipelineStreams;
    }
    return status;
}

// Queues a slice's host -> device copies on the slot's stream.  Pageable sources are bounced first, every one of the
// slice in ONE batch for the copy pool (three batches for three planes cost three wake-ups and waits, ~0.5 ms per slice,
// ahead of anything the GPU could do).
static int StageIn(avifgpu_context* ctx, Slot& slot, const SliceCopy* copies, int count)
{
    uint8_t* pinned[kSlotBuffers] = {};
    int status = EnsureDeviceStaging(ctx, slot, copies, count);
    if (status != AVIFGPU_OK || (status = TakePinned(ctx, slot, copies, count, pinned)) != AVIFGPU_OK) return status;
    RowCopy bounce[kSlotBuffers];
    int bounced = 0;
    for (int i = 0; i < count; ++i)
    {
        const SliceCopy& c = copies[i];
        if (!c.hostPinned)
        {
            bounce[bounced++] = RowCopy{ pinned[c.buffer], c.payload, c.host, c.hostStride, c.payload, c.rows };
        }
    }
    if (bounced > 0) CopyPool::Instance().Copy(bounce, bounced);
    for (int i = 0; i < count; ++i)
    {
        const SliceCopy& c = copies[i];
        const uint8_t* source = c.hostPinned ? c.host : pinned[c.buffer];
        const int64_t sourceStride = c.hostPinned ? c.hostStride : c.payload;
        if ((status = ctx->Cuda(cudaMemcpy2DAsync(slot.device[c.buffer].ptr, static_cast<size_t>(c.deviceStride), source,
                                                  static_cast<size_t>(sourceStride), static_cast<size_t>(c.payload),
                                                  static_cast<size_t>(c.rows), cudaMemcpyHostToDevice, slot.stream),
                                c.buffer == kRowsBuffer ? "H2D rows" : "H2D plane")) != AVIFGPU_OK) return status;
    }
    return AVIFGPU_OK;
}

// Queues a slice's device -> host copies on the slot's stream, once everything the slot still owes is paid (in one
// batch): paid here, after the slice's H2Ds and kernel are queued, the host copies while the link and the SMs work.  A
// pageable target gets its rows in the slot's pinned buffer, and the copy across becomes a debt of the slot.
static int StageOut(avifgpu_context* ctx, Slot& slot, const SliceCopy* copies, int count)
{
    PayDebts(slot);
    uint8_t* pinned[kSlotBuffers] = {};
    int status = TakePinned(ctx, slot, copies, count, pinned);
    if (status != AVIFGPU_OK) return status;
    for (int i = 0; i < count; ++i)
    {
        const SliceCopy& c = copies[i];
        uint8_t* target = c.host;
        int64_t targetStride = c.hostStride;
        if (!c.hostPinned)
        {
            slot.owed[c.buffer] = RowCopy{ c.host, c.hostStride, pinned[c.buffer], c.payload, c.payload, c.rows };
            target = pinned[c.buffer];
            targetStride = c.payload;
        }
        if ((status = ctx->Cuda(cudaMemcpy2DAsync(target, static_cast<size_t>(targetStride), slot.device[c.buffer].ptr,
                                                  static_cast<size_t>(c.deviceStride), static_cast<size_t>(c.payload),
                                                  static_cast<size_t>(c.rows), cudaMemcpyDeviceToHost, slot.stream),
                                c.buffer == kRowsBuffer ? "D2H rows" : "D2H plane")) != AVIFGPU_OK) return status;
    }
    return AVIFGPU_OK;
}

// Marks the end of the slice queued on the slot's stream; the slot belongs to the call with `ticket` until retired.
static int CloseSlice(avifgpu_context* ctx, Slot& slot, int64_t ticket)
{
    const int status = ctx->Cuda(cudaEventRecord(slot.sliceDone, slot.stream), "cudaEventRecord");
    if (status == AVIFGPU_OK)
    {
        slot.busy = true;
        slot.ticket = ticket;
    }
    return status;
}

// The light-level slice's first step, once the slot is acquired: the slot's accumulator, allocated at first use, cleared.
static int ClearSliceLight(avifgpu_context* ctx, Slot& slot)
{
    int status = AVIFGPU_OK;
    if (slot.lightDevice == nullptr)
    {
        status = ctx->Cuda(cudaMalloc(&slot.lightDevice, sizeof(avifgpu_light_level)), "cudaMalloc");
    }
    if (status == AVIFGPU_OK && slot.lightMirror == nullptr)
    {
        status = ctx->Cuda(cudaHostAlloc(&slot.lightMirror, sizeof(avifgpu_light_level), cudaHostAllocDefault), "cudaHostAlloc");
    }
    return status != AVIFGPU_OK ? status : ctx->Cuda(cudaMemsetAsync(slot.lightDevice, 0, sizeof(avifgpu_light_level), slot.stream), "cudaMemsetAsync");
}

// Queues, after the slice's kernel and StageOut, the copy of the slot's accumulator into its pinned mirror, and makes
// merging the mirror into the caller's `acc` a debt of the slot.  Like a pinned buffer, the mirror is not rewritten while
// the slot still owes out of it: StageOut has paid every debt of the slot's previous slice, its merge included.
static int StageLightOut(avifgpu_context* ctx, Slot& slot, avifgpu_light_level* acc)
{
    const int status = ctx->Cuda(cudaMemcpyAsync(slot.lightMirror, slot.lightDevice, sizeof(avifgpu_light_level), cudaMemcpyDeviceToHost, slot.stream),
                                 "D2H light level");
    if (status == AVIFGPU_OK)
    {
        slot.owedLight = acc;
    }
    return status;
}

// The host-pointer encode; `measure`: the light-level call, which adds the content light level of the rows into the host
// accumulator `acc` through the slots' own accumulators (merged as slot debts, see avifgpu.h for when `acc` is complete).
static int EncodeRowsHost(avifgpu_context* ctx, const avifgpu_encode_desc* desc, const void* host_rows, int64_t row_stride_bytes, int32_t y0,
                          int32_t nrows, const avifgpu_planes* dst, bool wait, int64_t* out_ticket, bool measure, avifgpu_light_level* acc)
{
    if (ctx == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    avifgpu_encode_desc full;
    desc = WidenEncodeDesc(desc, &full);
    std::string error;
    int status = ValidateEncodeDesc(desc, &error);
    if (status != AVIFGPU_OK)
    {
        return ctx->Fail(status, error);
    }
    if (measure && (status = CheckLightLevelCall(ctx, *desc, acc)) != AVIFGPU_OK)
    {
        return status;
    }
    if (DestLayoutOf(*desc) != AVIFGPU_SOURCE_PLANAR)
    {
        return ctx->Fail(AVIFGPU_ERR_UNSUPPORTED, "the host-pointer calls write planar, low-bit planes only (libheif's layout)");
    }
    if (dst == nullptr || (host_rows == nullptr && nrows > 0 && desc->width > 0))
    {
        return ctx->Fail(AVIFGPU_ERR_BAD_PARAM, "NULL buffer");
    }
    EncodeParams base;
    FillEncodeParams(*desc, &base);
    status = CheckBlock(ctx, desc->height, base.ys, y0, nrows);
    if (status != AVIFGPU_OK)
    {
        return status;
    }
    const int64_t ticket = ++ctx->lastTicket;
    if (out_ticket != nullptr)
    {
        *out_ticket = ticket;
    }
    DeviceGuard guard(ctx->device);
    if (nrows == 0 || desc->width == 0)
    {
        return FinishCall(ctx, TakeRowsRelease(ctx), ticket, wait);
    }
    PlaneGeometry geometry[AVIFGPU_MAX_PLANES];
    bool planePinned[AVIFGPU_MAX_PLANES] = {};
    for (int k = 0; k < AVIFGPU_MAX_PLANES; ++k)
    {
        geometry[k] = EncodePlaneGeometry(*desc, k);
        if (geometry[k].present && dst->data[k] == nullptr)
        {
            return ctx->Fail(AVIFGPU_ERR_BAD_PARAM, "missing destination plane");
        }
        planePinned[k] = geometry[k].present && IsPinned(dst->data[k]);
    }

    base.smCount = ctx->smCount;
    ctx->FirstUseEncode(*desc, static_cast<int64_t>(desc->width) * nrows, false, &base);
    const uint32_t* levels = LightLevelsFor(ctx, *desc);
    if (measure && levels == nullptr)
    {
        base.curveTable = nullptr; // no level table: the generic kernel evaluates the levels (as EncodeRowsDevice)
    }
    const int64_t rowPayload = static_cast<int64_t>(desc->width) * EncodeHostColBytes(*desc);
    const int64_t deviceRowStride = (rowPayload + 255) & ~255ll;
    const bool rowsPinned = IsPinned(host_rows);
    const int sliceRows = SliceRows(nrows, rowPayload);
    uint8_t* rowsIn = static_cast<uint8_t*>(const_cast<void*>(host_rows)); // only ever read

    const int previousRows = TakeRowsRelease(ctx);
    bool recordedCallRows = false;
    bool callSlots[kPipelineStreams] = {}; // the slots this call's H2Ds went through

    for (int begin = 0; begin < nrows; begin += sliceRows)
    {
        const int rows = std::min(sliceRows, nrows - begin);
        int index;
        if ((status = AcquireSlot(ctx, &index)) != AVIFGPU_OK) return AbandonCall(ctx, status);
        Slot& slot = ctx->slots[index];
        const SliceCopy in{ kRowsBuffer, rowsIn + static_cast<int64_t>(begin) * row_stride_bytes, row_stride_bytes, rowsPinned, rowPayload, deviceRowStride, rows };
        SliceCopy out[AVIFGPU_MAX_PLANES];
        const int planes = PlaneWindows(dst, geometry, planePinned, y0 + begin, rows, out);
        if ((status = StageIn(ctx, slot, &in, 1)) != AVIFGPU_OK ||
            (status = ctx->Cuda(cudaEventRecord(slot.rowsConsumed, slot.stream), "cudaEventRecord")) != AVIFGPU_OK) return AbandonCall(ctx, status);
        callSlots[index] = true;
        if (!wait && rowsPinned && begin + sliceRows >= nrows)
        {
            // The caller's own memory is on the wire until every H2D of the call has finished, and the H2Ds of different
            // streams may finish out of order: the last slice's stream waits for the other slots' before it records the
            // event the NEXT call waits for.
            for (int s = 0; s < kPipelineStreams; ++s)
            {
                if (s != index && callSlots[s] &&
                    (status = ctx->Cuda(cudaStreamWaitEvent(slot.stream, ctx->slots[s].rowsConsumed, 0), "cudaStreamWaitEvent")) != AVIFGPU_OK) return AbandonCall(ctx, status);
            }
            if ((status = ctx->Cuda(cudaEventRecord(ctx->callRowsConsumed[ctx->asyncEncodeCalls & 1], slot.stream), "cudaEventRecord")) != AVIFGPU_OK) return AbandonCall(ctx, status);
            recordedCallRows = true;
        }

        if ((status = EnsureDeviceStaging(ctx, slot, out, planes)) != AVIFGPU_OK) return AbandonCall(ctx, status);
        EncodeParams p = base;
        p.rows = slot.device[kRowsBuffer].ptr;
        p.rowStride = deviceRowStride;
        p.rowCount = rows;
        for (int i = 0; i < planes; ++i)
        {
            p.plane[out[i].buffer] = slot.device[out[i].buffer].ptr;
            p.planeStride[out[i].buffer] = out[i].deviceStride;
        }
        if (measure && (status = ClearSliceLight(ctx, slot)) != AVIFGPU_OK) return AbandonCall(ctx, status);
        const LightSink light = { slot.lightDevice, levels };
        const int launched = LaunchEncode(p, desc->host_depth, slot.stream, measure ? &light : nullptr);
        if (launched < 0)
        {
            return AbandonCall(ctx, ctx->LaunchFailed(launched, "encode kernel launch"));
        }
        ctx->launches += launched;

        if ((status = StageOut(ctx, slot, out, planes)) != AVIFGPU_OK || (measure && (status = StageLightOut(ctx, slot, acc)) != AVIFGPU_OK) ||
            (status = CloseSlice(ctx, slot, ticket)) != AVIFGPU_OK) return AbandonCall(ctx, status);
    }
    status = FinishCall(ctx, previousRows, ticket, wait);
    if (status == AVIFGPU_OK && !wait && recordedCallRows)
    {
        ctx->asyncEncodeCalls += 1;
        ctx->previousCallRowsPending = true;
    }
    return status;
}

static int DecodeRowsHost(avifgpu_context* ctx, const avifgpu_decode_desc* desc, const avifgpu_planes* src, int32_t y0, int32_t nrows,
                          void* host_rows, int64_t row_stride_bytes, bool wait, int64_t* out_ticket)
{
    if (ctx == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    avifgpu_decode_desc full;
    desc = WidenDecodeDesc(desc, &full);
    std::string error;
    int32_t transfer;
    int status = ValidateDecodeDesc(desc, &transfer, &error);
    if (status != AVIFGPU_OK)
    {
        return ctx->Fail(status, error);
    }
    if (SourceLayoutOf(*desc) != AVIFGPU_SOURCE_PLANAR)
    {
        return ctx->Fail(AVIFGPU_ERR_UNSUPPORTED, "the host-pointer calls read planar, low-bit sources only (libheif's layout)");
    }
    if (src == nullptr || (host_rows == nullptr && nrows > 0 && desc->width > 0))
    {
        return ctx->Fail(AVIFGPU_ERR_BAD_PARAM, "NULL buffer");
    }
    DecodeParams base;
    if (!FillDecodeParams(*desc, transfer, &base, &error))
    {
        return ctx->Fail(AVIFGPU_ERR_UNSUPPORTED, error);
    }
    if (y0 < 0 || nrows < 0 || y0 > desc->height || nrows > desc->height - y0)
    {
        return ctx->Fail(AVIFGPU_ERR_BAD_PARAM, "row block outside the image");
    }
    const int64_t ticket = ++ctx->lastTicket;
    if (out_ticket != nullptr)
    {
        *out_ticket = ticket;
    }
    DeviceGuard guard(ctx->device);
    if (nrows == 0 || desc->width == 0)
    {
        return FinishCall(ctx, TakeRowsRelease(ctx), ticket, wait);
    }
    PlaneGeometry geometry[AVIFGPU_MAX_PLANES];
    bool planePinned[AVIFGPU_MAX_PLANES] = {};
    for (int k = 0; k < AVIFGPU_MAX_PLANES; ++k)
    {
        geometry[k] = DecodePlaneGeometry(*desc, k);
        if (geometry[k].present && src->data[k] == nullptr)
        {
            return ctx->Fail(AVIFGPU_ERR_BAD_PARAM, "missing source plane");
        }
        planePinned[k] = geometry[k].present && IsPinned(src->data[k]);
    }

    ctx->FirstUseDecode(*desc, transfer, false, &base);
    const int64_t rowPayload = static_cast<int64_t>(desc->width) * DecodeHostColBytes(*desc);
    const int64_t deviceRowStride = (rowPayload + 255) & ~255ll;
    const int sliceRows = SliceRows(nrows, rowPayload);
    const bool rowsPinned = IsPinned(host_rows);
    const int previousRows = TakeRowsRelease(ctx);

    for (int begin = 0; begin < nrows; begin += sliceRows)
    {
        const int rows = std::min(sliceRows, nrows - begin);
        int index;
        if ((status = AcquireSlot(ctx, &index)) != AVIFGPU_OK) return AbandonCall(ctx, status);
        Slot& slot = ctx->slots[index];
        const int yFirst = y0 + begin;
        SliceCopy in[AVIFGPU_MAX_PLANES];
        const int planes = PlaneWindows(src, geometry, planePinned, yFirst, rows, in);
        const SliceCopy out{ kRowsBuffer, static_cast<uint8_t*>(host_rows) + static_cast<int64_t>(begin) * row_stride_bytes, row_stride_bytes, rowsPinned, rowPayload, deviceRowStride, rows };
        if ((status = StageIn(ctx, slot, in, planes)) != AVIFGPU_OK ||
            (status = EnsureDeviceStaging(ctx, slot, &out, 1)) != AVIFGPU_OK) return AbandonCall(ctx, status);
        DecodeParams p = base;
        p.rowCount = rows;
        p.yPhase = yFirst & p.ys;
        p.smCount = ctx->smCount;
        for (int i = 0; i < planes; ++i)
        {
            p.plane[in[i].buffer] = slot.device[in[i].buffer].ptr;
            p.planeStride[in[i].buffer] = in[i].deviceStride;
        }
        p.rows = slot.device[kRowsBuffer].ptr;
        p.rowStride = deviceRowStride;
        const int launched = LaunchDecode(p, slot.stream);
        if (launched < 0)
        {
            return AbandonCall(ctx, ctx->LaunchFailed(launched, "decode kernel launch"));
        }
        ctx->launches += launched;

        if ((status = StageOut(ctx, slot, &out, 1)) != AVIFGPU_OK || (status = CloseSlice(ctx, slot, ticket)) != AVIFGPU_OK) return AbandonCall(ctx, status);
    }
    return FinishCall(ctx, previousRows, ticket, wait);
}

extern "C" {

AVIFGPU_EXPORT int avifgpu_encode_rows(avifgpu_context* ctx, const avifgpu_encode_desc* desc, const void* host_rows,
                                       int64_t row_stride_bytes, int32_t y0, int32_t nrows, const avifgpu_planes* dst)
{
    return EncodeRowsHost(ctx, desc, host_rows, row_stride_bytes, y0, nrows, dst, true, nullptr, false, nullptr);
}

AVIFGPU_EXPORT int avifgpu_decode_rows(avifgpu_context* ctx, const avifgpu_decode_desc* desc, const avifgpu_planes* src,
                                       int32_t y0, int32_t nrows, void* host_rows, int64_t row_stride_bytes)
{
    return DecodeRowsHost(ctx, desc, src, y0, nrows, host_rows, row_stride_bytes, true, nullptr);
}

AVIFGPU_EXPORT int avifgpu_encode_rows_async(avifgpu_context* ctx, const avifgpu_encode_desc* desc, const void* host_rows,
                                             int64_t row_stride_bytes, int32_t y0, int32_t nrows, const avifgpu_planes* dst,
                                             int64_t* out_ticket)
{
    return EncodeRowsHost(ctx, desc, host_rows, row_stride_bytes, y0, nrows, dst, false, out_ticket, false, nullptr);
}

AVIFGPU_EXPORT int avifgpu_encode_rows_light_level(avifgpu_context* ctx, const avifgpu_encode_desc* desc, const void* host_rows,
                                                   int64_t row_stride_bytes, int32_t y0, int32_t nrows, const avifgpu_planes* dst,
                                                   avifgpu_light_level* host_acc)
{
    return EncodeRowsHost(ctx, desc, host_rows, row_stride_bytes, y0, nrows, dst, true, nullptr, true, host_acc);
}

AVIFGPU_EXPORT int avifgpu_encode_rows_async_light_level(avifgpu_context* ctx, const avifgpu_encode_desc* desc, const void* host_rows,
                                                         int64_t row_stride_bytes, int32_t y0, int32_t nrows, const avifgpu_planes* dst,
                                                         avifgpu_light_level* host_acc, int64_t* out_ticket)
{
    return EncodeRowsHost(ctx, desc, host_rows, row_stride_bytes, y0, nrows, dst, false, out_ticket, true, host_acc);
}

AVIFGPU_EXPORT int avifgpu_decode_rows_async(avifgpu_context* ctx, const avifgpu_decode_desc* desc, const avifgpu_planes* src,
                                             int32_t y0, int32_t nrows, void* host_rows, int64_t row_stride_bytes, int64_t* out_ticket)
{
    return DecodeRowsHost(ctx, desc, src, y0, nrows, host_rows, row_stride_bytes, false, out_ticket);
}

AVIFGPU_EXPORT int avifgpu_wait(avifgpu_context* ctx, int64_t ticket)
{
    if (ctx == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    DeviceGuard guard(ctx->device);
    if (ticket <= 0 || ticket >= ctx->lastTicket)
    {
        ticket = ctx->lastTicket;
        ctx->previousCallRowsPending = false; // everything is about to be drained
    }
    const int status = RetireThrough(ctx, ticket);
    return status == AVIFGPU_OK ? AVIFGPU_OK : AbandonCall(ctx, status);
}

// ---- several GPUs of one box -----------------------------------------------------------------------------------------

} // extern "C"

struct avifgpu_shard_group
{
    std::vector<avifgpu_context*> members;
    std::vector<int> devices;
    std::vector<uint8_t> peer; // peer[from * n + to]
    std::string lastError;

    int Fail(int status, const std::string& message)
    {
        lastError = message;
        return status;
    }

    // Runs work(r) for every member on its own host thread (each drives its own device and PCIe link); returns the
    // first failure and keeps its message.
    template <typename Work>
    int ForEachMember(Work work)
    {
        const int n = static_cast<int>(members.size());
        std::vector<int> status(n, AVIFGPU_OK);
        std::vector<std::thread> threads;
        threads.reserve(n > 0 ? n - 1 : 0);
        for (int r = 1; r < n; ++r)
        {
            threads.emplace_back([&, r] { status[r] = work(r); });
        }
        if (n > 0)
        {
            status[0] = work(0);
        }
        for (std::thread& t : threads)
        {
            t.join();
        }
        for (int r = 0; r < n; ++r)
        {
            if (status[r] != AVIFGPU_OK)
            {
                return Fail(status[r], "member " + std::to_string(r) + " (device " + std::to_string(devices[r]) + "): " + members[r]->lastError);
            }
        }
        return AVIFGPU_OK;
    }
};

static void RowBlocks(int y0, int nrows, int parts, int32_t* outY0, int32_t* outRows)
{
    // inner boundaries at even image rows: a 2x2 chroma site never straddles two blocks (4:2:0), and the same split
    // serves every other layout
    int previous = y0;
    for (int i = 0; i < parts; ++i)
    {
        int end = (i == parts - 1) ? y0 + nrows : y0 + static_cast<int>((static_cast<int64_t>(nrows) * (i + 1)) / parts);
        if (i != parts - 1)
        {
            end &= ~1;
        }
        end = std::min(std::max(end, previous), y0 + nrows);
        outY0[i] = previous;
        outRows[i] = end - previous;
        previous = end;
    }
}

extern "C" {

AVIFGPU_EXPORT int avifgpu_shard_row_blocks(int32_t y0, int32_t nrows, int32_t parts, int32_t* out_y0, int32_t* out_nrows)
{
    if (parts <= 0 || nrows < 0 || y0 < 0 || out_y0 == nullptr || out_nrows == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    RowBlocks(y0, nrows, parts, out_y0, out_nrows);
    return AVIFGPU_OK;
}

AVIFGPU_EXPORT int avifgpu_shard_group_create(const int32_t* device_ordinals, int32_t count, avifgpu_shard_group** out_group)
{
    if (out_group == nullptr)
    {
        g_creationError = "out_group is NULL";
        return AVIFGPU_ERR_BAD_PARAM;
    }
    *out_group = nullptr;
    if (device_ordinals == nullptr || count <= 0 || count > 64)
    {
        g_creationError = "a shard group needs 1..64 device ordinals";
        return AVIFGPU_ERR_BAD_PARAM;
    }
    for (int i = 0; i < count; ++i)
    {
        for (int j = 0; j < i; ++j)
        {
            if (device_ordinals[i] == device_ordinals[j])
            {
                g_creationError = "device ordinals of a shard group must be distinct";
                return AVIFGPU_ERR_BAD_PARAM;
            }
        }
    }
    avifgpu_shard_group* group = new (std::nothrow) avifgpu_shard_group();
    if (group == nullptr)
    {
        g_creationError = "out of host memory";
        return AVIFGPU_ERR_OOM;
    }
    for (int i = 0; i < count; ++i)
    {
        avifgpu_context* ctx = nullptr;
        const int status = avifgpu_create(device_ordinals[i], &ctx);
        if (status != AVIFGPU_OK)
        {
            avifgpu_shard_group_destroy(group);
            return status; // g_creationError set by avifgpu_create
        }
        group->members.push_back(ctx);
        group->devices.push_back(device_ordinals[i]);
    }
    group->peer.assign(static_cast<size_t>(count) * count, 0);
    for (int from = 0; from < count; ++from)
    {
        DeviceGuard guard(group->devices[from]);
        for (int to = 0; to < count; ++to)
        {
            if (from == to)
            {
                group->peer[from * count + to] = 1;
                continue;
            }
            int can = 0;
            if (cudaDeviceCanAccessPeer(&can, group->devices[from], group->devices[to]) != cudaSuccess || !can)
            {
                cudaGetLastError();
                continue;
            }
            const cudaError_t e = cudaDeviceEnablePeerAccess(group->devices[to], 0);
            if (e == cudaSuccess || e == cudaErrorPeerAccessAlreadyEnabled)
            {
                group->peer[from * count + to] = 1;
            }
            cudaGetLastError();
        }
    }
    *out_group = group;
    return AVIFGPU_OK;
}

AVIFGPU_EXPORT void avifgpu_shard_group_destroy(avifgpu_shard_group* group)
{
    if (group == nullptr)
    {
        return;
    }
    for (avifgpu_context* ctx : group->members)
    {
        avifgpu_destroy(ctx);
    }
    delete group;
}

AVIFGPU_EXPORT int32_t avifgpu_shard_group_size(const avifgpu_shard_group* group) { return group ? static_cast<int32_t>(group->members.size()) : 0; }

AVIFGPU_EXPORT avifgpu_context* avifgpu_shard_group_context(avifgpu_shard_group* group, int32_t index)
{
    return (group != nullptr && index >= 0 && index < static_cast<int32_t>(group->members.size())) ? group->members[index] : nullptr;
}

AVIFGPU_EXPORT int avifgpu_shard_group_peer_access(const avifgpu_shard_group* group, int32_t from, int32_t to)
{
    const int n = group ? static_cast<int>(group->members.size()) : 0;
    return (from >= 0 && to >= 0 && from < n && to < n) ? group->peer[from * n + to] : 0;
}

AVIFGPU_EXPORT const char* avifgpu_shard_group_last_error(const avifgpu_shard_group* group)
{
    return group ? group->lastError.c_str() : g_creationError.c_str();
}

AVIFGPU_EXPORT int avifgpu_shard_group_prepare_encode(avifgpu_shard_group* group, const avifgpu_encode_desc* desc)
{
    if (group == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    avifgpu_encode_desc full;
    desc = WidenEncodeDesc(desc, &full);
    return group->ForEachMember([&](int r) { return avifgpu_prepare_encode(group->members[r], desc, nullptr); });
}

AVIFGPU_EXPORT int avifgpu_shard_group_synchronize(avifgpu_shard_group* group)
{
    if (group == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    int result = AVIFGPU_OK;
    for (size_t r = 0; r < group->members.size(); ++r)
    {
        const int status = avifgpu_synchronize(group->members[r]);
        if (status != AVIFGPU_OK && result == AVIFGPU_OK)
        {
            result = group->Fail(status, "member " + std::to_string(r) + ": " + group->members[r]->lastError);
        }
    }
    return result;
}

} // extern "C"

// The sharded host-pointer encode; `partials` != nullptr: the light-level call, member r adding into partials[r].
static int EncodeRowsSharded(avifgpu_shard_group* group, const avifgpu_encode_desc* desc, const void* host_rows, int64_t row_stride_bytes,
                             int32_t y0, int32_t nrows, const avifgpu_planes* dst, avifgpu_light_level* partials)
{
    const int n = static_cast<int>(group->members.size());
    if (nrows < 0 || y0 < 0)
    {
        return group->Fail(AVIFGPU_ERR_BAD_PARAM, "row block outside the image");
    }
    avifgpu_encode_desc full;
    desc = WidenEncodeDesc(desc, &full);
    if (desc != nullptr && DestLayoutOf(*desc) != AVIFGPU_SOURCE_PLANAR)
    {
        return group->Fail(AVIFGPU_ERR_UNSUPPORTED, "the sharded calls write planar, low-bit planes only (libheif's layout)");
    }
    std::vector<int32_t> blockY0(n), blockRows(n);
    RowBlocks(y0, nrows, n, blockY0.data(), blockRows.data());
    return group->ForEachMember([&](int r) -> int
    {
        if (blockRows[r] == 0 && !(r == 0 && nrows == 0))
        {
            return AVIFGPU_OK;
        }
        const uint8_t* rows = host_rows ? static_cast<const uint8_t*>(host_rows) + static_cast<int64_t>(blockY0[r] - y0) * row_stride_bytes : nullptr;
        return partials != nullptr ? avifgpu_encode_rows_light_level(group->members[r], desc, rows, row_stride_bytes, blockY0[r], blockRows[r], dst, partials + r)
                                   : avifgpu_encode_rows(group->members[r], desc, rows, row_stride_bytes, blockY0[r], blockRows[r], dst);
    });
}

extern "C" {

AVIFGPU_EXPORT int avifgpu_encode_rows_sharded(avifgpu_shard_group* group, const avifgpu_encode_desc* desc, const void* host_rows,
                                               int64_t row_stride_bytes, int32_t y0, int32_t nrows, const avifgpu_planes* dst)
{
    if (group == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    return EncodeRowsSharded(group, desc, host_rows, row_stride_bytes, y0, nrows, dst, nullptr);
}

AVIFGPU_EXPORT int avifgpu_encode_rows_sharded_light_level(avifgpu_shard_group* group, const avifgpu_encode_desc* desc, const void* host_rows,
                                                           int64_t row_stride_bytes, int32_t y0, int32_t nrows, const avifgpu_planes* dst,
                                                           avifgpu_light_level* host_acc)
{
    if (group == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    if (host_acc == nullptr)
    {
        return group->Fail(AVIFGPU_ERR_BAD_PARAM, "NULL light-level accumulator");
    }
    // Each member adds into a zeroed partial of its own; *host_acc changes only once every member has succeeded.
    std::vector<avifgpu_light_level> partials(group->members.size(), avifgpu_light_level{});
    const int status = EncodeRowsSharded(group, desc, host_rows, row_stride_bytes, y0, nrows, dst, partials.data());
    if (status != AVIFGPU_OK)
    {
        return status;
    }
    for (const avifgpu_light_level& part : partials)
    {
        AddLightLevel(*host_acc, part);
    }
    return AVIFGPU_OK;
}

AVIFGPU_EXPORT int avifgpu_decode_rows_sharded(avifgpu_shard_group* group, const avifgpu_decode_desc* desc, const avifgpu_planes* src,
                                               int32_t y0, int32_t nrows, void* host_rows, int64_t row_stride_bytes)
{
    if (group == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    const int n = static_cast<int>(group->members.size());
    if (nrows < 0 || y0 < 0)
    {
        return group->Fail(AVIFGPU_ERR_BAD_PARAM, "row block outside the image");
    }
    if (desc != nullptr && SourceLayoutOf(*desc) != AVIFGPU_SOURCE_PLANAR)
    {
        return group->Fail(AVIFGPU_ERR_UNSUPPORTED, "the sharded calls read planar, low-bit sources only (libheif's layout)");
    }
    std::vector<int32_t> blockY0(n), blockRows(n);
    RowBlocks(y0, nrows, n, blockY0.data(), blockRows.data());
    return group->ForEachMember([&](int r) -> int
    {
        if (blockRows[r] == 0 && !(r == 0 && nrows == 0))
        {
            return AVIFGPU_OK;
        }
        uint8_t* rows = host_rows ? static_cast<uint8_t*>(host_rows) + static_cast<int64_t>(blockY0[r] - y0) * row_stride_bytes : nullptr;
        return avifgpu_decode_rows(group->members[r], desc, src, blockY0[r], blockRows[r], rows, row_stride_bytes);
    });
}

AVIFGPU_EXPORT int avifgpu_encode_rows_sharded_device(avifgpu_shard_group* group, const avifgpu_encode_desc* desc,
                                                      const void* const* device_rows, const int64_t* row_stride_bytes,
                                                      const avifgpu_planes* owner_planes, int32_t owner)
{
    if (group == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    const int n = static_cast<int>(group->members.size());
    if (desc == nullptr || device_rows == nullptr || row_stride_bytes == nullptr || owner_planes == nullptr || owner < 0 || owner >= n)
    {
        return group->Fail(AVIFGPU_ERR_BAD_PARAM, "NULL argument or owner outside the group");
    }
    avifgpu_encode_desc full;
    desc = WidenEncodeDesc(desc, &full);
    if (DestLayoutOf(*desc) != AVIFGPU_SOURCE_PLANAR)
    {
        return group->Fail(AVIFGPU_ERR_UNSUPPORTED, "the sharded calls write planar, low-bit planes only (libheif's layout)");
    }
    std::vector<int32_t> blockY0(n), blockRows(n);
    RowBlocks(0, desc->height, n, blockY0.data(), blockRows.data());
    for (int r = 0; r < n; ++r)
    {
        if (blockRows[r] > 0 && !group->peer[r * n + owner])
        {
            return group->Fail(AVIFGPU_ERR_UNSUPPORTED, "member " + std::to_string(r) + " has no peer access to the owner's memory");
        }
    }
    // Launches are asynchronous: a plain loop enqueues all of them in microseconds, each on its member's own stream.
    for (int r = 0; r < n; ++r)
    {
        if (blockRows[r] == 0)
        {
            continue;
        }
        avifgpu_context* ctx = group->members[r];
        const int status = avifgpu_encode_rows_device(ctx, desc, device_rows[r], row_stride_bytes[r], blockY0[r], blockRows[r], owner_planes,
                                                      ctx->slots[0].stream);
        if (status != AVIFGPU_OK)
        {
            return group->Fail(status, "member " + std::to_string(r) + ": " + ctx->lastError);
        }
    }
    return AVIFGPU_OK;
}

// ---- preparation ------------------------------------------------------------------------------------------------

AVIFGPU_EXPORT int avifgpu_prepare_encode(avifgpu_context* ctx, const avifgpu_encode_desc* desc, avifgpu_curve_stats* out_stats)
{
    if (ctx == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    avifgpu_encode_desc full;
    desc = WidenEncodeDesc(desc, &full);
    std::string error;
    const int status = ValidateEncodeDesc(desc, &error);
    if (status != AVIFGPU_OK)
    {
        return ctx->Fail(status, error);
    }
    DeviceGuard guard(ctx->device);
    CurveTable* table = ctx->CurveTableFor(*desc, 0, true, false);
    ctx->Gray16LutFor(*desc, false);
    if (out_stats != nullptr)
    {
        std::memset(out_stats, 0, sizeof(*out_stats));
        if (table != nullptr)
        {
            out_stats->applicable = 1;
            out_stats->valid = table->valid ? 1 : 0;
            out_stats->steps = table->stats.steps;
            out_stats->bands = table->stats.bands;
            out_stats->widest_band_ulps = table->stats.widestBand;
            out_stats->bucket_count = table->view.bucketCount;
            out_stats->swept_inputs = table->stats.sweptInputs;
            out_stats->in_band_inputs = table->stats.inBandInputs;
            out_stats->verify_mismatches = table->stats.verifyMismatches;
            out_stats->build_ms = table->stats.buildMilliseconds;
        }
    }
    if (table != nullptr && !table->valid)
    {
        ctx->lastError = "step table not used (generic exact kernel serves this configuration): " + table->error;
    }
    return AVIFGPU_OK;
}

AVIFGPU_EXPORT int avifgpu_prepare_decode(avifgpu_context* ctx, const avifgpu_decode_desc* desc)
{
    if (ctx == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    avifgpu_decode_desc full;
    desc = WidenDecodeDesc(desc, &full);
    std::string error;
    int32_t transfer;
    const int status = ValidateDecodeDesc(desc, &transfer, &error);
    if (status != AVIFGPU_OK)
    {
        return ctx->Fail(status, error);
    }
    DecodeParams p;
    if (!FillDecodeParams(*desc, transfer, &p, &error))
    {
        return ctx->Fail(AVIFGPU_ERR_UNSUPPORTED, error);
    }
    DeviceGuard guard(ctx->device);
    ctx->FirstUseDecode(*desc, transfer, false, &p);
    return AVIFGPU_OK;
}

AVIFGPU_EXPORT int avifgpu_set_table_autobuild(avifgpu_context* ctx, int64_t pixels)
{
    if (ctx == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    ctx->tableAutoBuildPixels = pixels;
    return AVIFGPU_OK;
}

// ---- primitives -------------------------------------------------------------------------------------------------

AVIFGPU_EXPORT int avifgpu_transfer_f32(avifgpu_context* ctx, int32_t function, float param, const float* in, float* out, size_t n)
{
    if (ctx == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    if (function < AVIFGPU_FN_LINEAR_TO_PQ || function > AVIFGPU_FN_LOGF)
    {
        return ctx->Fail(AVIFGPU_ERR_BAD_PARAM, "unknown function");
    }
    if (n == 0)
    {
        return AVIFGPU_OK;
    }
    if (in == nullptr || out == nullptr)
    {
        return ctx->Fail(AVIFGPU_ERR_BAD_PARAM, "NULL buffer");
    }
    DeviceGuard guard(ctx->device);
    int status;
    const size_t bytes = n * sizeof(float);
    if ((status = ctx->EnsureDevice(ctx->transferScratch[0], bytes)) != AVIFGPU_OK) return status;
    if ((status = ctx->EnsureDevice(ctx->transferScratch[1], bytes)) != AVIFGPU_OK) return status;
    cudaStream_t stream = ctx->slots[0].stream;
    if ((status = ctx->Cuda(cudaMemcpyAsync(ctx->transferScratch[0].ptr, in, bytes, cudaMemcpyHostToDevice, stream), "H2D")) != AVIFGPU_OK) return status;
    const int launched = LaunchTransfer(function, param, static_cast<const float*>(ctx->transferScratch[0].ptr),
                                        static_cast<float*>(ctx->transferScratch[1].ptr), n, stream);
    if (launched < 0)
    {
        return ctx->LaunchFailed(launched, "transfer kernel launch");
    }
    ctx->launches += launched;
    if ((status = ctx->Cuda(cudaMemcpyAsync(out, ctx->transferScratch[1].ptr, bytes, cudaMemcpyDeviceToHost, stream), "D2H")) != AVIFGPU_OK) return status;
    return ctx->Cuda(cudaStreamSynchronize(stream), "cudaStreamSynchronize");
}

AVIFGPU_EXPORT int avifgpu_hlg_ootf_f32(avifgpu_context* ctx, int32_t inverse, int32_t color_primaries, float display_gamma,
                                        float nominal_peak_nits, const float* rgb_in, float* rgb_out, size_t pixels)
{
    if (ctx == nullptr)
    {
        return AVIFGPU_ERR_BAD_PARAM;
    }
    float luma[3];
    if (!GetHlgLumaCoefficients(color_primaries, luma))
    {
        return ctx->Fail(AVIFGPU_ERR_UNSUPPORTED, "no HLG luma coefficients for these colour primaries");
    }
    if (pixels == 0)
    {
        return AVIFGPU_OK;
    }
    if (rgb_in == nullptr || rgb_out == nullptr)
    {
        return ctx->Fail(AVIFGPU_ERR_BAD_PARAM, "NULL buffer");
    }
    DeviceGuard guard(ctx->device);
    int status;
    const size_t bytes = pixels * 3 * sizeof(float);
    if ((status = ctx->EnsureDevice(ctx->transferScratch[0], bytes)) != AVIFGPU_OK) return status;
    if ((status = ctx->EnsureDevice(ctx->transferScratch[1], bytes)) != AVIFGPU_OK) return status;
    cudaStream_t stream = ctx->slots[0].stream;
    if ((status = ctx->Cuda(cudaMemcpyAsync(ctx->transferScratch[0].ptr, rgb_in, bytes, cudaMemcpyHostToDevice, stream), "H2D")) != AVIFGPU_OK) return status;
    const int launched = LaunchHlgOotf(inverse != 0, luma, display_gamma, nominal_peak_nits, static_cast<const float*>(ctx->transferScratch[0].ptr),
                                       static_cast<float*>(ctx->transferScratch[1].ptr), pixels, stream);
    if (launched < 0)
    {
        return ctx->LaunchFailed(launched, "OOTF kernel launch");
    }
    ctx->launches += launched;
    if ((status = ctx->Cuda(cudaMemcpyAsync(rgb_out, ctx->transferScratch[1].ptr, bytes, cudaMemcpyDeviceToHost, stream), "D2H")) != AVIFGPU_OK) return status;
    return ctx->Cuda(cudaStreamSynchronize(stream), "cudaStreamSynchronize");
}

} // extern "C"
