// tests/native/shuttle_light_level_test.cpp -- the row shuttle's content light level (avifgpu_host::SetContentLightLevelEnabled):
// 32-bit PQ saves through CreateHeifImage{RGB,Gray}ThirtyTwoBit with a mock Photoshop host and the mock libheif
// (oracle/shim/mock_heif.cpp), the attached `clli` compared with MaxCLL / MaxFALL of the CPU oracle's reference-layout
// codes (oracle_light_level.h).  libheif's content light level calls come from tests/native/mock_heif_content_light_level.cpp.
// Built against libavifgpu.so by tests/test_gpu_shuttle_light_level.py (needs an H100), and by
// tests/test_shuttle_light_level_cpu.py against tests/native/fake_avifgpu_on_oracle.cpp with
// tests/native/fake_light_level_on_oracle.cpp.  Exit code 0 = all passed.
#include "GpuRowShuttle.h"
#include "oracle_light_level.h"

#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

namespace
{
    struct MockHost
    {
        FormatRecord record{};
        BufferProcs procs{};
        const uint8_t* source = nullptr;
        int64_t stride = 0;
        int advanceCalls = 0;
        int abortAfterCalls = -1;
    };
    MockHost* g_host = nullptr;

    OSErr Advance()
    {
        MockHost& h = *g_host;
        FormatRecord& r = h.record;
        h.advanceCalls++;
        for (int y = r.theRect32.top; y < r.theRect32.bottom; ++y)
        {
            std::memcpy(static_cast<uint8_t*>(r.data) + static_cast<int64_t>(y - r.theRect32.top) * r.rowBytes, h.source + y * h.stride,
                        static_cast<size_t>(h.stride));
        }
        return noErr;
    }
    Boolean Abort() { return g_host->abortAfterCalls >= 0 && g_host->advanceCalls >= g_host->abortAfterCalls; }
    void Progress(int32, int32) {}

    void InitHost(MockHost& h, int w, int hgt, int channels, int depth, const void* rows)
    {
        FormatRecord& r = h.record;
        r.planes = static_cast<int16>(channels);
        r.depth = static_cast<int16>(depth);
        r.imageSize32.h = w;
        r.imageSize32.v = hgt;
        r.HostSupports32BitCoordinates = 1;
        r.PluginUsing32BitCoordinates = 1;
        r.advanceState = Advance;
        r.abortProc = Abort;
        r.progressProc = Progress;
        r.bufferProcs = &h.procs;
        h.source = static_cast<const uint8_t*>(rows);
        h.stride = static_cast<int64_t>(w) * channels * (depth / 8);
        g_host = &h;
    }

    // Every image stays alive to the end: the content light level stand-in keys its values by image address.
    std::vector<ScopedHeifImage> g_images;
    const heif_image* Keep(ScopedHeifImage image)
    {
        g_images.push_back(std::move(image));
        return g_images.back().get();
    }

    int g_failures = 0;
    void Expect(bool ok, const char* what)
    {
        std::printf("%s %s\n", ok ? "PASS" : "FAIL", what);
        if (!ok) ++g_failures;
    }

    // MaxCLL / MaxFALL (cd/m2) of an accumulator, as CTA-861.3 rounds them up: ceil(10000 level(max_code) / 2^22) and
    // ceil(10000 level_sum / (2^22 pixels)), in 128-bit integers.
    void CtaValues(const avifgpu_light_level& acc, int depth, uint16_t* maxCll, uint16_t* maxFall)
    {
        using Wide = unsigned __int128;
        const uint32_t maxCode = (1u << depth) - 1u;
        const Wide peak = avifgpu::LightLevelOf(acc.max_code, static_cast<float>(maxCode), avifmath::HostLibmTables());
        const Wide scale = Wide(1) << 22;
        *maxCll = acc.pixels ? static_cast<uint16_t>((Wide(10000) * peak + scale - 1) / scale) : 0;
        const Wide denominator = scale * acc.pixels;
        *maxFall = acc.pixels ? static_cast<uint16_t>((Wide(10000) * acc.level_sum + denominator - 1) / denominator) : 0;
    }

    std::vector<float> Rows(int w, int h, int channels, uint32_t seed)
    {
        std::mt19937 rng(seed);
        std::uniform_real_distribution<float> dist(-0.1f, 1.3f);
        std::vector<float> rows(static_cast<size_t>(w) * h * channels);
        for (float& v : rows) v = dist(rng);
        rows[rows.size() / 2] = 90.0f; // one pixel above the peak (the 80-nit scale puts 1.0 at 80 cd/m2)
        return rows;
    }

    struct Save
    {
        const char* name;
        bool gray;
        int channels;
        AlphaState alpha;
        ChromaSubsampling chroma;
        bool lossless;
        ImageBitDepth depth;
        int bits;
    };

    avifgpu_encode_desc DescOf(const Save& s, int w, int h)
    {
        avifgpu_encode_desc d{};
        d.struct_size = sizeof(d);
        d.width = w; d.height = h; d.host_depth = 32; d.host_channels = s.channels; d.alpha_state = static_cast<int>(s.alpha);
        d.image_bit_depth = s.bits; d.transfer = AVIFGPU_TRANSFER_PQ; d.pq_peak_nits = 80;
        d.layout = s.gray ? AVIFGPU_LAYOUT_REFERENCE : AVIFGPU_LAYOUT_PLANAR_YCBCR;
        return d;
    }

    ScopedHeifImage SaveThroughShuttle(const Save& s, MockHost& host, int w, int h, ColorTransferFunction transfer)
    {
        SaveUIOptions options{};
        options.chromaSubsampling = s.chroma;
        options.lossless = s.lossless;
        options.imageBitDepth = s.depth;
        options.hdrTransferFunction = transfer;
        options.pq.nominalPeakBrightness = 80;
        avifgpu_host::SetRowsPerBlock(6);
        const VPoint size{ h, w };
        return s.gray ? CreateHeifImageGrayThirtyTwoBit(&host.record, s.alpha, size, options)
                      : CreateHeifImageRGBThirtyTwoBit(&host.record, s.alpha, size, options);
    }

    void TestMeasuredSave(const Save& s, int w, int h)
    {
        const std::vector<float> rows = Rows(w, h, s.channels, 99u + static_cast<uint32_t>(w));
        MockHost host;
        InitHost(host, w, h, s.channels, 32, rows.data());
        avifgpu_host::SetContentLightLevelEnabled(true);
        const heif_image* image = Keep(SaveThroughShuttle(s, host, w, h, ColorTransferFunction::PQ));
        avifgpu_light_level acc{};
        const int status = OracleLightLevel(DescOf(s, w, h), rows.data(), host.stride, h, &acc);
        uint16_t maxCll = 0, maxFall = 0;
        CtaValues(acc, s.bits, &maxCll, &maxFall);
        heif_content_light_level clli{};
        const bool has = heif_image_has_content_light_level(image) != 0;
        heif_image_get_content_light_level(image, &clli);
        const avifgpu_host::ContentLightLevel last = avifgpu_host::LastContentLightLevel();
        char label[200];
        std::snprintf(label, sizeof(label), "%s %dx%d in %d blocks: clli attached = oracle codes' MaxCLL %u / MaxFALL %u (got %u / %u), reported alike",
                      s.name, w, h, host.advanceCalls, maxCll, maxFall, clli.max_content_light_level, clli.max_pic_average_light_level);
        Expect(status == 0 && has && host.advanceCalls > 1 && acc.pixels == static_cast<uint64_t>(w) * h && maxCll > 0 &&
                   clli.max_content_light_level == maxCll && clli.max_pic_average_light_level == maxFall && last.measured &&
                   last.maxCll == maxCll && last.maxFall == maxFall,
               label);
    }

    // A stand-in for the plug-in's lcms2 transform (halves every colour sample, exactly): the statistic covers the rows
    // as transformed, not as the host handed them out.
    struct HalvingTransform final : avifgpu_host::RowTransform
    {
        void ConvertRow(void* row, uint32_t pixelsPerLine, uint32_t) override
        {
            float* v = static_cast<float*>(row);
            for (uint32_t i = 0; i < pixelsPerLine * 3; ++i) v[i] *= 0.5f;
        }
    };
    avifgpu_host::RowTransform* HalvingFactory(FormatRecordPtr, bool, int hostBits, ColorTransferFunction, bool, void*)
    {
        return hostBits == 32 ? new HalvingTransform() : nullptr;
    }

    void TestAfterRowTransform()
    {
        const int w = 40, h = 22;
        const Save s{ "RGB32f PQ 4:4:4 12-bit with a row transform", false, 3, AlphaState::None, ChromaSubsampling::Yuv444, false, ImageBitDepth::Twelve, 12 };
        const std::vector<float> rows = Rows(w, h, 3, 5);
        static const unsigned char fakeProfile[16] = { 1 };
        MockHost host;
        InitHost(host, w, h, 3, 32, rows.data());
        host.record.canUseICCProfiles = 1;
        host.record.iCCprofileData = const_cast<unsigned char*>(fakeProfile);
        host.record.iCCprofileSize = sizeof(fakeProfile);
        avifgpu_host::SetRowTransformFactory(HalvingFactory, nullptr);
        avifgpu_host::SetContentLightLevelEnabled(true);
        const heif_image* image = Keep(SaveThroughShuttle(s, host, w, h, ColorTransferFunction::PQ));
        avifgpu_host::SetRowTransformFactory(nullptr, nullptr);
        std::vector<float> halved(rows);
        for (float& v : halved) v *= 0.5f;
        avifgpu_light_level acc{};
        const int status = OracleLightLevel(DescOf(s, w, h), halved.data(), host.stride, h, &acc);
        uint16_t maxCll = 0, maxFall = 0;
        CtaValues(acc, 12, &maxCll, &maxFall);
        heif_content_light_level clli{};
        heif_image_get_content_light_level(image, &clli);
        Expect(status == 0 && heif_image_has_content_light_level(image) && clli.max_content_light_level == maxCll &&
                   clli.max_pic_average_light_level == maxFall,
               "row transform: clli measured on the transformed rows");
    }

    void TestNothingAttached()
    {
        const int w = 36, h = 14;
        const Save rgb{ "RGB32f", false, 3, AlphaState::None, ChromaSubsampling::Yuv420, false, ImageBitDepth::Twelve, 12 };
        const std::vector<float> rows = Rows(w, h, 3, 11);
        {
            MockHost host;
            InitHost(host, w, h, 3, 32, rows.data());
            avifgpu_host::SetContentLightLevelEnabled(false);
            const heif_image* image = Keep(SaveThroughShuttle(rgb, host, w, h, ColorTransferFunction::PQ));
            Expect(!heif_image_has_content_light_level(image) && !avifgpu_host::LastContentLightLevel().measured,
                   "switch off (the default): a PQ save attaches no clli");
        }
        avifgpu_host::SetContentLightLevelEnabled(true);
        {
            MockHost host;
            InitHost(host, w, h, 3, 32, rows.data());
            const heif_image* image = Keep(SaveThroughShuttle(rgb, host, w, h, ColorTransferFunction::SMPTE428));
            Expect(!heif_image_has_content_light_level(image) && !avifgpu_host::LastContentLightLevel().measured,
                   "switch on, SMPTE 428 save: no clli");
        }
        {
            std::vector<uint8_t> bytes(static_cast<size_t>(w) * h * 3, 200);
            MockHost host;
            InitHost(host, w, h, 3, 8, bytes.data());
            SaveUIOptions options{};
            options.chromaSubsampling = ChromaSubsampling::Yuv420;
            options.imageBitDepth = ImageBitDepth::Ten;
            options.hdrTransferFunction = ColorTransferFunction::PQ; // ignored by 8-bit saves
            const heif_image* image = Keep(CreateHeifImageRGBEightBit(&host.record, AlphaState::None, VPoint{ h, w }, options));
            Expect(!heif_image_has_content_light_level(image) && !avifgpu_host::LastContentLightLevel().measured,
                   "switch on, 8-bit save: no clli");
        }
        {
            TestMeasuredSave(rgb, w, h); // a measured save first, so that a stale report would show
            MockHost host;
            InitHost(host, w, h, 3, 32, rows.data());
            host.abortAfterCalls = 2;
            bool canceled = false;
            try { SaveThroughShuttle(rgb, host, w, h, ColorTransferFunction::PQ); }
            catch (const OSErrException& e) { canceled = e.GetErrorCode() == userCanceledErr; }
            Expect(canceled && !avifgpu_host::LastContentLightLevel().measured, "switch on, cancelled save: userCanceledErr, nothing measured");
        }
        avifgpu_host::SetContentLightLevelEnabled(false);
    }
}

int main()
{
    try
    {
        TestMeasuredSave({ "RGB32f PQ 4:2:0 12-bit", false, 3, AlphaState::None, ChromaSubsampling::Yuv420, false, ImageBitDepth::Twelve, 12 }, 70, 21);
        TestMeasuredSave({ "RGB32f PQ lossless 4:4:4 10-bit", false, 3, AlphaState::None, ChromaSubsampling::Yuv420, true, ImageBitDepth::Ten, 10 }, 33, 17);
        TestMeasuredSave({ "RGBA32f PQ 4:2:2 12-bit", false, 4, AlphaState::Straight, ChromaSubsampling::Yuv422, false, ImageBitDepth::Twelve, 12 }, 64, 16);
        TestMeasuredSave({ "Gray32f PQ 10-bit", true, 1, AlphaState::None, ChromaSubsampling::Yuv420, false, ImageBitDepth::Ten, 10 }, 45, 13);
        TestMeasuredSave({ "Gray+A 32f PQ 12-bit", true, 2, AlphaState::Straight, ChromaSubsampling::Yuv420, false, ImageBitDepth::Twelve, 12 }, 29, 9);
        TestAfterRowTransform();
        TestNothingAttached();
    }
    catch (const std::exception& e)
    {
        std::printf("FAIL unexpected exception: %s\n", e.what());
        ++g_failures;
    }
    g_images.clear();
    avifgpu_host::ReleaseSharedContext();
    std::printf("%s\n", g_failures == 0 ? "ALL PASSED" : "SOME FAILED");
    return g_failures == 0 ? 0 : 1;
}
