// tests/native/oracle_light_level.h -- TEST INFRASTRUCTURE: the content light level (avifgpu_light_level, DESIGN.md
// section 5) of host rows from the CPU oracle's own codes.  The reference-layout encode of the rows gives each pixel's
// transfer-curve codes interleaved (after clamp, premultiplication and row matrix); k = max(R', G', B') (the Y code for
// gray hosts), and level(k) is LightLevelOf (avif-format_b200/csrc/light_level.cuh), the host arithmetic the library
// builds its level tables with.  Used by the oracle-backed stand-in of the light-level calls and by the shuttle's
// light-level test.
#ifndef TESTS_NATIVE_ORACLE_LIGHT_LEVEL_H
#define TESTS_NATIVE_ORACLE_LIGHT_LEVEL_H

#include "../../include/avifgpu.h"
#include "../../oracle/avif_oracle.h"
#include "light_level.cuh"

#include <algorithm>
#include <vector>

// Adds the statistic of `nrows` rows of `desc`'s width into *acc; returns the oracle's status.
inline int OracleLightLevel(const avifgpu_encode_desc& desc, const void* rows, int64_t rowStride, int32_t nrows, avifgpu_light_level* acc)
{
    if (nrows == 0 || desc.width == 0)
    {
        return 0;
    }
    avifgpu_encode_desc ref = desc;
    ref.layout = AVIFGPU_LAYOUT_REFERENCE;
    ref.chroma = AVIFGPU_CHROMA_444;
    ref.dest_layout = 0;
    ref.height = nrows;
    const bool colour = desc.host_channels >= 3;
    const int interleaved = colour ? desc.host_channels : 1; // gray: Y in plane 0, alpha in plane 3
    std::vector<uint16_t> codes(static_cast<size_t>(desc.width) * nrows * interleaved), alpha(static_cast<size_t>(desc.width) * nrows);
    avifgpu_planes planes{};
    planes.data[0] = codes.data();
    planes.stride[0] = static_cast<int64_t>(desc.width) * interleaved * 2;
    if (!colour && desc.host_channels == 2)
    {
        planes.data[3] = alpha.data();
        planes.stride[3] = static_cast<int64_t>(desc.width) * 2;
    }
    const int status = avif_oracle_encode_image(&ref, rows, rowStride, &planes);
    if (status != 0)
    {
        return status;
    }
    const uint32_t maxCode = (1u << desc.image_bit_depth) - 1u;
    std::vector<uint32_t> levels(maxCode + 1);
    const avifmath::LibmTables tables = avifmath::HostLibmTables();
    for (uint32_t k = 0; k <= maxCode; ++k)
    {
        levels[k] = avifgpu::LightLevelOf(k, static_cast<float>(maxCode), tables);
    }
    const size_t pixels = static_cast<size_t>(desc.width) * nrows;
    for (size_t i = 0; i < pixels; ++i)
    {
        const uint16_t* c = codes.data() + i * interleaved;
        const uint32_t k = colour ? std::max({ c[0], c[1], c[2] }) : c[0];
        acc->max_code = std::max(acc->max_code, k);
        acc->level_sum += levels[k];
    }
    acc->pixels += pixels;
    return 0;
}

#endif
