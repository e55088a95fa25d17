// tests/native/fake_light_level_on_oracle.cpp -- TEST INFRASTRUCTURE: the single-context light-level host encodes
// (avifgpu_encode_rows_light_level, avifgpu_encode_rows_async_light_level) for programs linked with the oracle-backed
// stand-in tests/native/fake_avifgpu_on_oracle.cpp.  The planes come from the stand-in's own encode calls; the statistic
// of the rows is added from the CPU oracle's reference-layout codes (oracle_light_level.h).  Linked by
// tests/test_shuttle_light_level_cpu.py; never part of the product.
#include "oracle_light_level.h"

namespace
{
    // The light-level calls' own checks (include/avifgpu.h): float-host PQ encodes only, and an accumulator.
    int CheckLightLevelCall(const avifgpu_context* ctx, const avifgpu_encode_desc* desc, const avifgpu_light_level* acc)
    {
        if (ctx == nullptr || desc == nullptr)
        {
            return AVIFGPU_ERR_BAD_PARAM;
        }
        if (desc->host_depth != 32 || desc->transfer != AVIFGPU_TRANSFER_PQ)
        {
            return AVIFGPU_ERR_UNSUPPORTED;
        }
        return acc == nullptr ? AVIFGPU_ERR_BAD_PARAM : AVIFGPU_OK;
    }

    int Measure(int status, const avifgpu_encode_desc* desc, const void* host_rows, int64_t row_stride_bytes, int32_t nrows, avifgpu_light_level* acc)
    {
        return status == AVIFGPU_OK ? OracleLightLevel(*desc, host_rows, row_stride_bytes, nrows, acc) : status;
    }
}

extern "C" {

int avifgpu_encode_rows_light_level(avifgpu_context* ctx, const avifgpu_encode_desc* desc, const void* host_rows, int64_t row_stride_bytes,
                                    int32_t y0, int32_t nrows, const avifgpu_planes* dst, avifgpu_light_level* host_acc)
{
    const int status = CheckLightLevelCall(ctx, desc, host_acc);
    if (status != AVIFGPU_OK)
    {
        return status;
    }
    return Measure(avifgpu_encode_rows(ctx, desc, host_rows, row_stride_bytes, y0, nrows, dst), desc, host_rows, row_stride_bytes, nrows, host_acc);
}

int avifgpu_encode_rows_async_light_level(avifgpu_context* ctx, const avifgpu_encode_desc* desc, const void* host_rows, int64_t row_stride_bytes,
                                          int32_t y0, int32_t nrows, const avifgpu_planes* dst, avifgpu_light_level* host_acc, int64_t* out_ticket)
{
    const int status = CheckLightLevelCall(ctx, desc, host_acc);
    if (status != AVIFGPU_OK)
    {
        return status;
    }
    return Measure(avifgpu_encode_rows_async(ctx, desc, host_rows, row_stride_bytes, y0, nrows, dst, out_ticket), desc, host_rows, row_stride_bytes,
                   nrows, host_acc);
}

} // extern "C"
