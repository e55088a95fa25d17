// Writes level(k) of every code of one image depth (avif-format_b200/csrc/light_level.cuh, the host arithmetic the library
// builds its level tables with) to stdout as native uint32 words, for tests/test_light_level.py.
#include "light_level.cuh"

#include <cstdio>
#include <cstdlib>
#include <vector>

int main(int argc, char** argv)
{
    if (argc != 2)
    {
        std::fprintf(stderr, "usage: %s image_bit_depth\n", argv[0]);
        return 2;
    }
    const int depth = std::atoi(argv[1]);
    const uint32_t count = 1u << depth;
    const avifmath::LibmTables tables = avifmath::HostLibmTables();
    std::vector<uint32_t> levels(count);
    for (uint32_t k = 0; k < count; ++k)
    {
        levels[k] = avifgpu::LightLevelOf(k, static_cast<float>(count - 1), tables);
    }
    return std::fwrite(levels.data(), sizeof(uint32_t), count, stdout) == count ? 0 : 1;
}
