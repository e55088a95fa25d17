// tests/native/mock_heif_content_light_level.cpp -- TEST INFRASTRUCTURE ONLY: libheif's content light level calls
// (heif_image_set_content_light_level, heif_image_has_content_light_level, heif_image_get_content_light_level: the values
// libheif writes as the `clli` property) for images of the mock libheif (oracle/shim/mock_heif.cpp), which has none.
// Written from the public API description.  The values are kept beside the images, keyed by image: a program that links
// this keeps every image it checks alive, so no image address is reused while its entry exists.
#include "compat/PluginTypes.h"

#include <map>

namespace
{
    std::map<const heif_image*, heif_content_light_level> g_contentLightLevels;
}

extern "C" {

void heif_image_set_content_light_level(const heif_image* image, const heif_content_light_level* in)
{
    if (image != nullptr && in != nullptr)
    {
        g_contentLightLevels[image] = *in;
    }
}

int heif_image_has_content_light_level(const heif_image* image) { return g_contentLightLevels.count(image) ? 1 : 0; }

void heif_image_get_content_light_level(const heif_image* image, heif_content_light_level* out)
{
    const auto it = g_contentLightLevels.find(image);
    if (it != g_contentLightLevels.end() && out != nullptr)
    {
        *out = it->second;
    }
}

} // extern "C"
