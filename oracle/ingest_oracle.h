// CPU restatement of the frame ingest (orb_ingest.cpp): test infrastructure, never product.
#pragma once
#include <cstddef>
#include <cstdint>

extern "C" {
void orc_gray_from_color(const uint8_t* src, size_t src_row_bytes, int width, int height, int channels, int rgb,
                         uint8_t* out, size_t out_row_bytes);
void orc_remap_linear(const uint8_t* src, size_t src_row_bytes, int src_width, int src_height, int channels,
                      const float* mapx, const float* mapy, size_t map_row_bytes, int width, int height, uint8_t* dst);
float orc_depth_u16(const uint16_t* raw, size_t n, float depth_map_factor, float* out);
}
