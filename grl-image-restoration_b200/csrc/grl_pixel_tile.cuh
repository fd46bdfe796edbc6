// grl_pixel_tile.cuh -- the 32 x 32 pixel tile between 8-bit HWC pixels and fp32 CHW planes, shared by the conversion
// kernels (image_u8.cu) and the image-list gather / crop (image_list.cu).
//
// A CTA of 32 x 8 threads owns one tile.  The 8-bit side of a tile row is one run of (pixels x C) contiguous bytes, walked
// byte by byte with threadIdx.x; the fp32 side is C runs of 32 floats, walked with threadIdx.x as well.  The bytes are
// staged in shared memory between the two, so every global load and store is coalesced.  The callers supply the
// addressing as functors, so the same staging serves whole images, padded batches and crops.
#pragma once

#include <stdint.h>

#include "grl_image_u8.h"

namespace grl {

constexpr int kTile = 32, kTileRows = 8, kTileMaxC = 8;  // 32 x 8 threads, 4 rows each; 1 <= C <= 8
constexpr int kTileMinBlocks = 8;  // 8 CTAs of 256 threads fill an SM: caps the tile kernels at 32 registers

using PixelTile = uint8_t[kTile][kTile * kTileMaxC];

// tile[r][i] = at(r, i) for the `rows` tile rows and the `run` bytes (pixels x C) of each: byte i is channel i % C of
// pixel i / C.
template <class At>
__device__ __forceinline__ void tile_load_u8(PixelTile& tile, int rows, int run, At at) {
  for (int r = threadIdx.y; r < rows; r += kTileRows)
    for (int i = threadIdx.x; i < run; i += kTile) tile[r][i] = at(r, i);
}

// put(r, i, byte) for the same bytes.
template <class Put>
__device__ __forceinline__ void tile_store_u8(const PixelTile& tile, int rows, int run, Put put) {
  for (int r = threadIdx.y; r < rows; r += kTileRows)
    for (int i = threadIdx.x; i < run; i += kTile) put(r, i, tile[r][i]);
}

// put(c, r, u8_unit(byte)) for channel c of the pixel of column threadIdx.x < cols in tile row r.
template <class Put>
__device__ __forceinline__ void tile_store_f32(const PixelTile& tile, int rows, int cols, int C, Put put) {
  if ((int)threadIdx.x >= cols) return;
  for (int c = 0; c < C; ++c)
    for (int r = threadIdx.y; r < rows; r += kTileRows) put(c, r, u8_unit(tile[r][threadIdx.x * C + c]));
}

// The byte round8(get(c, r)) for channel c of the pixel of column threadIdx.x < cols in tile row r.
template <class Get>
__device__ __forceinline__ void tile_load_f32(PixelTile& tile, int rows, int cols, int C, Get get) {
  if ((int)threadIdx.x >= cols) return;
  for (int c = 0; c < C; ++c)
    for (int r = threadIdx.y; r < rows; r += kTileRows) tile[r][threadIdx.x * C + c] = (uint8_t)round8(get(c, r));
}

}  // namespace grl
