// grl_tiles.h -- the tile grid of tiled inference (engines/base.py:90-116, tiling.forward_tile) as closed forms shared by
// the host expansion grl_tile_cover_host (capi.cu) and the overlap-blend kernels (image_list.cu).
//
// On an axis of `size` samples with tile side t (1 <= t <= size) and overlap 0 <= overlap < t, tiling.tile_origins is
// range(0, size - t, stride) + [size - t] with stride = t - overlap: origin k * stride for k < n - 1, then size - t, where
// n = ceil((size - t) / stride) + 1.  The origins strictly increase and every tile has the same side, so the tiles that
// cover sample r are one run [tile_first, tile_last] in origin order, and the blend's divisor at output pixel (Y, X) of
// an x`scale` model is the exact float (run length of Y / scale on the row axis) * (run length of X / scale on the
// column axis).
#pragma once

#include "grl_hd.h"

namespace grl {

struct TileAxis {
  int size, t, stride, n;
};

GRL_HD TileAxis tile_axis(int size, int t, int overlap) {
  const int stride = t - overlap;
  return {size, t, stride, (size - t + stride - 1) / stride + 1};
}

GRL_HD int tile_origin(const TileAxis& a, int k) { return k < a.n - 1 ? k * a.stride : a.size - a.t; }

// The first tile whose window reaches past sample r: the first k < n - 1 with k * stride + t > r, else the last tile.
GRL_HD int tile_first(const TileAxis& a, int r) {
  const int k = r < a.t ? 0 : (r - a.t) / a.stride + 1;
  return k < a.n - 1 ? k : a.n - 1;
}

// The last tile whose origin is at or before sample r: the last tile once r >= size - t, else the last k * stride <= r
// (which is below n - 1, since (n - 1) * stride >= size - t).
GRL_HD int tile_last(const TileAxis& a, int r) { return r >= a.size - a.t ? a.n - 1 : r / a.stride; }

}  // namespace grl
