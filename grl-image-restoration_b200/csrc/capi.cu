// capi.cu -- the parts of the extern "C" surface (include/grl_b200.h) that launch nothing: the error buffer and launch
// counter every entry point reports through, and the host expansions of the geometry closed forms.  Each entry point that
// launches a kernel is defined beside that kernel.
#include <math.h>

#include "grl_common.cuh"
#include "grl_tiles.h"

namespace grl {
char* error_buffer() {
  static thread_local char buf[512] = {0};
  return buf;
}
unsigned long long& launch_counter() {
  static unsigned long long n = 0;
  return n;
}
}  // namespace grl

using namespace grl;

extern "C" {

const char* grl_last_error(void) { return error_buffer(); }
int grl_abi_version(void) { return GRL_B200_ABI_VERSION; }
uint64_t grl_launch_count(void) { return launch_counter(); }

int grl_device_ok(void) {
  int dev = 0, major = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return 0;
  return major == 9;
}

// ---------------------------------------------------------------- geometry (host)
int grl_rel_index_host(int wh, int ww, int df, int window_to_anchor, int64_t* out) {
  GRL_REQUIRE(wh > 0 && ww > 0 && df > 0 && out, "rel_index: bad arguments");
  const int awh = wh / df, aww = ww / df;
  const int n1 = window_to_anchor ? wh * ww : awh * aww;
  const int n2 = window_to_anchor ? awh * aww : wh * ww;
  const int qww = window_to_anchor ? ww : aww;
  const int kwh = window_to_anchor ? awh : wh, kww = window_to_anchor ? aww : ww;
  for (int i = 0; i < n1; ++i)
    for (int j = 0; j < n2; ++j)
      out[(size_t)i * n2 + j] = rel_index(i / qww, i % qww, j / kww, j % kww, qww, kwh, kww);
  return GRL_OK;
}

int grl_token_map_host(GrlGrid g, int32_t* out) {
  GRL_REQUIRE(out != nullptr, "token_map: null output");
  int rc;
  if ((rc = check_grid(g, "token_map")) != GRL_OK) return rc;
  const int nwh = g.H / g.wh, nww = g.W / g.ww, n = g.wh * g.ww;
  for (int wr = 0; wr < nwh; ++wr)
    for (int wc = 0; wc < nww; ++wc)
      for (int i = 0; i < n; ++i) {
        const Tok t = locate(g, wr, wc, i);
        out[((size_t)wr * nww + wc) * n + i] = t.y * g.W + t.x;
      }
  return GRL_OK;
}

int grl_shift_mask_host(int H, int W, int wh, int ww, int sh, int sw, int df, int window_to_anchor, float* out) {
  GRL_REQUIRE(df > 0 && out, "shift_mask: bad arguments");
  GrlGrid gt = {H, W, wh, ww, sh, sw};
  GrlGrid ga = {H / df, W / df, wh / df, ww / df, sh / df, sw / df};
  int rc;
  if ((rc = check_grid(gt, "shift_mask(tokens)")) != GRL_OK) return rc;
  if ((rc = check_grid(ga, "shift_mask(anchors)")) != GRL_OK) return rc;
  const GrlGrid& gq = window_to_anchor ? gt : ga;
  const GrlGrid& gk = window_to_anchor ? ga : gt;
  const int n1 = gq.wh * gq.ww, n2 = gk.wh * gk.ww;
  const int nwh = gq.H / gq.wh, nww = gq.W / gq.ww;
  for (int wr = 0; wr < nwh; ++wr)
    for (int wc = 0; wc < nww; ++wc) {
      float* o = out + (size_t)(wr * nww + wc) * n1 * n2;
      for (int i = 0; i < n1; ++i) {
        Tok tq = locate(gq, wr, wc, i);
        const int rq = region_id(gq, tq.r, tq.c);
        for (int j = 0; j < n2; ++j) {
          Tok tk = locate(gk, wr, wc, j);
          o[(size_t)i * n2 + j] = (rq != region_id(gk, tk.r, tk.c)) ? -100.0f : 0.0f;
        }
      }
    }
  return GRL_OK;
}

int grl_coords_table_host(int wh, int ww, int df, float* out) {
  GRL_REQUIRE(wh > 0 && ww > 0 && df > 0 && out, "coords_table: bad arguments");
  const int ws[2] = {wh, ww}, aws[2] = {wh / df, ww / df};
  int hi[2], lo[2];
  for (int a = 0; a < 2; ++a) {
    hi[a] = ws[a] - 1 - (ws[a] - aws[a]) / 2;
    lo[a] = -(aws[a] - 1) - (ws[a] - aws[a]) / 2;
  }
  const int nh = hi[0] - lo[0] + 1, nw = hi[1] - lo[1] + 1;
  // same operation order as ops.py:257-269: v / hi (fp32), * 8 (fp32), sign * log2(|v| + 1) (fp32), then a
  // division by the float64 scalar np.log2(8) == 3.0 carried out in fp32 (torch keeps the tensor dtype).
  for (int i = 0; i < nh; ++i)
    for (int j = 0; j < nw; ++j) {
      const int c[2] = {lo[0] + i, lo[1] + j};
      for (int a = 0; a < 2; ++a) {
        float v = (float)c[a] / (float)hi[a];
        v = v * 8.0f;
        float s = (v > 0.f) ? 1.f : (v < 0.f ? -1.f : 0.f);
        out[((size_t)i * nw + j) * 2 + a] = s * log2f(fabsf(v) + 1.0f) / 3.0f;
      }
    }
  return GRL_OK;
}

// ---------------------------------------------------------------- tiled inference (host)
int grl_tile_cover_host(int size, int tile, int overlap, int scale, int32_t* out) {
  GRL_REQUIRE(out, "tile_cover: null output");
  GRL_REQUIRE(tile >= 1 && tile <= size && overlap >= 0 && overlap < tile && scale >= 1,
              "tile_cover: needs 1 <= tile <= size, 0 <= overlap < tile, scale >= 1 (size %d, tile %d, overlap %d, scale %d)",
              size, tile, overlap, scale);
  const TileAxis a = tile_axis(size, tile, overlap);
  for (int Y = 0; Y < size * scale; ++Y) {
    out[2 * Y] = tile_first(a, Y / scale);
    out[2 * Y + 1] = tile_last(a, Y / scale);
  }
  return GRL_OK;
}

}  // extern "C"
