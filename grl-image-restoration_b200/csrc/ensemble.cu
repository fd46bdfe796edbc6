// ensemble.cu -- the x8 self-ensemble's data movement: the 8 dihedral views of the input (augment_img_tensor4,
// utils/utils_bsr/utils_image.py:444-460) and the average of the 8 network outputs mapped back.
//
// Both kernels are HBM-bound copies over 32 x 32 pixel tiles of one (b, c) plane (grid.z = B * C planes).  Every global
// store walks a view row (or an output row) with threadIdx.x, so it is coalesced; a transposing view (group B) would make
// the matching global loads walk a column, so those go through a padded shared-memory tile that is loaded row-wise and
// read column-wise (stride 33 floats: no bank conflicts).  The flips only reverse the order inside a row.
#include "grl_common.cuh"

namespace grl {

namespace {

constexpr int kTile = 32, kRows = 8;  // 32 x 8 threads, 4 rows each

// One source tile of x, staged once and written to the 4 views of `group` (mode = 2 * i + group).
__global__ void __launch_bounds__(kTile * kRows) ens_gather_kernel(const float* __restrict__ x, int B, int C, int H, int W,
                                                                   int group, float* __restrict__ views) {
  __shared__ float tile[kTile][kTile + 1];
  const long long plane = blockIdx.z, hw = (long long)H * W, planes = (long long)B * C;
  const int y0 = blockIdx.y * kTile, x0 = blockIdx.x * kTile;
  const float* src = x + plane * hw;
  for (int r = threadIdx.y; r < kTile; r += kRows) {
    const int y = y0 + r, xx = x0 + threadIdx.x;
    if (y < H && xx < W) tile[r][threadIdx.x] = src[(long long)y * W + xx];
  }
  __syncthreads();
  const int Wv = group ? H : W;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int mode = 2 * i + group;
    float* dst = views + (i * planes + plane) * hw;
    for (int r = threadIdx.y; r < kTile; r += kRows) {
      // a transposing view's column index is the source row: let threadIdx.x walk the source rows there
      const int ly = group ? (int)threadIdx.x : r, lx = group ? r : (int)threadIdx.x;
      const int sy = y0 + ly, sx = x0 + lx;
      if (sy < H && sx < W) {
        const Pix p = d8_inv(mode, sy, sx, H, W);
        dst[(long long)p.y * Wv + p.x] = tile[ly][lx];
      }
    }
  }
}

// Smallest (row, column) of group-B view `mode` that an output tile [y0, y1] x [x0, x1] maps to.
__device__ __forceinline__ Pix box_origin(int mode, int y0, int y1, int x0, int x1, int Hs, int Ws) {
  return d8_inv(mode, (mode & 2) ? y1 : y0, (mode & 4) ? x1 : x0, Hs, Ws);
}

// One output tile: the 4 group-A views are read in place (row order, possibly reversed), the 4 group-B views are staged
// through shared memory; then V_0 + V_1 + ... + V_7 in mode order and the 1/8 scale.
__global__ void __launch_bounds__(kTile * kRows) ens_merge_kernel(const float* __restrict__ ya, const float* __restrict__ yb,
                                                                  int B, int C, int Hs, int Ws, float* __restrict__ y) {
  __shared__ float tb[4][kTile][kTile + 1];
  const long long plane = blockIdx.z, hw = (long long)Hs * Ws, planes = (long long)B * C;
  const int y0 = blockIdx.y * kTile, x0 = blockIdx.x * kTile;
  const int y1 = min(y0 + kTile, Hs) - 1, x1 = min(x0 + kTile, Ws) - 1;  // last row / column of the tile
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const Pix o = box_origin(2 * i + 1, y0, y1, x0, x1, Hs, Ws);
    const float* src = yb + (i * planes + plane) * hw;  // a (Ws, Hs) view: rows of Hs floats
    for (int r = threadIdx.y; r <= x1 - x0; r += kRows)
      if ((int)threadIdx.x <= y1 - y0) tb[i][r][threadIdx.x] = src[(long long)(o.y + r) * Hs + o.x + threadIdx.x];
  }
  __syncthreads();
  float* dst = y + plane * hw;
  for (int r = threadIdx.y; r < kTile; r += kRows) {
    const int yy = y0 + r, xx = x0 + threadIdx.x;
    if (yy > y1 || xx > x1) continue;
    float acc = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const Pix pa = d8_inv(2 * i, yy, xx, Hs, Ws);
      const float va = ya[(i * planes + plane) * hw + (long long)pa.y * Ws + pa.x];
      const Pix pb = d8_inv(2 * i + 1, yy, xx, Hs, Ws);
      const Pix o = box_origin(2 * i + 1, y0, y1, x0, x1, Hs, Ws);
      const float vb = tb[i][pb.y - o.y][pb.x - o.x];
      acc = (i == 0) ? va : acc + va;
      acc = acc + vb;
    }
    dst[(long long)yy * Ws + xx] = acc * 0.125f;
  }
}

int check_planes(int B, int C, int H, int W, const char* what) {
  GRL_REQUIRE(B > 0 && C > 0 && H > 0 && W > 0, "%s: bad shape B=%d C=%d H=%d W=%d", what, B, C, H, W);
  GRL_REQUIRE((long long)B * C <= 65535, "%s: B * C = %lld planes exceed the grid limit 65535", what, (long long)B * C);
  return GRL_OK;
}

}  // namespace

}  // namespace grl

using namespace grl;

extern "C" {

int grl_d8_index_host(int mode, int H, int W, int inverse, int32_t* out) {
  GRL_REQUIRE(mode >= 0 && mode < 8 && H > 0 && W > 0 && (long long)H * W <= 0x7fffffffLL && out,
              "d8_index: bad arguments mode=%d H=%d W=%d", mode, H, W);
  const int Hv = d8_transposes(mode) ? W : H, Wv = d8_transposes(mode) ? H : W;
  if (!inverse) {
    for (int y = 0; y < Hv; ++y)
      for (int x = 0; x < Wv; ++x) {
        const Pix p = d8_src(mode, y, x, H, W);
        out[(size_t)y * Wv + x] = p.y * W + p.x;
      }
  } else {
    for (int y = 0; y < H; ++y)
      for (int x = 0; x < W; ++x) {
        const Pix p = d8_inv(mode, y, x, H, W);
        out[(size_t)y * W + x] = p.y * Wv + p.x;
      }
  }
  return GRL_OK;
}

int grl_ens_gather_f32(const float* x, int B, int C, int H, int W, int group, float* views, void* stream) {
  GRL_REQUIRE(x && views, "ens_gather: null argument");
  GRL_REQUIRE(group == 0 || group == 1, "ens_gather: group must be 0 (modes 0,2,4,6) or 1 (modes 1,3,5,7), got %d", group);
  int rc = check_planes(B, C, H, W, "ens_gather");
  if (rc != GRL_OK) return rc;
  const dim3 grid(ceil_div(W, kTile), ceil_div(H, kTile), B * C);
  ens_gather_kernel<<<grid, dim3(kTile, kRows), 0, (cudaStream_t)stream>>>(x, B, C, H, W, group, views);
  GRL_LAUNCH_CHECK("ens_gather_kernel");
  return GRL_OK;
}

int grl_ens_merge_f32(const float* ya, const float* yb, int B, int C, int Hs, int Ws, float* y, void* stream) {
  GRL_REQUIRE(ya && yb && y, "ens_merge: null argument");
  int rc = check_planes(B, C, Hs, Ws, "ens_merge");
  if (rc != GRL_OK) return rc;
  const dim3 grid(ceil_div(Ws, kTile), ceil_div(Hs, kTile), B * C);
  ens_merge_kernel<<<grid, dim3(kTile, kRows), 0, (cudaStream_t)stream>>>(ya, yb, B, C, Hs, Ws, y);
  GRL_LAUNCH_CHECK("ens_merge_kernel");
  return GRL_OK;
}

}  // extern "C"
