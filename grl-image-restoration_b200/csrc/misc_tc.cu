// misc_tc.cu -- small memory-bound kernels around the tensor-core path: the network head (from RGB planes or from packed
// Bayer planes), fp32 -> padded bf16 packing, 16-bit average / max pooling (anchors), channel means of the CAB features, per-block
// preparation of the attention constants.
#include "grl_common.cuh"
#include "grl_demosaic.h"
#include "tc_common.cuh"

namespace grl {
namespace tc {

// fp32 (M, C) -> bf16 (M, Cpad), zero in [C, Cpad).  Each thread converts 8 channels (one 16-byte store).
__global__ void pack_bf16_kernel(const float* __restrict__ x, long long ldx, uint16_t* __restrict__ y, long long M,
                                 int C, int Cpad, int fmt) {
  const int per_row = Cpad / 8;
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * per_row) return;
  const long long m = i / per_row;
  const int c0 = (int)(i - m * per_row) * 8;
  float v[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) v[e] = (c0 + e < C) ? x[m * ldx + c0 + e] : 0.f;
  *reinterpret_cast<uint4*>(y + m * Cpad + c0) =
      make_uint4(pack16(v[0], v[1], fmt), pack16(v[2], v[3], fmt), pack16(v[4], v[5], fmt), pack16(v[6], v[7], fmt));
}

// bf16 (M, ld) -> fp32 (M, C)
__global__ void unpack_bf16_kernel(const uint16_t* __restrict__ x, long long ldx, int x_off, float* __restrict__ y,
                                   long long ldy, long long M, int C, int fmt) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * C) return;
  const long long m = i / C;
  const int c = (int)(i - m * C);
  y[m * ldy + c] = unpack16_one(x[m * ldx + x_off + c], fmt);
}

// AvgPool2d(df) / MaxPool2d(df) on 16-bit channels-last data, fp32 accumulation; 8 channels per thread.  Rounding to 16
// bits is monotone, so the max of the rounded inputs is the rounded fp32 max.
template <bool MAX>
__global__ void pool16_kernel(const uint16_t* __restrict__ x, uint16_t* __restrict__ y, int B, int H, int W, int Cpad,
                              int df, int fmt) {
  const int Ho = H / df, Wo = W / df, per = Cpad / 8;
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * Ho * Wo * per) return;
  const int c0 = (int)(i % per) * 8;
  long long t = i / per;
  const int xo = (int)(t % Wo);
  t /= Wo;
  const int yo = (int)(t % Ho);
  const int b = (int)(t / Ho);
  const float s0 = MAX ? -INFINITY : 0.f;
  float s[8] = {s0, s0, s0, s0, s0, s0, s0, s0};
  for (int dy = 0; dy < df; ++dy)
    for (int dx = 0; dx < df; ++dx) {
      const uint4 raw = *reinterpret_cast<const uint4*>(x + (((long long)b * H + yo * df + dy) * W + xo * df + dx) * Cpad + c0);
      const uint32_t* p = reinterpret_cast<const uint32_t*>(&raw);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = unpack16(p[e], fmt);
        if (MAX) {
          s[2 * e] = (f.x > s[2 * e] || f.x != f.x) ? f.x : s[2 * e];
          s[2 * e + 1] = (f.y > s[2 * e + 1] || f.y != f.y) ? f.y : s[2 * e + 1];
        } else {
          s[2 * e] += f.x;
          s[2 * e + 1] += f.y;
        }
      }
    }
  const float inv = MAX ? 1.f : 1.f / (float)(df * df);
  *reinterpret_cast<uint4*>(y + i * 8) =
      make_uint4(pack16(s[0] * inv, s[1] * inv, fmt), pack16(s[2] * inv, s[3] * inv, fmt),
                 pack16(s[4] * inv, s[5] * inv, fmt), pack16(s[6] * inv, s[7] * inv, fmt));
}

static int launch_pool16(const void* x, void* y, int B, int H, int W, int Cpad, int df, int fmt, bool max, cudaStream_t st) {
  if (check_fmt(fmt)) return GRL_ERR_INVALID;
  GRL_REQUIRE(df >= 1 && H % df == 0 && W % df == 0 && Cpad % 8 == 0, "pool16: bad shape");
  long long total = (long long)B * (H / df) * (W / df) * (Cpad / 8);
  if (total == 0) return GRL_OK;
  if (max)
    pool16_kernel<true><<<ceil_div(total, 256), 256, 0, st>>>((const uint16_t*)x, (uint16_t*)y, B, H, W, Cpad, df, fmt);
  else
    pool16_kernel<false><<<ceil_div(total, 256), 256, 0, st>>>((const uint16_t*)x, (uint16_t*)y, B, H, W, Cpad, df, fmt);
  GRL_LAUNCH_CHECK("pool16_kernel");
  return GRL_OK;
}

// Network input: check_image_size (reflect pad to a multiple of pad_size, grl.py:479-489) + (x - mean) * img_range
// (grl.py:510-511) + bchw -> channels-last + 16-bit operand pack, one pass.  One thread per padded pixel; Src reads raw
// channel c of image b at the source pixel (ys, xs) the padding maps the padded pixel to.
struct HeadMean {
  float m[8];  // Cin <= 8: the channels one 16-byte operand store holds
};
struct PlanarSrc {  // (B, Cin, H, W) planes
  const float* x;
  int Cin, H, W;
  __device__ __forceinline__ float operator()(int b, int c, int ys, int xs) const {
    return x[(((long long)b * Cin + c) * H + ys) * W + xs];
  }
};
struct RggbSrc {  // packed RGGB planes (B, 4, h, w), demosaiced on the fly (dm_matlab, grl_demosaic.h)
  const float* cfa4;
  int h, w;
  __device__ __forceinline__ float operator()(int b, int c, int ys, int xs) const {
    return dm_pixel(cfa4 + (long long)b * 4 * h * w, h, w, c, ys, xs);
  }
};
template <class Src>
__global__ void head_pack_kernel(Src src, int B, int Cin, int H, int W, int Hp, int Wp, HeadMean mean, float range,
                                 int reflect, uint16_t* __restrict__ y16, int Cpad, float* __restrict__ y32, int fmt) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * Hp * Wp) return;
  const int xp = (int)(i % Wp);
  const long long t = i / Wp;
  const int yp = (int)(t % Hp), b = (int)(t / Hp);
  int ys = yp, xs = xp;
  bool inside = true;
  if (reflect) {  // F.pad(..., "reflect") on the bottom / right: index 2 (n - 1) - p
    if (ys >= H) ys = 2 * (H - 1) - ys;
    if (xs >= W) xs = 2 * (W - 1) - xs;
  } else {
    inside = ys < H && xs < W;  // constant (zero) padding of the RAW image, normalised like every other pixel
  }
  float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int c = 0; c < 8; ++c) {  // unrolled: v and mean stay in registers / the parameter bank
    if (c >= Cin) break;
    const float raw = inside ? src(b, c, ys, xs) : 0.f;
    v[c] = (raw - mean.m[c]) * range;
    if (y32) y32[i * Cin + c] = v[c];
  }
  uint4* dst = reinterpret_cast<uint4*>(y16 + i * Cpad);
  dst[0] = make_uint4(pack16(v[0], v[1], fmt), pack16(v[2], v[3], fmt), pack16(v[4], v[5], fmt), pack16(v[6], v[7], fmt));
  for (int c8 = 1; c8 < Cpad / 8; ++c8) dst[c8] = make_uint4(0u, 0u, 0u, 0u);
}

// Deterministic partial channel sums of bf16 features y (B, L, ld): partial (B, chunks, C) fp32.
constexpr int kPoolRowsTc = 512;
__global__ void channel_partial_bf16_kernel(const uint16_t* __restrict__ y, long long L, long long ld, int C, int fmt,
                                            float* __restrict__ partial, int chunks) {
  const int b = blockIdx.y, ch = blockIdx.x;
  const long long r0 = (long long)ch * kPoolRowsTc, r1 = min(L, r0 + kPoolRowsTc);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float s = 0.f;
    for (long long r = r0; r < r1; ++r) s += unpack16_one(y[((long long)b * L + r) * ld + c], fmt);
    partial[((long long)b * chunks + ch) * C + c] = s;
  }
}

// Per-block attention constants.  slot_scale[slot] for the packed qkv layout
//   slots: [win q h..][win k h..][win v h..][str q h..][str k h..][str v h..]
// q^ of the window half carries exp(min(ls_w, ln100)) * log2(e); stripe k^ carries scale1 (anchors are the queries of
// pass 1), stripe q^ carries scale2; keys / anchors that are not scaled get 1; value slots get 0 (= leave untouched).
__global__ void slot_scale_kernel(const float* __restrict__ ls_w, const float* __restrict__ ls_s1,
                                  const float* __restrict__ ls_s2, int hw, int hs, float* __restrict__ out) {
  const float LOG2E = 1.4426950408889634f, LN100 = 4.605170185988092f;
  const int n = 3 * hw + 3 * hs;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    float v;
    if (i < hw) v = expf(fminf(ls_w[i], LN100)) * LOG2E;
    else if (i < 2 * hw) v = 1.f;
    else if (i < 3 * hw) v = 0.f;
    else if (i < 3 * hw + hs) v = expf(fminf(ls_s2[i - 3 * hw], LN100)) * LOG2E;
    else if (i < 3 * hw + 2 * hs) v = expf(fminf(ls_s1[i - 3 * hw - hs], LN100)) * LOG2E;
    else v = 0.f;
    out[i] = v;
  }
}

template <class Src>
static int launch_head(Src src, int B, int Cin, int H, int W, int Hp, int Wp, const float* mean4, float range, void* y16,
                       int Cpad, float* y32, int fmt, cudaStream_t st) {
  GRL_REQUIRE(Cin >= 1 && Cin <= 8 && Cpad % 8 == 0 && Cpad >= 8 && Hp >= H && Wp >= W && H > 0 && W > 0,
              "head_pack: bad shape (Cin %d, %dx%d -> %dx%d, Cpad %d)", Cin, H, W, Hp, Wp, Cpad);
  const long long total = (long long)B * Hp * Wp;
  if (total == 0) return GRL_OK;
  HeadMean m;
  const int n_mean = Cin > 4 ? Cin : 4;  // max(4, Cin) host floats: callers of the Cin <= 4 head pass exactly 4
  for (int c = 0; c < 8; ++c) m.m[c] = (mean4 && c < n_mean) ? mean4[c] : 0.f;
  const int reflect = (Hp - H < H && Wp - W < W) ? 1 : 0;  // torch raises otherwise and the reference pads with zeros
  head_pack_kernel<<<ceil_div(total, 256), 256, 0, st>>>(src, B, Cin, H, W, Hp, Wp, m, range, reflect, (uint16_t*)y16, Cpad, y32, fmt);
  GRL_LAUNCH_CHECK("head_pack_kernel");
  return GRL_OK;
}

}  // namespace tc
}  // namespace grl

using namespace grl;
using namespace grl::tc;

extern "C" {

int grl_tc_pack16(const float* x, int64_t ldx, void* y, int64_t M, int C, int Cpad, int fmt, void* stream) {
  if (check_fmt(fmt)) return GRL_ERR_INVALID;
  GRL_REQUIRE(Cpad % 8 == 0 && Cpad >= C, "pack_bf16: bad padding %d for %d channels", Cpad, C);
  if (M == 0) return GRL_OK;
  pack_bf16_kernel<<<ceil_div(M * (Cpad / 8), 256), 256, 0, (cudaStream_t)stream>>>(x, ldx, (uint16_t*)y, M, C, Cpad, fmt);
  GRL_LAUNCH_CHECK("pack_bf16_kernel");
  return GRL_OK;
}

int grl_tc_unpack16(const void* x, int64_t ldx, int x_off, float* y, int64_t ldy, int64_t M, int C, int fmt,
                    void* stream) {
  if (check_fmt(fmt)) return GRL_ERR_INVALID;
  if (M == 0) return GRL_OK;
  unpack_bf16_kernel<<<ceil_div(M * C, 256), 256, 0, (cudaStream_t)stream>>>((const uint16_t*)x, ldx, x_off, y, ldy, M, C, fmt);
  GRL_LAUNCH_CHECK("unpack_bf16_kernel");
  return GRL_OK;
}

int grl_tc_head_pack(const float* x, int B, int Cin, int H, int W, int Hp, int Wp, const float* mean4, float range, void* y16,
                     int Cpad, float* y32, int fmt, void* stream) {
  if (check_fmt(fmt)) return GRL_ERR_INVALID;
  GRL_REQUIRE(x && y16, "head_pack: null argument");
  return launch_head(PlanarSrc{x, Cin, H, W}, B, Cin, H, W, Hp, Wp, mean4, range, y16, Cpad, y32, fmt, (cudaStream_t)stream);
}

int grl_tc_head_pack_rggb(const float* cfa4, int B, int h, int w, int Hp, int Wp, const float* mean4, float range, void* y16,
                          int Cpad, float* y32, int fmt, void* stream) {
  if (check_fmt(fmt)) return GRL_ERR_INVALID;
  GRL_REQUIRE(cfa4 && y16, "head_pack_rggb: null argument");
  GRL_REQUIRE(h >= 2 && w >= 2, "head_pack_rggb: packed RGGB planes need h, w >= 2, got %dx%d", h, w);
  return launch_head(RggbSrc{cfa4, h, w}, B, 3, 2 * h, 2 * w, Hp, Wp, mean4, range, y16, Cpad, y32, fmt, (cudaStream_t)stream);
}

int grl_tc_avgpool16(const void* x, void* y, int B, int H, int W, int Cpad, int df, int fmt, void* stream) {
  return launch_pool16(x, y, B, H, W, Cpad, df, fmt, false, (cudaStream_t)stream);
}

int grl_tc_maxpool16(const void* x, void* y, int B, int H, int W, int Cpad, int df, int fmt, void* stream) {
  return launch_pool16(x, y, B, H, W, Cpad, df, fmt, true, (cudaStream_t)stream);
}

int grl_tc_slot_scale(const float* ls_w, const float* ls_s1, const float* ls_s2, int hw, int hs, float* out,
                      void* stream) {
  GRL_REQUIRE(hw >= 1 && hs >= 1 && hw <= 8 && hs <= 8, "slot_scale: bad head counts");
  slot_scale_kernel<<<1, 64, 0, (cudaStream_t)stream>>>(ls_w, ls_s1, ls_s2, hw, hs, out);
  GRL_LAUNCH_CHECK("slot_scale_kernel");
  return GRL_OK;
}

size_t grl_tc_channel_gate_workspace(int B, int64_t L, int C) {
  return sizeof(float) * (size_t)B * ceil_div(L, kPoolRowsTc) * C;
}

int grl_tc_channel_gate(const void* y, int64_t ld, int fmt, int B, int64_t L, int C, const float* w1, const float* b1,
                        const float* w2, const float* b2, int R, float* gate, void* ws, size_t ws_bytes, void* stream) {
  if (check_fmt(fmt)) return GRL_ERR_INVALID;
  if (ws_bytes < grl_tc_channel_gate_workspace(B, L, C)) return fail(GRL_ERR_WORKSPACE, "tc_channel_gate: workspace too small");
  if (B == 0) return GRL_OK;
  const cudaStream_t st = (cudaStream_t)stream;
  const int chunks = ceil_div(L, kPoolRowsTc);
  channel_partial_bf16_kernel<<<dim3(chunks, B), 256, 0, st>>>((const uint16_t*)y, L, ld, C, fmt, (float*)ws, chunks);
  GRL_LAUNCH_CHECK("channel_partial_bf16_kernel");
  return channel_gate_from_partial((const float*)ws, chunks, B, L, C, w1, b1, w2, b2, R, gate, st);
}

}  // extern "C"
