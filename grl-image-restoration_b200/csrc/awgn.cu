// awgn.cu -- the denoising test command's noisy input (DnDataset.__getitem__, validation branch,
// data/datasets/restoration_dn.py:134-143) for a list of 8-bit images: k / 255 plus numpy's seeded legacy Gaussian noise,
// rounded to float32, bit for bit, from the closed forms of grl_awgn.h.
//
// One CTA per image runs that image's MT19937 stream from its seed to its last sample; a launch takes up to
// kAwgnPerLaunch images, whose records (pointers, size and key) travel by value in the kernel parameters
// (grl_param_list.cuh).  The number
// of twists an image needs depends on how many polar candidates are rejected, so only the CTA knows it: no host sync, no
// workspace.  Per twist of the 624-word state (shared memory, double-buffered so that no pass overwrites a word another
// thread of that pass still has to read):
//   three passes [0, 227), [227, 454), [454, 624) -- word i reads word i + 397 (mod 624), which the previous pass made --
//   each also tempering its words into tw;
//   156 threads test one candidate each (4 tempered words), a ballot / CTA scan gives the accepted ones their pair indices
//   k (running over the twists), and pair k writes samples 2k (f x2) and 2k + 1 (f x1, if inside the image).
// Sample i = (c H + y) W + x reads byte (y, x, c) of the HWC source and writes dst[i] of the CHW output, so consecutive
// pairs write consecutive addresses.
#include "grl_awgn.h"
#include "grl_common.cuh"
#include "grl_param_list.cuh"

namespace grl {

namespace {

constexpr int kAwgnPerLaunch = 64;
constexpr int kAwgnThreads = 256, kAwgnWarps = kAwgnThreads / 32;
constexpr int kPass = kMtN - kMtM;  // 227: the passes are [0, 227), [227, 454), [454, 624)
static_assert(kPass <= kAwgnThreads && kMtN - 2 * kPass <= kPass && kAwgnPairsPerTwist <= kAwgnThreads,
              "one word / candidate per thread");

struct AwgnRecord {  // 56 bytes
  const uint8_t* src;
  float* dst;
  int H, W;
  uint32_t key[8];
};
using AwgnRecords = ParamList<AwgnRecord, kAwgnPerLaunch, sizeof(int) + sizeof(double)>;

__global__ void __launch_bounds__(kAwgnThreads) awgn_kernel(const AwgnRecords L, int C, double scale) {
  __shared__ uint32_t mt[2][kMtN];  // the state, double-buffered over twists
  __shared__ uint32_t tw[kMtN];     // the current twist's tempered words
  __shared__ uint32_t key[8];
  __shared__ int accepted[kAwgnWarps];
  const AwgnRecord& im = L.at[blockIdx.x];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int plane = im.H * im.W, count = C * plane, npairs = (count + 1) >> 1;
  const uint8_t* src = im.src;
  float* dst = im.dst;
  if (tid < 8) key[tid] = im.key[tid];
  __syncthreads();
  if (tid == 0) awgn_mt_seed(mt[0], key);  // a dependent chain of ~1.9k steps
  __syncthreads();
  int cur = 0, k0 = 0;  // the buffer holding the state; the pairs accepted so far
  while (k0 < npairs) {
    const uint32_t* o = mt[cur];
    uint32_t* n = mt[cur ^ 1];
#pragma unroll
    for (int p = 0; p < 3; ++p) {
      const int i = p * kPass + tid;
      if (i < (p < 2 ? (p + 1) * kPass : kMtN)) {
        // the far word: old for pass 0, made by the previous pass otherwise; word 623's next word is the new word 0
        const uint32_t far = p == 0 ? o[i + kMtM] : n[i + kMtM - kMtN];
        const uint32_t v = awgn_twist_word(o[i], i + 1 < kMtN ? o[i + 1] : n[0], far);
        n[i] = v;
        tw[i] = awgn_temper(v);
      }
      __syncthreads();
    }
    cur ^= 1;
    double x1 = 0.0, x2 = 0.0, r2 = 0.0;
    bool acc = false;
    if (tid < kAwgnPairsPerTwist) {
      x1 = awgn_signed_unit(tw[4 * tid], tw[4 * tid + 1]);
      x2 = awgn_signed_unit(tw[4 * tid + 2], tw[4 * tid + 3]);
      r2 = awgn_r2(x1, x2);
      acc = awgn_accept(r2);
    }
    const unsigned ballot = __ballot_sync(0xffffffffu, acc);
    if (lane == 0) accepted[warp] = __popc(ballot);
    __syncthreads();
    int base = k0 + __popc(ballot & ((1u << lane) - 1u)), total = 0;
#pragma unroll
    for (int w = 0; w < kAwgnWarps; ++w) {
      const int a = accepted[w];
      base += w < warp ? a : 0;
      total += a;
    }
    k0 += total;
    if (acc && base < npairs) {
      const double f = awgn_polar_f(r2);
      const double g[2] = {dmul_rn(f, x2), dmul_rn(f, x1)};
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int i = 2 * base + h;
        if (i < count) {
          const int c = i / plane, px = i - c * plane;
          dst[i] = awgn_pixel(src[px * C + c], awgn_normal(scale, g[h]));
        }
      }
    }
    // tw was read before the barrier above; accepted is written again only after the next twist's three barriers
  }
}

int check_awgn(const GrlImageRef* src, const GrlImageRef* dst, const uint32_t* keys, int n, int C, double scale,
               const char* what) {
  GRL_REQUIRE(C == 1 || C == 3, "%s: C = %d, a denoising image is gray (C = 1) or RGB (C = 3)", what, C);
  GRL_REQUIRE(isfinite(scale) && scale >= 0.0, "%s: scale %g is not a finite value >= 0", what, scale);
  const int rc = check_list_args(n, keys != nullptr, "key", what);
  if (rc != GRL_OK) return rc;
  return check_u8_pairs(
      src, dst, n, GRL_IMAGE_F32, [](const GrlImageRef& s) { return make_int2(s.H, s.W); },
      [&](const GrlImageRef& s, int i) -> int {
        GRL_REQUIRE((long long)s.H * s.W * C <= 0x7fffffffLL, "%s: image %d: %d x %d x %d samples is too large", what, i,
                    s.H, s.W, C);
        return GRL_OK;
      },
      what);
}

}  // namespace

}  // namespace grl

using namespace grl;

extern "C" {

int grl_awgn_noise_host(const uint32_t* key, int64_t count, double scale, double* out) {
  GRL_REQUIRE(key && (out || count == 0) && count >= 0, "awgn_noise_host: bad arguments (count = %lld)",
              (long long)count);
  GRL_REQUIRE(isfinite(scale) && scale >= 0.0, "awgn_noise_host: scale %g is not a finite value >= 0", scale);
  uint32_t mt[kMtN], tw[kMtN];
  awgn_mt_seed(mt, key);
  for (int64_t i = 0; i < count;) {
    awgn_mt_twist(mt);
    for (int w = 0; w < kMtN; ++w) tw[w] = awgn_temper(mt[w]);
    for (int j = 0; j < kAwgnPairsPerTwist && i < count; ++j) {
      const double x1 = awgn_signed_unit(tw[4 * j], tw[4 * j + 1]), x2 = awgn_signed_unit(tw[4 * j + 2], tw[4 * j + 3]);
      const double r2 = awgn_r2(x1, x2);
      if (!awgn_accept(r2)) continue;
      const double f = awgn_polar_f(r2);
      out[i++] = awgn_normal(scale, dmul_rn(f, x2));
      if (i < count) out[i++] = awgn_normal(scale, dmul_rn(f, x1));
    }
  }
  return GRL_OK;
}

int grl_awgn_log_host(const double* x, int64_t n, double* out) {
  GRL_REQUIRE((x && out) || n == 0, "awgn_log_host: null argument");
  GRL_REQUIRE(n >= 0, "awgn_log_host: n = %lld", (long long)n);
  for (int64_t i = 0; i < n; ++i) {
    GRL_REQUIRE(isnormal(x[i]) && x[i] > 0.0, "awgn_log_host: x[%lld] = %g is not a positive normal number", (long long)i,
                x[i]);
    out[i] = awgn_log_cr(x[i]);
  }
  return GRL_OK;
}

int grl_awgn_u8(const GrlImageRef* src, const GrlImageRef* dst, const uint32_t* keys, int n, int C, double scale,
                void* stream) {
  const int rc = check_awgn(src, dst, keys, n, C, scale, "awgn_u8");
  if (rc != GRL_OK) return rc;
  const auto add = [&](AwgnRecord& r, int, int i) {
    r.src = static_cast<const uint8_t*>(src[i].data);
    r.dst = static_cast<float*>(dst[i].data);
    r.H = src[i].H;
    r.W = src[i].W;
    for (int w = 0; w < 8; ++w) r.key[w] = keys[8 * i + w];
    return 1LL;
  };
  return launch_list<AwgnRecords>(n, add, [&](const AwgnRecords& L, int, int m) -> int {
    awgn_kernel<<<m, kAwgnThreads, 0, (cudaStream_t)stream>>>(L, C, scale);
    GRL_LAUNCH_CHECK("awgn_kernel");
    return GRL_OK;
  });
}

}  // extern "C"
