// attn_tc.cuh -- constants and shared-memory layout common to the attention kernels (attn_tc.cu).
#pragma once
#include <stdint.h>

#include "tc_common.cuh"

namespace grl {
namespace tc {

constexpr int kQT = 128;
constexpr int kDP = 32;  // padded head dim (slot width)
constexpr float kMaskLog2 = -100.0f * 1.4426950408889634f;
// lazy-rescale threshold (log2 units): P = exp2(x - m_ref) <= 2^kTau, the running reference moves only past it
constexpr float kTau = 8.0f;

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// byte offset of 16-byte chunk c of row r in a 64-byte-row SWIZZLE_64B tile
__device__ __forceinline__ uint32_t sw64(int r, int c) { return (uint32_t)(r * 64 + ((c ^ ((r >> 1) & 3)) << 4)); }

// Q, then a ring of NS stages of K / V tiles and their key metadata (stage = tile % NS), the consumer threads' row
// records, then the ring's mbarriers.
template <int KT, int NS>
struct AttnSmem {
  static constexpr int Q_BYTES = kQT * 64;
  static constexpr int KV_BYTES = KT * 64;
  static constexpr int OFF_K = Q_BYTES;
  static constexpr int OFF_V = OFF_K + NS * KV_BYTES;
  static constexpr int OFF_META = OFF_V + NS * KV_BYTES;  // int koff[NS][KT], rid[NS][KT]
  static constexpr int OFF_ROWS = OFF_META + 2 * NS * KT * 4;  // int4 per consumer thread: bias bases, region ids
  static constexpr int OFF_DST = OFF_ROWS + 2 * kQT * 16;       // 2 x int64 per consumer thread: output offsets
  static constexpr int OFF_BAR = OFF_DST + 2 * kQT * 16;
  static constexpr int TOTAL = OFF_BAR + 2 * NS * 8 + 1024;
  static_assert(KV_BYTES % 512 == 0, "K / V tiles must stay aligned to the 64-byte swizzle repeat");
};

}  // namespace tc
}  // namespace grl
