// gemm_tc.cu -- 16-bit wgmma GEMM / implicit-GEMM 3x3 convolution with fused epilogues (the non-attention half
// of a GRL block on the throughput path).
//
//   D[128 x BN] (fp32) = A[128 x K] (fp16|bf16, TMA -> smem, SWIZZLE_128B) * W[BN x K]^T (fp16|bf16, TMA -> smem)
//
// A is either a row-major (tokens x Kpad) activation matrix (nn.Linear: QKVProjection, AnchorLinear, proj, Mlp) or
// the channels-last image itself read through a 4-D tensor map: one CTA owns an 8x16 pixel patch and each of the
// 9 taps is the same TMA box shifted by (dy, dx) -- the zero padding of the convolution is TMA's out-of-bounds
// fill, no im2col buffer exists (CAB convs mixed_attn_block.py:973-977, TransformerStage.conv grl.py:164-170).
//
// Warp roles (288 threads): warps 0-7 = two consumer warpgroups (rows 0-63 / 64-127 of the tile, wgmma m64n64k16 per
// 64 output columns, accumulators in registers), warp 8 = TMA producer feeding a 4-stage ring.  After the main loop the
// accumulators go to an fp32 tile in shared memory, and the same 256 threads run the epilogue with two threads per
// accumulator row (the row's 32-column chunks split between them, LayerNorm moments merged through shared memory).
// These GEMMs are short-K and HBM / epilogue bound, not tensor bound (DESIGN.md).
//
// Epilogues:
//   EPI_BIAS_ACT : y = act(acc + b) (+ res)                       -> bf16 and/or fp32     (fc1, CAB, convs, heads)
//   EPI_QKV      : per 32-wide head slot  y = (acc + b) * scale / max(||.||, 1e-12)  -> bf16 (q^, k^, a^; v untouched)
//                  (F.normalize + logit scale of Attention.attn / AffineTransform, efficient.py:39,:85)
//   EPI_LN       : x' = x + rs * LayerNorm(acc + b) (+ cab_y * gate) -> fp32 residual stream + bf16 operand copy
//                  (efficient.py:543-554)
#include <algorithm>

#include "grl_common.cuh"
#include "tc_common.cuh"

namespace grl {
namespace tc {

EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

// erf-form GELU for the tensor-core epilogues: Abramowitz-Stegun 7.1.26, 2 MUFU + 11 FMA-class instructions instead
// of erff's ~30.  The fp32 parity path keeps erff.  |gelu_as - GELU| <= 3.8e-7 absolute over [-12, 12] with a correctly
// rounded rcp / exp2 (tests/test_gpu_tc_gemm.py::test_gelu_as_bound pins 5e-7; the .approx errors are not modelled).
// That is NOT below the 16-bit rounding that follows: up to 1.2 fp16 ulp on [-4, -1] and 2 subnormal ulp below -4, so
// an fp16 store of the result is not always the correctly rounded GELU.  The values only feed fc2 / the second CAB conv.
__device__ __forceinline__ float gelu_as(float x) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  float t, e;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-z * z * 1.4426950408889634f));
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  const float erf_abs = fmaf(-p * t, e, 1.0f);  // erf(|x| / sqrt 2)
  const float half_x = 0.5f * x;
  return fmaf(half_x, copysignf(erf_abs, x), half_x);  // 0.5 x (1 + erf(x / sqrt 2))
}
__device__ __forceinline__ float tc_act(float v, int act, float slope) {
  if (act == GRL_ACT_GELU) return gelu_as(v);
  if (act == GRL_ACT_LEAKY) return v > 0.f ? v : v * slope;
  return v;
}

constexpr int kStages = 4;
constexpr int kBM = 128, kBK = 64;
constexpr int kTH = 8, kTW = 16;  // conv patch (kTH * kTW == kBM)
constexpr int kEpiWarps = 8, kEpiThreads = kEpiWarps * 32, kThreads = kEpiThreads + 32;

// Epilogue staging: the accumulator tile is first written to shared memory by its row owners (phase A, thread = row),
// then streamed to global memory row-major by all epilogue threads with 16-byte accesses (phase B) -- fully coalesced
// residual reads and stores with many independent requests in flight.
//   fp32 staging (LayerNorm / fp32 outputs): [128][pitch32] floats, pitch32 % 8 == 4  -> conflict-free 16 B rows
//   16-bit staging (fp16/bf16-only outputs): [128][BN + 8] halves
__host__ __device__ constexpr int stage_pitch32(int c) { return (c % 8 == 4) ? c : ((c + 3) / 4 * 4 % 8 == 4 ? (c + 3) / 4 * 4 : (c + 3) / 4 * 4 + 4); }

// Shared memory: the operand ring and, once the main loop is over, the fp32 accumulator tile [128][BN + 4] followed by
// the staging tile (both alias the ring).
template <int BN>
struct GemmSmem {
  static constexpr int A_BYTES = kBM * kBK * 2;
  static constexpr int B_BYTES = BN * kBK * 2;
  static constexpr int STAGE = A_BYTES + B_BYTES;
  static constexpr int PIPE = kStages * STAGE;
  static constexpr int AP = BN + 4;  // accumulator pitch (floats): AP % 8 == 4, conflict-free 16-byte row reads
  static constexpr int ACC = kBM * AP * 4;
  static constexpr int STG32 = kBM * stage_pitch32(BN <= 192 ? (BN == 192 ? 188 : BN) : 4) * 4;  // C <= 188 at BN = 192
  static constexpr int STG16 = kBM * (BN + 8) * 2;
  static constexpr int STG = (STG32 > STG16 ? STG32 : STG16);
  static constexpr int OFF_STG = ACC;
  static constexpr int OFF_TOK = ((PIPE > ACC + STG ? PIPE : ACC + STG) + 15) / 16 * 16;  // long long tok[128]
  static constexpr int OFF_PAR = OFF_TOK + 128 * 8 + 128 * 4;  // (+ int img[128]) float bias[BN], gamma[BN], beta[BN]
  static constexpr int OFF_MOM = OFF_PAR + 3 * BN * 4;         // float mom[2][128][3]
  static constexpr int OFF_BAR = OFF_MOM + 2 * 128 * 3 * 4;
  static constexpr int TOTAL = OFF_BAR + 128 + 1024 /*align slack*/;
  static_assert(AP % 8 == 4, "accumulator pitch");
  static_assert(TOTAL <= 232448, "shared memory budget");
};

__device__ __forceinline__ void epi_barrier() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// 32 consecutive fp32 accumulator values of one row
__device__ __forceinline__ void acc_row32(const float* p, uint32_t (&v)[32]) {
#pragma unroll
  for (int j = 0; j < 32; j += 4) {
    const uint4 x = *reinterpret_cast<const uint4*>(p + j);
    v[j] = x.x, v[j + 1] = x.y, v[j + 2] = x.z, v[j + 3] = x.w;
  }
}

// Main loop of consumer warpgroup `half`: rows [64 half, 64 half + 64) of the tile, BN / 64 accumulators of m64n64.
// FMT is a template argument so that no branch separates the wgmma instructions of one k step.
template <int BN, int FMT>
__device__ __forceinline__ void mma_loop(float (&acc)[BN / 64][32], uint8_t* smem, uint64_t* full, uint64_t* empty,
                                         int nk_total, int half, int et) {
  using S = GemmSmem<BN>;
  for (int kc = 0; kc < nk_total; ++kc) {
    const int s = kc % kStages;
    mbar_wait(&full[s], (kc / kStages) & 1);
    const uint32_t sa = smem_u32(smem + s * S::STAGE) + half * (64 * 128);
    const uint32_t sb = smem_u32(smem + s * S::STAGE + S::A_BYTES);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kBK / 16; ++k) {
      const uint64_t ad = gmma_desc(sa + k * 32, 16, 1024, SWZ_128B);
#pragma unroll
      for (int j = 0; j < BN / 64; ++j) {
        const uint64_t bd = gmma_desc(sb + j * (64 * 128) + k * 32, 16, 1024, SWZ_128B);
        if (FMT == FMT_BF16) wgmma_n64_bf16(acc[j], ad, bd, true);
        else wgmma_n64_f16(acc[j], ad, bd, true);
      }
    }
    wgmma_commit();
    // this k step's MMAs stay in flight; the previous step's are complete, so its stage goes back to the producer
    wgmma_wait<1>();
    if (kc > 0 && (et & 127) == 0) mbar_arrive(&empty[(kc - 1) % kStages]);
  }
  wgmma_wait<0>();
}

// What the host derives from a GrlTcGemm for its launch (plan_gemm_tc); the kernel takes both.
struct GemmTcPlan {
  long long M;   // rows: GrlTcGemm::M, or B * H * W for a conv
  int nk;        // 64-wide k chunks per tap
  int n_tiles, total_tiles;
  int tiles_x, tiles_y;  // conv: 8 x 16 pixel patches per image
  int epi_mode;  // 0 = 16-bit staging, 1 = fp32 staging, 2 = direct
  int nchw_r;    // GrlTcGemm::nchw_r, at least 1
};

template <int BN, int EPI, bool CONV>
__global__ void __launch_bounds__(kThreads, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GrlTcGemm a,
              const GemmTcPlan pl) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  using S = GemmSmem<BN>;
  constexpr int AP = S::AP;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + S::OFF_BAR);
  uint64_t* empty = full + kStages;
  long long* s_tok = reinterpret_cast<long long*>(smem + S::OFF_TOK);
  int* s_img = reinterpret_cast<int*>(smem + S::OFF_TOK + 128 * 8);  // image (batch) index of every row (CAB gate)
  float* s_bias = reinterpret_cast<float*>(smem + S::OFF_PAR);      // this tile's columns [n0, n0 + BN)
  float* s_gamma = s_bias + BN;
  float* s_beta = s_gamma + BN;
  float* s_mom = reinterpret_cast<float*>(smem + S::OFF_MOM);  // [2][128][3]: (mean, M2, n) of each column half of a row
  float* accs = reinterpret_cast<float*>(smem);                // [128][AP] after the main loop

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // 1-D grid, N tile fastest: the CTAs that share an A tile (same rows, different output columns) are scheduled
  // together, so the tile is read from DRAM once and from L2 afterwards (QKV: 3 column tiles, fc1: 2).
  const int n_tiles = pl.n_tiles;
  const int m_idx = blockIdx.x / n_tiles;
  const int n0 = (blockIdx.x - m_idx * n_tiles) * BN;
  const int nk_total = a.taps * pl.nk;
  int m0 = 0, tb = 0, ty0 = 0, tx0 = 0;
  if (CONV) {
    int t = m_idx;
    const int tx = t % pl.tiles_x;
    t /= pl.tiles_x;
    const int ty = t % pl.tiles_y;
    tb = t / pl.tiles_y;
    ty0 = ty * kTH;
    tx0 = tx * kTW;
  } else {
    m0 = m_idx * kBM;
  }

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 2);  // one arrival per consumer warpgroup
    }
    mbar_init_fence();
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
  }
  __syncthreads();

  if (warp == kEpiWarps) {
    // ================================================================== TMA producer
    if (lane == 0) {
      for (int kc = 0; kc < nk_total; ++kc) {
        const int s = kc % kStages;
        mbar_wait(&empty[s], ((kc / kStages) & 1) ^ 1);
        uint8_t* sa = smem + s * S::STAGE;
        uint8_t* sb = sa + S::A_BYTES;
        mbar_expect_tx(&full[s], S::STAGE);
        if (CONV) {
          const int tap = kc / pl.nk, c0 = (kc - tap * pl.nk) * kBK;
          tma_load_4d(sa, &tmA, &full[s], c0, tx0 + (tap % 3) - 1, ty0 + (tap / 3) - 1, tb);
        } else {
          tma_load_2d(sa, &tmA, &full[s], kc * kBK, m0);
        }
        tma_load_2d(sb, &tmB, &full[s], kc * kBK, n0);
      }
    }
    return;
  }

  // ================================================================== consumers: MMA, then the epilogue (256 threads)
  const int et = threadIdx.x;      // 0..255
  const int q = warp & 3;          // row quarter of this warp in phase A
  const int row = q * 32 + lane;   // accumulator row owned in phase A
  const int half = et >> 7;        // which chunks of the row: c0 = 32 * half, + 64, ...  (also: the MMA warpgroup)
  const int fmt = a.fmt;
  uint16_t* out16 = reinterpret_cast<uint16_t*>(a.out_bf16);
  // per-tile tables: token (global row) of every accumulator row (-1 = outside the problem), its image, and the
  // per-column constants of this N tile (every row-owner thread needs all of them: smem broadcast)
  {
    long long tok;
    if (CONV) {
      const int y = ty0 + row / kTW, x = tx0 + row % kTW;
      tok = (y < a.H && x < a.W) ? ((long long)tb * a.H + y) * a.W + x : -1;
    } else {
      tok = (long long)m0 + row;
      if (tok >= pl.M) tok = -1;
    }
    if (half == 0) {
      s_tok[row] = tok;
      s_img[row] = (EPI == EPI_LN && tok >= 0) ? (int)(tok / a.L) : 0;  // one 64-bit division per row, not per access
    }
    for (int c = et; c < BN; c += kEpiThreads) {
      const int n = n0 + c;
      s_bias[c] = (n < a.n_store) ? a.bias[n] : 0.f;
      if (EPI == EPI_LN) {
        s_gamma[c] = (c < a.C) ? a.gamma[c] : 0.f;
        s_beta[c] = (c < a.C) ? a.beta[c] : 0.f;
      }
    }
  }
  {
    // warpgroup `half` computes rows [64 half, 64 half + 64): BN / 64 accumulators of m64n64
    float acc[BN / 64][32];
#pragma unroll
    for (int j = 0; j < BN / 64; ++j)
#pragma unroll
      for (int e = 0; e < 32; ++e) acc[j][e] = 0.f;
    if (fmt == FMT_BF16) mma_loop<BN, FMT_BF16>(acc, smem, full, empty, nk_total, half, et);
    else mma_loop<BN, FMT_F16>(acc, smem, full, empty, nk_total, half, et);
    epi_barrier();  // both warpgroups are done reading the ring: it becomes the accumulator / staging tile
    const int w = (et >> 5) & 3, r0 = half * 64 + 16 * w + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < BN / 64; ++j)
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int c = j * 64 + 8 * i + cq;
        *reinterpret_cast<float2*>(accs + r0 * AP + c) = make_float2(acc[j][4 * i], acc[j][4 * i + 1]);
        *reinterpret_cast<float2*>(accs + (r0 + 8) * AP + c) = make_float2(acc[j][4 * i + 2], acc[j][4 * i + 3]);
      }
  }
  epi_barrier();
  uint32_t v[32];

    // epi_mode (chosen on the host): 1 = fp32 staging (LayerNorm / fp32 result / residual, whole row in this tile),
    // 0 = 16-bit staging, 2 = direct per-row stores (odd widths such as the 3-channel image head)
    if (EPI == EPI_BIAS_ACT && pl.epi_mode == 2) {
      const long long tok = s_tok[row];
      for (int c0 = 32 * half; c0 < BN; c0 += 64) {
        if (n0 + c0 >= a.n_store) break;
        acc_row32(accs + row * AP + c0, v);
        if (tok < 0) continue;
        float o[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const int n = n0 + c0 + j;
          float val = tc_act(__uint_as_float(v[j]) + s_bias[c0 + j], a.act, a.slope);
          if (a.res_f32 && n < a.n_real) val += __ldg(a.res_f32 + tok * a.ldr + n);
          o[j] = (n < a.n_store) ? val : 0.f;
          if (a.out_f32 && n < a.n_real) a.out_f32[tok * a.ldo_f32 + n] = o[j];
          if (CONV && a.out_nchw && n < a.n_real) {
            // tail fusion: x / img_range + mean (grl.py:549), the crop (:551), channels-last -> bchw and, for the one-step
            // head, PixelShuffle (upsample.py:33-50; torch order n = c r^2 + dy r + dx) folded into the store
            const int r = pl.nchw_r, rr = r * r;
            const int c = n / rr, q = n - c * rr;
            const int yy = (ty0 + row / kTW) * r + q / r, xx = (tx0 + row % kTW) * r + q % r;
            if (yy < a.Hc && xx < a.Wc)
              a.out_nchw[(((long long)tb * (a.n_real / rr) + c) * a.Hc + yy) * a.Wc + xx] = fmaf(o[j], a.post_scale, a.post_shift[c & 3]);
          }
        }
        if (out16) {
#pragma unroll
          for (int j = 0; j < 32; j += 8)
            if (n0 + c0 + j < a.ldo_bf16)
              *reinterpret_cast<uint4*>(out16 + tok * a.ldo_bf16 + n0 + c0 + j) =
                  make_uint4(pack16(o[j], o[j + 1], fmt), pack16(o[j + 2], o[j + 3], fmt), pack16(o[j + 4], o[j + 5], fmt),
                             pack16(o[j + 6], o[j + 7], fmt));
        }
      }
    } else if (pl.epi_mode == 1) {
      const int Cw = (EPI == EPI_LN) ? a.C : a.n_real;  // real fp32 columns of this tile row (n0 == 0 when wide)
      const int pitch = stage_pitch32(Cw);
      float* stg = reinterpret_cast<float*>(smem + S::OFF_STG);
      // ---------------- residual tile -> staging, asynchronously (cp.async, 16 B per request, the whole 128 x C
      // tile in flight at once); it lands while the row moments are computed from the accumulator tile.  Phase A then adds its
      // result in place, so phase B has no fp32 loads left.
      const bool res_in_stage = a.res_f32 != nullptr;
      if (res_in_stage) {
        const int C4r = Cw >> 2, ewr = et >> 5;
        for (int r = ewr; r < kBM; r += kEpiWarps) {
          const long long rtok = s_tok[r];
          for (int c4 = lane; c4 < C4r; c4 += 32)
            cp_async_16(stg + r * pitch + c4 * 4, a.res_f32 + (rtok >= 0 ? rtok : 0) * a.ldr + c4 * 4, rtok >= 0);
        }
        cp_async_commit();
      }
      // ---------------- phase A
      if (EPI == EPI_LN) {
        // One pass over the accumulator row for the moments of THIS THREAD'S HALF of the row (its 32-column chunks), shifted by the half's
        // first element (no catastrophic cancellation): mean_h = x0 + S1/n, M2_h = S2 - S1^2/n with S1 = sum(x - x0),
        // S2 = sum((x - x0)^2).  The two halves are merged with the pairwise update (Chan et al.):
        //   mean = mean_0 + d n_1 / n,  M2 = M2_0 + M2_1 + d^2 n_0 n_1 / n,  d = mean_1 - mean_0.
        float s1 = 0.f, s2 = 0.f, x0 = 0.f;
        int nh = 0;
        for (int c0 = 32 * half; c0 < Cw; c0 += 64) {
          acc_row32(accs + row * AP + c0, v);
          if (c0 == 32 * half) x0 = __uint_as_float(v[0]) + s_bias[c0];
#pragma unroll
          for (int j = 0; j < 32; ++j)
            if (c0 + j < Cw) {
              const float d = __uint_as_float(v[j]) + s_bias[c0 + j] - x0;
              s1 += d;
              s2 = fmaf(d, d, s2);
              ++nh;
            }
        }
        {
          const float fn = (float)nh;
          const float m1 = nh > 0 ? s1 / fn : 0.f;
          s_mom[(half * kBM + row) * 3 + 0] = x0 + m1;
          s_mom[(half * kBM + row) * 3 + 1] = nh > 0 ? fmaxf(s2 - s1 * m1, 0.f) : 0.f;
          s_mom[(half * kBM + row) * 3 + 2] = fn;
        }
        if (res_in_stage) cp_async_wait<0>();  // this thread's share of the residual tile has landed ...
        epi_barrier();                         // ... and is visible to the row owners; so are both halves' moments
        float mean, rstd;
        {
          const float m0 = s_mom[row * 3 + 0], q0 = s_mom[row * 3 + 1], c0n = s_mom[row * 3 + 2];
          const float m1 = s_mom[(kBM + row) * 3 + 0], q1 = s_mom[(kBM + row) * 3 + 1], c1n = s_mom[(kBM + row) * 3 + 2];
          const float n = c0n + c1n, d = (c1n > 0.f) ? m1 - m0 : 0.f;
          mean = m0 + d * (c1n / n);
          const float M2 = q0 + q1 + d * d * (c0n * c1n / n);
          rstd = rsqrtf(M2 / n + a.eps);
        }
        for (int c0 = 32 * half; c0 < Cw; c0 += 64) {
          acc_row32(accs + row * AP + c0, v);
#pragma unroll
          for (int j = 0; j < 32; j += 4) {
            if (c0 + j < Cw) {  // Cw % 4 == 0
              float4* sp = reinterpret_cast<float4*>(stg + row * pitch + c0 + j);
              float4 acc4 = res_in_stage ? *sp : make_float4(0.f, 0.f, 0.f, 0.f);
              float o4[4] = {acc4.x, acc4.y, acc4.z, acc4.w};
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const int c = c0 + j + e;
                o4[e] += ((__uint_as_float(v[j + e]) + s_bias[c] - mean) * rstd * s_gamma[c] + s_beta[c]) * a.res_scale;
              }
              *sp = make_float4(o4[0], o4[1], o4[2], o4[3]);
            }
          }
        }
      } else {
        if (res_in_stage) {
          cp_async_wait<0>();
          epi_barrier();
        }
        for (int c0 = 32 * half; c0 < Cw; c0 += 64) {
          acc_row32(accs + row * AP + c0, v);
#pragma unroll
          for (int j = 0; j < 32; j += 4) {
            if (c0 + j < Cw) {
              float4* sp = reinterpret_cast<float4*>(stg + row * pitch + c0 + j);
              float4 acc4 = res_in_stage ? *sp : make_float4(0.f, 0.f, 0.f, 0.f);
              float o4[4] = {acc4.x, acc4.y, acc4.z, acc4.w};
#pragma unroll
              for (int e = 0; e < 4; ++e) o4[e] += tc_act(__uint_as_float(v[j + e]) + s_bias[c0 + j + e], a.act, a.slope);
              *sp = make_float4(o4[0], o4[1], o4[2], o4[3]);
            }
          }
        }
      }
      epi_barrier();
      // ---------------- phase B: row-major streaming, 4 columns per thread, warp = row group.
      // All global loads of a batch of RB rows are issued before any store (the compiler cannot prove the output
      // and residual pointers distinct, so interleaving would serialise every row on a DRAM round trip).
      const int C4 = Cw >> 2;                              // float4 items with real data
      const int P4 = out16 ? (int)(a.ldo_bf16 >> 2) : C4;  // the 16-bit copy is written up to its (zero) pad
      const int ew = et >> 5;
      const bool has_cab = (EPI == EPI_LN) && a.cab_y != nullptr;
      const uint16_t* caby = reinterpret_cast<const uint16_t*>(a.cab_y);
      constexpr int RB = 8;
      for (int cbase = 0; cbase < P4; cbase += 32) {
        const int c4 = cbase + lane;
        const bool col_real = c4 < C4, col_any = c4 < P4;
        for (int rb = 0; rb < kBM / kEpiWarps; rb += RB) {  // this warp's rows: ew, ew + 8, ...
          long long tok[RB];
          float4 gg[RB];
          uint2 cy[RB];
#pragma unroll
          for (int i = 0; i < RB; ++i) {
            tok[i] = s_tok[ew + kEpiWarps * (rb + i)];
            gg[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            cy[i] = make_uint2(0u, 0u);
            if (tok[i] >= 0 && col_real) {
              if (has_cab) {
                cy[i] = __ldg(reinterpret_cast<const uint2*>(caby + tok[i] * a.ld_caby + c4 * 4));
                gg[i] = __ldg(reinterpret_cast<const float4*>(a.cab_gate + (long long)s_img[ew + kEpiWarps * (rb + i)] * Cw + c4 * 4));
              }
            }
          }
#pragma unroll
          for (int i = 0; i < RB; ++i) {
            if (tok[i] < 0 || !col_any) continue;
            float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
            if (col_real) {
              val = *reinterpret_cast<const float4*>(stg + (ew + kEpiWarps * (rb + i)) * pitch + c4 * 4);
              if (has_cab) {
                const float2 c01 = unpack16(cy[i].x, fmt), c23 = unpack16(cy[i].y, fmt);
                val.x = fmaf(c01.x, gg[i].x, val.x), val.y = fmaf(c01.y, gg[i].y, val.y);
                val.z = fmaf(c23.x, gg[i].z, val.z), val.w = fmaf(c23.y, gg[i].w, val.w);
              }
              if (a.out_f32) *reinterpret_cast<float4*>(a.out_f32 + tok[i] * a.ldo_f32 + c4 * 4) = val;
            }
            if (out16)
              *reinterpret_cast<uint2*>(out16 + tok[i] * a.ldo_bf16 + c4 * 4) =
                  make_uint2(pack16(val.x, val.y, fmt), pack16(val.z, val.w, fmt));
          }
        }
      }
    } else {
      // ---------------- 16-bit outputs only: phase A packs into a [128][BN + 8] tile
      constexpr int P16 = BN + 8;
      uint16_t* stg = reinterpret_cast<uint16_t*>(smem + S::OFF_STG);
      const int ncols = min(BN, a.n_store - n0);  // columns of this tile that exist (multiple of 32)
      for (int c0 = 32 * half; c0 < ncols; c0 += 64) {
        acc_row32(accs + row * AP + c0, v);
        float o[32];
        if (EPI == EPI_QKV) {
          const int slot = (n0 + c0) >> 5;
          float ss = 0.f;
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            o[j] = __uint_as_float(v[j]) + s_bias[c0 + j];
            ss = fmaf(o[j], o[j], ss);
          }
          const float sc = __ldg(a.slot_scale + slot);
          // x / max(||x||, 1e-12) == x * rsqrt(max(||x||^2, 1e-24));  scale <= 0 marks a value slot
          const float mul = sc > 0.f ? sc * rsqrtf(fmaxf(ss, 1e-24f)) : 1.0f;
#pragma unroll
          for (int j = 0; j < 32; ++j) o[j] *= mul;
        } else {
#pragma unroll
          for (int j = 0; j < 32; ++j) o[j] = tc_act(__uint_as_float(v[j]) + s_bias[c0 + j], a.act, a.slope);
        }
#pragma unroll
        for (int j = 0; j < 32; j += 8)
          *reinterpret_cast<uint4*>(stg + row * P16 + c0 + j) =
              make_uint4(pack16(o[j], o[j + 1], fmt), pack16(o[j + 2], o[j + 3], fmt), pack16(o[j + 4], o[j + 5], fmt),
                         pack16(o[j + 6], o[j + 7], fmt));
      }
      epi_barrier();
      const int nvec = min((long long)ncols, (long long)a.ldo_bf16 - n0) >> 3;  // 16-byte vectors per row
      const int ew = et >> 5;
      if (CONV && a.ps_r > 0) {
        // PixelShuffle folded into the store (upsample.py:6-30): the weights are packed so that column n' = q * Cq + c
        // holds torch's channel c r^2 + q, i.e. Cq consecutive columns are ONE output pixel's channels
        const int ps = a.ps_r, Cq = a.n_store / (ps * ps);
        const int nv = min(BN, a.n_store - n0) >> 3;
#pragma unroll 4
        for (int r = ew; r < kBM; r += kEpiWarps) {
          if (s_tok[r] < 0) continue;
          const int y = ty0 + r / kTW, x = tx0 + r % kTW;
          for (int vv = lane; vv < nv; vv += 32) {
            const int n = n0 + vv * 8;
            const int q = n / Cq, c = n - q * Cq;
            const long long dtok = ((long long)tb * a.H * ps + y * ps + q / ps) * ((long long)a.W * ps) + x * ps + q % ps;
            *reinterpret_cast<uint4*>(out16 + dtok * a.ldo_bf16 + c) = *reinterpret_cast<const uint4*>(stg + r * P16 + vv * 8);
          }
        }
      } else {
#pragma unroll 4
        for (int r = ew; r < kBM; r += kEpiWarps) {
          const long long tok = s_tok[r];
          if (tok < 0) continue;
          for (int vv = lane; vv < nvec; vv += 32)
            *reinterpret_cast<uint4*>(out16 + tok * a.ldo_bf16 + n0 + vv * 8) = *reinterpret_cast<const uint4*>(stg + r * P16 + vv * 8);
        }
      }
    }

}

// -------------------------------------------------------------------------------------
// host side
// -------------------------------------------------------------------------------------
static int make_map(CUtensorMap* m, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                    const cuuint32_t* box, int fmt) {
  EncodeTiledFn fn = encode_tiled_fn();
  if (!fn) return fail(GRL_ERR_CUDA, "cuTensorMapEncodeTiled is not available from the driver");
  cuuint32_t ones[5] = {1, 1, 1, 1, 1};
  CUresult rc = fn(m, fmt == FMT_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(base), dims, strides_bytes,
                   box, ones, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (rc != CUDA_SUCCESS) return fail(GRL_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int)rc);
  return GRL_OK;
}

template <int BN, int EPI, bool CONV>
static int launch_one(const CUtensorMap& tmA, const CUtensorMap& tmB, const GrlTcGemm& a, const GemmTcPlan& pl, dim3 grid,
                      cudaStream_t st) {
  auto kern = gemm_tc_kernel<BN, EPI, CONV>;
  // the attribute is per device: a process that drives several GPUs configures each one once
  static bool configured[kMaxDevices] = {false};
  int dev = 0;
  GRL_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= kMaxDevices || !configured[dev]) {
    GRL_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, GemmSmem<BN>::TOTAL));
    if (dev >= 0 && dev < kMaxDevices) configured[dev] = true;
  }
  kern<<<grid, kThreads, GemmSmem<BN>::TOTAL, st>>>(tmA, tmB, a, pl);
  GRL_LAUNCH_CHECK("gemm_tc_kernel");
  return GRL_OK;
}

template <int EPI, bool CONV>
static int dispatch_bn(int bn, const CUtensorMap& tmA, const CUtensorMap& tmB, const GrlTcGemm& a, const GemmTcPlan& pl,
                       dim3 grid, cudaStream_t st) {
  switch (bn) {
    case 64: return launch_one<64, EPI, CONV>(tmA, tmB, a, pl, grid, st);
    case 128: return launch_one<128, EPI, CONV>(tmA, tmB, a, pl, grid, st);
    case 192: return launch_one<192, EPI, CONV>(tmA, tmB, a, pl, grid, st);
    case 256: return launch_one<256, EPI, CONV>(tmA, tmB, a, pl, grid, st);
  }
  return fail(GRL_ERR_INVALID, "gemm_tc: unsupported tile width %d", bn);
}

static int pick_bn(int npad) {
  if (npad <= 64) return 64;
  if (npad <= 128) return 128;
  if (npad % 192 == 0 || npad <= 192) return 192;
  if (npad % 256 == 0) return 256;
  return npad % 128 == 0 ? 128 : 192;
}

// Host-side validation and launch selection, shared by grl_tc_gemm and grl_tc_gemm_path (so the path a test asks about is
// the path that runs): checks every argument of p but its null test, fills the plan (epi_mode, nk, M, conv tiling,
// n_tiles, total_tiles = grid) and returns the N tile width in *bn.  Needs no device.
static int plan_gemm_tc(const GrlTcGemm& p, GemmTcPlan& pl, int* bn_out) {
  pl = GemmTcPlan{};
  pl.nchw_r = p.nchw_r > 0 ? p.nchw_r : 1;
  if (check_fmt(p.fmt)) return GRL_ERR_INVALID;
  GRL_REQUIRE(p.bias != nullptr, "tc_gemm: bias is required (pass zeros)");
  GRL_REQUIRE(p.n_store <= p.npad && p.n_real <= p.npad, "tc_gemm: n_store/n_real exceed npad");
  if (p.epi == EPI_QKV) GRL_REQUIRE(p.slot_scale && p.out_bf16 && p.ldo_bf16 >= p.npad, "tc_gemm: QKV epilogue arguments");
  if (p.epi == EPI_LN)
    GRL_REQUIRE(p.gamma && p.beta && p.res_f32 && p.out_f32 && p.out_bf16 && p.C > 0 && p.C <= p.npad &&
                    p.L > 0 && (p.ldo_f32 % 4) == 0 && (p.ldo_bf16 % 8) == 0,
                "tc_gemm: LN epilogue arguments");
  if (p.out_bf16) GRL_REQUIRE((p.ldo_bf16 % 8) == 0, "tc_gemm: bf16 output pitch must be a multiple of 8");
  GRL_REQUIRE(p.kpad % kBK == 0 && p.kpad > 0, "gemm_tc: K pad %d must be a multiple of 64", p.kpad);
  GRL_REQUIRE(p.npad % 32 == 0 && p.npad > 0, "gemm_tc: N pad %d must be a multiple of 32", p.npad);
  int bn = (p.epi == EPI_LN) ? (p.npad <= 64 ? 64 : p.npad <= 128 ? 128 : p.npad <= 192 ? 192 : 256) : pick_bn(p.npad);
  GRL_REQUIRE(p.epi != EPI_LN || p.npad <= 256, "gemm_tc: LayerNorm epilogue needs the whole row in one tile (N=%d)",
              p.npad);
  const bool conv = p.taps == 9;
  if (p.ps_r > 0)
    GRL_REQUIRE(conv && p.epi == EPI_BIAS_ACT && !p.out_f32 && !p.res_f32 && p.out_bf16 && p.n_store % (p.ps_r * p.ps_r) == 0 &&
                    (p.n_store / (p.ps_r * p.ps_r)) % 8 == 0 && p.ldo_bf16 >= p.n_store / (p.ps_r * p.ps_r),
                "gemm_tc: pixel-shuffle store needs a 16-bit-only conv epilogue with N %% r^2 == 0 and N / r^2 %% 8 == 0");
  if (p.out_nchw)
    GRL_REQUIRE(conv && p.epi == EPI_BIAS_ACT && pl.nchw_r >= 1 && p.n_real % (pl.nchw_r * pl.nchw_r) == 0 &&
                    p.n_real / (pl.nchw_r * pl.nchw_r) <= 4 && p.Hc > 0 && p.Wc > 0,
                "gemm_tc: NCHW tail store needs a conv with <= 4 output channels");
  GRL_REQUIRE(p.taps == 1 || p.taps == 9, "gemm_tc: taps must be 1 or 9");
  // Epilogue mode.  fp32 staging (LayerNorm, fp32 output, residual) needs the whole output row in one tile, 16-byte
  // aligned fp32 rows and a tile that fits the staging area; anything else with an fp32 side takes the direct path.
  pl.epi_mode = 0;
  if (p.epi == EPI_LN || (p.epi == EPI_BIAS_ACT && (p.out_f32 || p.res_f32))) {
    const int cw = p.epi == EPI_LN ? p.C : p.n_real;
    const int cap = bn == 64 ? GemmSmem<64>::STG : bn == 128 ? GemmSmem<128>::STG : bn == 192 ? GemmSmem<192>::STG
                                                                                               : GemmSmem<256>::STG;
    const bool ok = p.npad <= bn && cw > 0 && cw % 4 == 0 && kBM * stage_pitch32(cw) * 4 <= cap &&
                    (!p.out_f32 || p.ldo_f32 % 4 == 0) && (!p.res_f32 || p.ldr % 4 == 0) &&
                    (!p.out_bf16 || p.ldo_bf16 % 4 == 0);
    GRL_REQUIRE(ok || p.epi != EPI_LN, "gemm_tc: LayerNorm epilogue needs C %% 4 == 0 and C <= 188 (got %d)", cw);
    pl.epi_mode = ok ? 1 : 2;
  }
  if (p.out_nchw) pl.epi_mode = 2;
  GRL_REQUIRE(p.epi == EPI_BIAS_ACT || p.epi == EPI_QKV || p.epi == EPI_LN, "gemm_tc: unknown epilogue %d", p.epi);
  GRL_REQUIRE(!conv || p.epi == EPI_BIAS_ACT, "gemm_tc: %s epilogue is linear-only", p.epi == EPI_QKV ? "QKV" : "LN");
  pl.nk = p.kpad / kBK;
  pl.n_tiles = ceil_div(p.npad, bn);
  if (conv) {
    pl.tiles_x = ceil_div(p.W, kTW), pl.tiles_y = ceil_div(p.H, kTH);
    pl.M = (long long)p.B * p.H * p.W;
    GRL_REQUIRE((long long)pl.tiles_x * pl.tiles_y * p.B * pl.n_tiles < (1ll << 31), "gemm_tc: grid too large");
    pl.total_tiles = pl.tiles_x * pl.tiles_y * p.B * pl.n_tiles;
  } else {
    pl.M = p.M;
    GRL_REQUIRE((long long)ceil_div(p.M, kBM) * pl.n_tiles < (1ll << 31), "gemm_tc: grid too large");
    pl.total_tiles = (int)(ceil_div(p.M, kBM) * pl.n_tiles);
  }
  *bn_out = bn;
  return GRL_OK;
}

}  // namespace tc
}  // namespace grl

using namespace grl;
using namespace grl::tc;

extern "C" {

// x: bf16 (M, Kpad) row-major or (B, H, W, Kpad) channels-last; w: bf16 (Npad, taps*Kpad) K-major.
int grl_tc_gemm(const GrlTcGemm* p, void* stream) {
  GRL_REQUIRE(p != nullptr, "tc_gemm: null problem");
  if (!grl_device_ok()) return fail(GRL_ERR_ARCH, "tc_gemm: wgmma kernels need an sm_90 device");
  GemmTcPlan pl;
  int bn = 0, rc;
  if ((rc = plan_gemm_tc(*p, pl, &bn)) != GRL_OK) return rc;
  if (pl.M == 0) return GRL_OK;
  CUtensorMap tmA, tmB;
  if (p->taps == 9) {
    cuuint64_t dims[4] = {(cuuint64_t)p->kpad, (cuuint64_t)p->W, (cuuint64_t)p->H, (cuuint64_t)p->B};
    cuuint64_t str[3] = {(cuuint64_t)p->kpad * 2, (cuuint64_t)p->W * p->kpad * 2, (cuuint64_t)p->H * p->W * p->kpad * 2};
    cuuint32_t box[4] = {(cuuint32_t)kBK, (cuuint32_t)kTW, (cuuint32_t)kTH, 1};
    if ((rc = make_map(&tmA, p->x, 4, dims, str, box, p->fmt)) != GRL_OK) return rc;
  } else {
    cuuint64_t dims[2] = {(cuuint64_t)p->kpad, (cuuint64_t)p->M};
    cuuint64_t str[1] = {(cuuint64_t)p->kpad * 2};
    cuuint32_t box[2] = {(cuuint32_t)kBK, (cuuint32_t)kBM};
    if ((rc = make_map(&tmA, p->x, 2, dims, str, box, p->fmt)) != GRL_OK) return rc;
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)p->kpad * p->taps, (cuuint64_t)p->npad};
    cuuint64_t str[1] = {(cuuint64_t)p->kpad * p->taps * 2};
    cuuint32_t box[2] = {(cuuint32_t)kBK, (cuuint32_t)bn};
    if ((rc = make_map(&tmB, p->w, 2, dims, str, box, p->fmt)) != GRL_OK) return rc;
  }
  const dim3 grid((unsigned)pl.total_tiles);
  const cudaStream_t st = (cudaStream_t)stream;
  switch (p->epi) {
    case EPI_QKV: return dispatch_bn<EPI_QKV, false>(bn, tmA, tmB, *p, pl, grid, st);
    case EPI_LN: return dispatch_bn<EPI_LN, false>(bn, tmA, tmB, *p, pl, grid, st);
  }
  return p->taps == 9 ? dispatch_bn<EPI_BIAS_ACT, true>(bn, tmA, tmB, *p, pl, grid, st)
                      : dispatch_bn<EPI_BIAS_ACT, false>(bn, tmA, tmB, *p, pl, grid, st);
}

int grl_tc_gemm_path(const GrlTcGemm* p, GrlTcGemmPath* out) {
  GRL_REQUIRE(out != nullptr, "tc_gemm_path: null output");
  GRL_REQUIRE(p != nullptr, "tc_gemm: null problem");
  GemmTcPlan pl;
  int bn = 0, rc;
  if ((rc = plan_gemm_tc(*p, pl, &bn)) != GRL_OK) return rc;
  out->bn = bn, out->epi_mode = pl.epi_mode, out->conv = p->taps == 9, out->n_tiles = pl.n_tiles;
  out->nk_total = p->taps * pl.nk, out->grid = pl.total_tiles;
  return GRL_OK;
}

}  // extern "C"
