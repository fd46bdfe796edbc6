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
// 256 threads = two warpgroups (rows 0-63 / 64-127 of the tile, wgmma m64n64k16 per 64 output columns, accumulators
// in registers); thread 0 also issues the TMA loads into a 2-4 stage ring.  The epilogue works on the accumulator
// fragments themselves: the 4 threads of a quad hold whole rows, so LayerNorm moments and per-slot norms are quad
// shuffles.  No fp32 tile goes through shared memory, and up to BN = 192 two CTAs share an SM, one tile's epilogue
// overlapping the other's loads and MMAs.  These GEMMs are short-K and HBM / epilogue bound, not tensor bound
// (DESIGN.md).
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

constexpr int kBM = 128, kBK = 64;
constexpr int kTH = 8, kTW = 16;  // conv patch (kTH * kTW == kBM)
constexpr int kWarps = 8, kThreads = kWarps * 32;
// CTAs per SM.  Up to BN = 192 two CTAs share an SM, so that one tile's epilogue runs while the other tile's loads and
// MMAs are in flight: 2 x 8 warps leave 128 registers per thread (each quarter of the register file serves 4 warps;
// BN = 192 holds 96 accumulators) and ~113 KB of shared memory per CTA.  BN = 256 holds 128 accumulators: one CTA.
__host__ __device__ constexpr int ctas_per_sm(int bn) { return bn <= 192 ? 2 : 1; }

// Shared memory: the operand ring (up to 4 stages, at most 100 KB when two CTAs share the SM) and, once the main loop
// is over, the epilogue's staging (aliases the ring): the 16-bit output tile [128][BN + 8] that makes row-major 16-byte
// stores, or two fp32 row chunks [128][72]; then the per-CTA tables.
template <int BN>
struct GemmSmem {
  static constexpr int A_BYTES = kBM * kBK * 2;
  static constexpr int B_BYTES = BN * kBK * 2;
  static constexpr int STAGE = A_BYTES + B_BYTES;
  static constexpr int RING = ctas_per_sm(BN) == 2 ? 100 * 1024 : 4 * STAGE;
  static constexpr int STAGES = RING / STAGE < 4 ? RING / STAGE : 4;
  static constexpr int PIPE = STAGES * STAGE;
  static constexpr int P16 = BN + 8;  // 16-bit tile pitch (halves): (BN + 8) / 2 % 32 == 4, conflict-free quad writes
  static constexpr int OFF_TOK = PIPE;                         // long long tok[128], int img[128]
  static constexpr int OFF_PAR = OFF_TOK + 128 * 8 + 128 * 4;  // float bias[BN], gamma[BN], beta[BN]
  static constexpr int OFF_BAR = OFF_PAR + 3 * BN * 4;
  static constexpr int TOTAL = OFF_BAR + STAGES * 8 + 1024 /*align slack*/;
  static_assert(STAGES >= 2, "operand ring");
  static_assert(kBM * P16 * 2 <= PIPE, "16-bit tile fits the ring");
  static_assert(ctas_per_sm(BN) * (TOTAL + 1024) <= 232448, "shared memory per SM (1 KB reserved per CTA)");
};

// sum over the 4 threads of a quad (the threads that hold one accumulator row)
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// Main loop of warpgroup `half`: rows [64 half, 64 half + 64) of the tile, BN / 64 accumulators of m64n64.  Thread 0
// issues the TMA loads (load(kc) fills stage kc % STAGES and arms its full barrier): the first STAGES chunks up front,
// then chunk kc - 1 + STAGES once both warpgroups have finished the MMAs that read chunk kc - 1.
// FMT is a template argument so that no branch separates the wgmma instructions of one k step.
template <int BN, int FMT, class Load>
__device__ __forceinline__ void mma_loop(float (&acc)[BN / 64][32], uint8_t* smem, uint64_t* full, int nk_total,
                                         int half, const Load& load) {
  using S = GemmSmem<BN>;
  for (int kc = 0; kc < nk_total; ++kc) {
    const int s = kc % S::STAGES;
    // The previous step's MMAs are in flight here.  ptxas reports C7517 for every instance: it puts a wait for them on
    // mbar_wait's trap branch (a protocol fault), not on this path, which keeps one k step in flight.
    mbar_wait(&full[s], (kc / S::STAGES) & 1);
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
    // this k step's MMAs stay in flight; the previous step's are complete, so its stage can be refilled
    wgmma_wait<1>();
    if (kc > 0 && kc - 1 + S::STAGES < nk_total) {
      __syncthreads();  // ... by both warpgroups
      if (threadIdx.x == 0) load(kc - 1 + S::STAGES);
    }
  }
  wgmma_wait<0>();
}

// What the host derives from a GrlTcGemm for its launch (plan_gemm_tc); the kernel takes both.
struct GemmTcPlan {
  long long M;   // rows: GrlTcGemm::M, or B * H * W for a conv
  int nk;        // 64-wide k chunks per tap
  int n_tiles, total_tiles;
  int tiles_x, tiles_y;  // conv: 8 x 16 pixel patches per image
  int epi_mode;  // 0 = 16-bit outputs, 1 = whole fp32 rows (LayerNorm / fp32 output / residual), 2 = direct
  int nchw_r;    // GrlTcGemm::nchw_r, at least 1
};

template <int BN, int EPI, bool CONV>
__global__ void __launch_bounds__(kThreads, ctas_per_sm(BN))
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GrlTcGemm a,
              const GemmTcPlan pl) {
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte aligned (SWIZZLE_128B operands) by pointer arithmetic, so that the compiler keeps the shared state space
  // (LDS / STS with 32-bit addresses in the epilogue, not generic accesses)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  using S = GemmSmem<BN>;
  constexpr int NJ = BN / 64;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + S::OFF_BAR);
  long long* s_tok = reinterpret_cast<long long*>(smem + S::OFF_TOK);
  int* s_img = reinterpret_cast<int*>(smem + S::OFF_TOK + 128 * 8);  // image (batch) index of every row (CAB gate)
  float* s_bias = reinterpret_cast<float*>(smem + S::OFF_PAR);      // this tile's columns [n0, n0 + BN)
  float* s_gamma = s_bias + BN;
  float* s_beta = s_gamma + BN;

  const int lane = threadIdx.x & 31;
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

  // TMA: chunk kc of the A tile (a tap's shifted box for a conv) and of the W tile into stage kc % STAGES
  auto load = [&](int kc) {
    const int s = kc % S::STAGES;
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
  };
  if (threadIdx.x == 0) {
    for (int s = 0; s < S::STAGES; ++s) mbar_init(&full[s], 1);
    mbar_init_fence();
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int kc = 0; kc < S::STAGES && kc < nk_total; ++kc) load(kc);
  }

  const int et = threadIdx.x;  // 0..255
  const int half = et >> 7;    // MMA warpgroup: rows [64 half, 64 half + 64)
  const int fmt = a.fmt;
  uint16_t* out16 = reinterpret_cast<uint16_t*>(a.out_bf16);
  // per-tile tables: token (global row) of every accumulator row (-1 = outside the problem), its image, and the
  // per-column constants of this N tile
  if (et < kBM) {
    long long tok;
    if (CONV) {
      const int y = ty0 + et / kTW, x = tx0 + et % kTW;
      tok = (y < a.H && x < a.W) ? ((long long)tb * a.H + y) * a.W + x : -1;
    } else {
      tok = (long long)m0 + et;
      if (tok >= pl.M) tok = -1;
    }
    s_tok[et] = tok;
    s_img[et] = (EPI == EPI_LN && tok >= 0) ? (int)(tok / a.L) : 0;  // one 64-bit division per row, not per access
  }
  for (int c = et; c < BN; c += kThreads) {
    const int n = n0 + c;
    s_bias[c] = (n < a.n_store) ? a.bias[n] : 0.f;
    if (EPI == EPI_LN) {
      s_gamma[c] = (c < a.C) ? a.gamma[c] : 0.f;
      s_beta[c] = (c < a.C) ? a.beta[c] : 0.f;
    }
  }

  float acc[NJ][32];
#pragma unroll
  for (int j = 0; j < NJ; ++j)
#pragma unroll
    for (int e = 0; e < 32; ++e) acc[j][e] = 0.f;
  __syncthreads();  // the barriers are initialised and the tables written
  if (fmt == FMT_BF16) mma_loop<BN, FMT_BF16>(acc, smem, full, nk_total, half, load);
  else mma_loop<BN, FMT_F16>(acc, smem, full, nk_total, half, load);
  __syncthreads();  // both warpgroups are done reading the ring: it becomes the epilogue's staging area

  // ---------------- epilogue on the accumulator fragments (tc_common.cuh): this thread holds rows r0 and r0 + 8
  // (h = 0, 1), columns 64 j + 8 i + cq + {0, 1}; the 4 threads of a quad hold the whole of both rows.
  // acc[j][4 i + 2 h + e]  <->  row r0 + 8 h, column 64 j + 8 i + cq + e
  const int r0 = half * 64 + 16 * ((et >> 5) & 3) + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < NJ; ++j)
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float2 b = *reinterpret_cast<const float2*>(s_bias + 64 * j + 8 * i + cq);
      acc[j][4 * i] += b.x, acc[j][4 * i + 1] += b.y, acc[j][4 * i + 2] += b.x, acc[j][4 * i + 3] += b.y;
    }
  uint16_t* stg = reinterpret_cast<uint16_t*>(smem);  // [128][P16]
  constexpr int P16 = S::P16;

  // epi_mode (chosen on the host): 1 = whole fp32 rows in this tile (LayerNorm / fp32 result / residual), 0 = 16-bit
  // outputs only, 2 = direct per-element stores (odd widths such as the 3-channel image head)
  if (EPI == EPI_BIAS_ACT && pl.epi_mode == 2) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = r0 + 8 * h;
      const long long t = s_tok[row];
      if (t < 0) continue;
#pragma unroll
      for (int j = 0; j < NJ; ++j)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int c = 64 * j + 8 * i + cq;
          if (n0 + (c & ~31) >= a.n_store) continue;  // 32-column chunks past the stored columns are not written
          float o[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int n = n0 + c + e;
            float val = tc_act(acc[j][4 * i + 2 * h + e], a.act, a.slope);
            if (a.res_f32 && n < a.n_real) val += __ldg(a.res_f32 + t * a.ldr + n);
            o[e] = (n < a.n_store) ? val : 0.f;
            if (a.out_f32 && n < a.n_real) a.out_f32[t * a.ldo_f32 + n] = o[e];
            if (CONV && a.out_nchw && n < a.n_real) {
              // tail fusion: x / img_range + mean (grl.py:549), the crop (:551), channels-last -> bchw and, for the
              // one-step head, PixelShuffle (upsample.py:33-50; torch order n = c r^2 + dy r + dx) folded into the store
              const int r = pl.nchw_r, rr = r * r;
              const int ch = n / rr, q = n - ch * rr;
              const int yy = (ty0 + row / kTW) * r + q / r, xx = (tx0 + row % kTW) * r + q % r;
              if (yy < a.Hc && xx < a.Wc)
                a.out_nchw[(((long long)tb * (a.n_real / rr) + ch) * a.Hc + yy) * a.Wc + xx] =
                    fmaf(o[e], a.post_scale, a.post_shift[ch & 3]);
            }
          }
          if (out16 && n0 + (c & ~7) < a.ldo_bf16)
            *reinterpret_cast<uint32_t*>(out16 + t * a.ldo_bf16 + n0 + c) = pack16(o[0], o[1], fmt);
        }
    }
    return;
  }

  if (EPI == EPI_LN || pl.epi_mode == 1) {  // LayerNorm always has mode 1
    // n0 == 0: the tile holds whole rows.  The rows go through shared memory 64 columns at a time, in two fp32 buffers
    // [128][72] that alias the idle ring: the residual of chunk j + 1 is fetched with cp.async (16 B per request) while
    // chunk j is finished, the fragments add their result in place, and the chunk is streamed row-major (CAB term,
    // fp32 store, 16-bit copy) -- coalesced residual reads and stores with many requests in flight.
    const int Cw = (EPI == EPI_LN) ? a.C : a.n_real;  // real fp32 columns, Cw % 4 == 0
    constexpr int RP = 72;                             // pitch % 32 == 8: conflict-free float2 quad writes
    static_assert(2 * kBM * RP * 4 <= S::PIPE, "two fp32 chunk buffers fit the ring");
    float* rbuf = reinterpret_cast<float*>(smem);
    const bool has_res = a.res_f32 != nullptr;
    auto fetch = [&](int j) {  // residual columns [64 j, 64 j + 64) of every row -> buffer j % 2
      if (has_res)
        for (int idx = et; idx < kBM * 16; idx += kThreads) {
          const int r = idx >> 4, c = 64 * j + 4 * (idx & 15);
          const long long t = s_tok[r];
          if (c < Cw) cp_async_16(rbuf + (j & 1) * kBM * RP + r * RP + (c & 63), a.res_f32 + (t >= 0 ? t : 0) * a.ldr + c, t >= 0);
        }
      cp_async_commit();
    };
    fetch(0);
    float mean[2] = {0.f, 0.f}, rstd[2] = {0.f, 0.f};
    if (EPI == EPI_LN) {
      // Shifted single-pass moments of each row: x0 = the row's first element (no catastrophic cancellation),
      // mean = x0 + S1/n, M2 = S2 - S1^2/n with S1 = sum(x - x0), S2 = sum((x - x0)^2); the quad's partial sums are added.
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float x0 = __shfl_sync(0xffffffffu, acc[0][2 * h], lane & ~3);
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int j = 0; j < NJ; ++j)
#pragma unroll
          for (int i = 0; i < 8; ++i)
            if (64 * j + 8 * i < Cw - cq) {  // both columns of the pair: Cw and cq are even
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const float d = acc[j][4 * i + 2 * h + e] - x0;
                s1 += d;
                s2 = fmaf(d, d, s2);
              }
            }
        s1 = quad_sum(s1);
        s2 = quad_sum(s2);
        const float fn = (float)Cw, m1 = s1 / fn;
        mean[h] = x0 + m1;
        rstd[h] = rsqrtf(fmaxf(s2 - s1 * m1, 0.f) / fn + a.eps);
      }
    }
    const bool has_cab = (EPI == EPI_LN) && a.cab_y != nullptr;
    const uint16_t* caby = reinterpret_cast<const uint16_t*>(a.cab_y);
    const int ew = et >> 5, c4 = lane & 15;  // row-major pass: a warp covers 2 rows of a chunk per step
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      if (64 * j >= Cw) break;
      if (j > 0) __syncthreads();  // every thread is done reading chunk j - 1's buffer, which chunk j + 1 refills
      if (64 * (j + 1) < Cw) {
        fetch(j + 1);
        cp_async_wait<1>();
      } else {
        cp_async_wait<0>();
      }
      __syncthreads();  // chunk j's residual has landed for every thread
      float* buf = rbuf + (j & 1) * kBM * RP;
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < 8; ++i)
          if (64 * j + 8 * i < Cw - cq) {
            float2* p = reinterpret_cast<float2*>(buf + (r0 + 8 * h) * RP + 8 * i + cq);
            float2 o = has_res ? *p : make_float2(0.f, 0.f);
            const float v0 = acc[j][4 * i + 2 * h], v1 = acc[j][4 * i + 2 * h + 1];
            if (EPI == EPI_LN) {
              const int c = 64 * j + 8 * i + cq;
              const float2 g = *reinterpret_cast<const float2*>(s_gamma + c), be = *reinterpret_cast<const float2*>(s_beta + c);
              o.x += ((v0 - mean[h]) * rstd[h] * g.x + be.x) * a.res_scale;
              o.y += ((v1 - mean[h]) * rstd[h] * g.y + be.y) * a.res_scale;
            } else {
              o.x += tc_act(v0, a.act, a.slope);
              o.y += tc_act(v1, a.act, a.slope);
            }
            *p = o;
          }
      __syncthreads();
      // rows ew + 8 k (k = 0..15), two per step; the loads of RB steps are issued before their stores (the compiler
      // cannot prove the output and CAB pointers distinct).  The LayerNorm instance batches 2 steps: its CAB operands
      // are 6 registers per step, and at BN = 192 a batch of 4 spills next to the chunks' accumulators.
      const int c = 64 * j + 4 * c4;
      const bool col_real = c < Cw;
      constexpr int RB = EPI == EPI_LN ? 2 : 4;
#pragma unroll
      for (int k0 = 0; k0 < 16; k0 += 2 * RB) {
        long long tk[RB];
        uint2 cy[RB];
        float4 gg[RB];
#pragma unroll
        for (int u = 0; u < RB; ++u) {
          const int r = ew + 8 * (k0 + 2 * u + (lane >> 4));
          tk[u] = s_tok[r];
          cy[u] = make_uint2(0u, 0u);
          gg[u] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (has_cab && tk[u] >= 0 && col_real) {
            cy[u] = __ldg(reinterpret_cast<const uint2*>(caby + tk[u] * a.ld_caby + c));
            gg[u] = __ldg(reinterpret_cast<const float4*>(a.cab_gate + (long long)s_img[r] * Cw + c));
          }
        }
#pragma unroll
        for (int u = 0; u < RB; ++u) {
          const int r = ew + 8 * (k0 + 2 * u + (lane >> 4));
          if (tk[u] < 0) continue;
          float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
          if (col_real) {
            val = *reinterpret_cast<const float4*>(buf + r * RP + 4 * c4);
            if (has_cab) {
              const float2 c01 = unpack16(cy[u].x, fmt), c23 = unpack16(cy[u].y, fmt);
              val.x = fmaf(c01.x, gg[u].x, val.x), val.y = fmaf(c01.y, gg[u].y, val.y);
              val.z = fmaf(c23.x, gg[u].z, val.z), val.w = fmaf(c23.y, gg[u].w, val.w);
            }
            if (a.out_f32) *reinterpret_cast<float4*>(a.out_f32 + tk[u] * a.ldo_f32 + c) = val;
          }
          if (out16 && c < a.ldo_bf16)
            *reinterpret_cast<uint2*>(out16 + tk[u] * a.ldo_bf16 + c) =
                make_uint2(pack16(val.x, val.y, fmt), pack16(val.z, val.w, fmt));
        }
      }
    }
    // the 16-bit copy is written up to its pitch: zero beyond the last chunk
    if (out16) {
      const int cz = (Cw + 63) / 64 * 64;
      for (int idx = et; idx < kBM * ((a.ldo_bf16 - cz) >> 2); idx += kThreads) {
        const int per = (a.ldo_bf16 - cz) >> 2, r = idx / per, c = cz + 4 * (idx - r * per);
        const long long t = s_tok[r];
        if (t >= 0) *reinterpret_cast<uint2*>(out16 + t * a.ldo_bf16 + c) = make_uint2(0u, 0u);
      }
    }
    return;
  }
  {
    // 16-bit outputs only
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      if (EPI == EPI_QKV) {
        // per 32-wide head slot: x / max(||x||, 1e-12) == x * rsqrt(max(||x||^2, 1e-24)); scale <= 0 marks a value slot
#pragma unroll
        for (int sh = 0; sh < 2; ++sh) {
          const int n = n0 + 64 * j + 32 * sh;
          const float sc = n < a.n_store ? __ldg(a.slot_scale + (n >> 5)) : 0.f;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float ss = 0.f;
#pragma unroll
            for (int i = 4 * sh; i < 4 * sh + 4; ++i)
#pragma unroll
              for (int e = 0; e < 2; ++e) ss = fmaf(acc[j][4 * i + 2 * h + e], acc[j][4 * i + 2 * h + e], ss);
            ss = quad_sum(ss);
            const float mul = sc > 0.f ? sc * rsqrtf(fmaxf(ss, 1e-24f)) : 1.0f;
#pragma unroll
            for (int i = 4 * sh; i < 4 * sh + 4; ++i) acc[j][4 * i + 2 * h] *= mul, acc[j][4 * i + 2 * h + 1] *= mul;
          }
        }
      } else {
#pragma unroll
        for (int e = 0; e < 32; ++e) acc[j][e] = tc_act(acc[j][e], a.act, a.slope);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int h = 0; h < 2; ++h)
          *reinterpret_cast<uint32_t*>(stg + (r0 + 8 * h) * P16 + 64 * j + 8 * i + cq) =
              pack16(acc[j][4 * i + 2 * h], acc[j][4 * i + 2 * h + 1], fmt);
    }
  }
  if (!out16) return;
  __syncthreads();
  // ---------------- the 16-bit tile -> global memory, row-major with 16-byte stores, warp = row group
  const int ew = et >> 5;
  if (CONV && a.ps_r > 0) {
    // PixelShuffle folded into the store (upsample.py:6-30): the weights are packed so that column n' = q * Cq + c
    // holds torch's channel c r^2 + q, i.e. Cq consecutive columns are ONE output pixel's channels
    const int ps = a.ps_r, Cq = a.n_store / (ps * ps);
    const int nv = min(BN, a.n_store - n0) >> 3;
#pragma unroll 4
    for (int r = ew; r < kBM; r += kWarps) {
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
    const int nvec = (int)(min((long long)min(BN, a.n_store - n0), (long long)a.ldo_bf16 - n0) >> 3);
#pragma unroll 4
    for (int r = ew; r < kBM; r += kWarps) {
      const long long t = s_tok[r];
      if (t < 0) continue;
      for (int vv = lane; vv < nvec; vv += 32)
        *reinterpret_cast<uint4*>(out16 + t * a.ldo_bf16 + n0 + vv * 8) = *reinterpret_cast<const uint4*>(stg + r * P16 + vv * 8);
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
  // Epilogue mode.  Whole fp32 rows (LayerNorm, fp32 output, residual) need the whole output row in one tile, rows of
  // 4-column multiples, and at most 188 fp32 columns (132 at BN = 256: the widths the mode has always covered, so that
  // a launch keeps its path); anything else with an fp32 side takes the direct path.
  pl.epi_mode = 0;
  if (p.epi == EPI_LN || (p.epi == EPI_BIAS_ACT && (p.out_f32 || p.res_f32))) {
    const int cw = p.epi == EPI_LN ? p.C : p.n_real;
    const int cw_max = bn == 256 ? 132 : bn == 192 ? 188 : bn;
    const bool ok = p.npad <= bn && cw > 0 && cw % 4 == 0 && cw <= cw_max &&
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
