// attn_tc.cu -- fused cosine attention on wgmma tensor cores (the throughput path of WindowAttention and both
// passes of AnchorStripeAttention; mixed_attn_block_efficient.py:77-94,:128-165,:215-270).
//
// Inputs are the packed bf16 head slots written by the QKV / anchor projection epilogue (gemm_tc.cu, EPI_QKV):
// every head is a 32-wide slot (head_dim zero-padded), q^ / k^ / a^ are already L2-normalised and the side that
// carries the learned logit scale is pre-multiplied by exp(min(logit_scale, ln 100)) * log2(e); the bias table is
// 16*sigmoid(CPB(.))*log2(e).  So   S' = Q K^T   (wgmma, fp32)   and
// P = exp2(S' + bias' + mask' - rowmax')   is softmax(cos*scale + bias + mask) exactly.
//
// One CTA = one (window|stripe, head, 128-query tile).  Keys stream through shared memory in tiles of KT (TMA boxes where
// the rolled window rows have contiguous runs, else cp.async gathers with the roll / partition address arithmetic of
// grl_geometry.h folded in; 64-byte swizzle either way, so the tiles are valid wgmma operands as they land).  Two
// consumer warpgroups own 64 query rows each and keep everything of their rows in registers:
//   S  = Q K^T        m64n64k16, A = Q rows [64 x 32] K-major SW64 (smem), B = K tile [KT x 32] K-major SW64
//   P                 exp2(S + bias + mask - m_ref) on the accumulator fragment (lazily rescaled reference, kTau), 16-bit
//   O += P V          m64n32k16, A = P from registers (the S fragment is the A fragment), B = V tile [KT x 32] MN-major SW64
// O stays in the wgmma accumulator across tiles and is rescaled in place on the rare tiles whose reference moves.  The
// tensor core overlaps one warpgroup's products with the softmax of the other three warpgroups on the SM (two CTAs).
#include <stdlib.h>
#include <string.h>

#include "grl_common.cuh"
#include "attn_tc.cuh"
#include "tc_common.cuh"

namespace grl {
namespace tc {

// One 64-byte row of a Q / K / V tile -> shared memory: the lane that owns the row issues its four 16-byte cp.async.
#define GRL_ROW_COPY(base, r, src, ok)                                                      \
  do {                                                                                      \
    _Pragma("unroll") for (int c_ = 0; c_ < 4; ++c_) cp_async_16((base) + sw64((r), c_), (src) + c_ * 8, (ok)); \
  } while (0)

constexpr int kAttnStages = 4;                 // K / V ring depth
constexpr int kAttnThreads = 2 * 128 + 32;     // two consumer warpgroups (64 query rows each) + 1 producer warp
// Two CTAs per SM: four consumer warpgroups hide each other's MMA, load and barrier latency.  Registers are allocated
// per SM sub-partition (16,384 each, a quarter of the resident warps): the 18 warps of two CTAs put 5 warps on one, so
// ptxas is capped at 16,384 / (5 x 32) rounded down to the allocation granularity of 8, 96 registers per thread.  Three
// CTAs (27 warps, 7 on one sub-partition) would cap it at 72, where the loop spills its O accumulator (DESIGN 5.2).
constexpr int kAttnCtasPerSm = 2;
static_assert(kAttnCtasPerSm * (AttnSmem<64, kAttnStages>::TOTAL + 1024) <= 228 * 1024,
              "the attention CTAs of one SM (plus the 1 KB the runtime reserves per CTA) must fit in its 228 KB of shared memory");

// OR of `pred` over the 64 threads of named barrier `id` (one warp pair = 32 consecutive query rows)
__device__ __forceinline__ bool pair_any(bool pred, int id) {
  uint32_t r;
  asm volatile(
      "{\n\t.reg .pred p, q;\n\tsetp.ne.u32 q, %1, 0;\n\tbar.red.or.pred p, %2, 64, q;\n\tselp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(r)
      : "r"((uint32_t)pred), "r"(id)
      : "memory");
  return r != 0;
}

// Warp-specialised pipeline (tiles t = 0..nt-1 of KT keys, a ring of kAttnStages buffers of K / V / key metadata):
//   warp 8 (producer): TMA boxes or cp.async gathers of Q / K_t / V_t (roll + partition addressing), the key offsets / region ids
//       of tile t, into stage t % NS once the consumers have released it (kv_empty); publishes them on kv_full.
//   warpgroups 0, 1 (query rows 64g..64g+63): wait kv_full(t) -> bias into the accumulator -> S_t = bias + Q K_t^T
//       (fragment) -> mask -> lazy rescale -> 16-bit P_t in registers -> O += P_t V_t -> release stage t.
// KW: key-window width when it is a power of two >= 8 (each column pair's bias read as one aligned float2 from the
// shifted table copies), 0 = generic scalar path.
// VAR: bit 0 = bf16 operands (else fp16), bit 1 = ones-column denominators -- compile-time so the exp / pack loop has no
// uniform branches.
// TMA boxes of the token tensors for geometries whose window rows split into aligned runs of box tokens that are
// contiguous in memory (attn_tma_box_tokens); box_* = 0: that operand is gathered row by row with cp.async.
struct AttnMaps {
  CUtensorMap q, k, v;  // (tokens, ld) 16-bit, box {32 channels, box_* tokens}, SWIZZLE_64B
  int box_q, box_k;
};

template <int KT, int KW, int VAR>
__global__ void __launch_bounds__(kAttnThreads, kAttnCtasPerSm) attn_tc_kernel(const __grid_constant__ AttnMaps tm, const GrlTcAttn a) {
  static_assert(KT == 64, "S fragments of m64n64 products: one key tile per product");
  constexpr int NS = kAttnStages;
  extern __shared__ uint8_t smem_raw[];
  // aligned up to 1024 bytes by an offset from smem_raw, so that the compiler keeps every pointer below in the shared
  // window (LDS / STS rather than generic loads)
  uint8_t* smem = smem_raw + ((0u - smem_u32(smem_raw)) & 1023u);
  using S = AttnSmem<KT, NS>;
  uint8_t* Qs = smem;
  uint8_t* Ks = smem + S::OFF_K;
  uint8_t* Vs = smem + S::OFF_V;
  int* koff_s = reinterpret_cast<int*>(smem + S::OFF_META);  // [NS][KT]
  int* krid_s = koff_s + NS * KT;                             // [NS][KT]
  uint64_t* kv_full = reinterpret_cast<uint64_t*>(smem + S::OFF_BAR);  // [NS] tile landed (32 producer arrivals)
  uint64_t* kv_empty = kv_full + NS;                                   // [NS] tile consumed (1 arrival per warpgroup)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int Nq = a.gq.wh * a.gq.ww, Nk = a.gk.wh * a.gk.ww;
  const int nqt = (Nq + kQT - 1) / kQT;
  const int nww = a.gq.W / a.gq.ww;
  const int nwh = a.gq.H / a.gq.wh;
  const int nW = nwh * nww;
  int bid = blockIdx.x;
  const int qt = bid % nqt;
  bid /= nqt;
  const int h = bid % a.heads;
  const int bw = bid / a.heads;
  const int b = bw / nW, w = bw - b * nW;
  const int wr = w / nww, wc = w - wr * nww;
  const int Wt = a.gq.ww + a.gk.ww - 1;
  const int ntiles = (Nk + KT - 1) / KT;
  // a warpgroup whose 64 rows all lie beyond Nq has nothing to compute (its rows form rescale groups of their own)
  const int nwg = Nq - qt * kQT > 64 ? 2 : 1;

  if (tid == 0) {
    for (int i = 0; i < NS; ++i) {
      mbar_init(&kv_full[i], 32);
      mbar_init(&kv_empty[i], nwg);
    }
    mbar_init_fence();
  }
  __syncthreads();
  constexpr int fmt = (VAR & 1) ? FMT_BF16 : FMT_F16;

  if (warp == 8) {
    // =============================================================== producer
    for (int t = 0; t < ntiles; ++t) {
      const int buf = t % NS, k0 = t * KT;
      if (t >= NS) mbar_wait(&kv_empty[buf], (t / NS - 1) & 1);  // tile t - NS is consumed
      // Q (first tile) and K / V of full tiles come as TMA boxes where the geometry has them; tails and dense V are gathered
      const bool tma_q = t == 0 && tm.box_q > 0 && (qt + 1) * kQT <= Nq;
      const bool tma_k = tm.box_k > 0 && k0 + KT <= Nk;
      const bool tma_v = tma_k && !a.v_dense;
      if (t == 0 && !tma_q) {
        for (int r = lane; r < kQT; r += 32) {
          const int qi = qt * kQT + r;
          const bool ok = qi < Nq;
          const Tok tq = locate(a.gq, wr, wc, ok ? qi : 0);
          const __nv_bfloat16* src = static_cast<const __nv_bfloat16*>(a.q) + ((long long)(b * a.gq.H + tq.y) * a.gq.W + tq.x) * a.ldq + a.q_off + h * kDP;
          GRL_ROW_COPY(Qs, r, src, ok);
        }
      }
      for (int r = lane; r < KT; r += 32) {
        const int kj = k0 + r;
        const bool ok = kj < Nk;
        const Tok tk = locate(a.gk, wr, wc, ok ? kj : 0);
        const __nv_bfloat16* ksrc = static_cast<const __nv_bfloat16*>(a.k) + ((long long)(b * a.gk.H + tk.y) * a.gk.W + tk.x) * a.ldk + a.k_off + h * kDP;
        if (!tma_k) GRL_ROW_COPY(Ks + buf * S::KV_BYTES, r, ksrc, ok);
        koff_s[buf * KT + r] = tk.ih * Wt + tk.iw;
        krid_s[buf * KT + r] = region_id(a.gk, tk.r, tk.c);
        const __nv_bfloat16* vsrc;
        if (a.v_dense) {
          vsrc = static_cast<const __nv_bfloat16*>(a.v) + (((long long)bw * a.heads + h) * Nk + (ok ? kj : 0)) * kDP;
        } else {
          vsrc = static_cast<const __nv_bfloat16*>(a.v) + ((long long)(b * a.gk.H + tk.y) * a.gk.W + tk.x) * a.ldv + a.v_off + h * kDP;
        }
        if (!tma_v) GRL_ROW_COPY(Vs + buf * S::KV_BYTES, r, vsrc, ok);
      }
      cp_async_commit();
      cp_async_wait<0>();
      fence_proxy_async_smem();  // the gathered rows -> visible to the tensor core (async proxy)
      if (lane == 0 && (tma_q || tma_k)) {
        // this lane's arrival announces the bytes of the boxes; each box lands at a multiple of 512 bytes, so the
        // 64-byte swizzle TMA applies is the sw64 layout of the gathered rows
        mbar_expect_tx(&kv_full[buf], (tma_q ? S::Q_BYTES : 0) + (tma_k ? S::KV_BYTES : 0) + (tma_v ? S::KV_BYTES : 0));
        if (tma_q)
          for (int j = 0; j < kQT; j += tm.box_q) {
            const Tok tq = locate(a.gq, wr, wc, qt * kQT + j);
            tma_load_2d(Qs + j * 64, &tm.q, &kv_full[buf], a.q_off + h * kDP, (b * a.gq.H + tq.y) * a.gq.W + tq.x);
          }
        if (tma_k)
          for (int j = 0; j < KT; j += tm.box_k) {
            const Tok tk = locate(a.gk, wr, wc, k0 + j);
            const int row = (b * a.gk.H + tk.y) * a.gk.W + tk.x;
            tma_load_2d(Ks + buf * S::KV_BYTES + j * 64, &tm.k, &kv_full[buf], a.k_off + h * kDP, row);
            if (tma_v) tma_load_2d(Vs + buf * S::KV_BYTES + j * 64, &tm.v, &kv_full[buf], a.v_off + h * kDP, row);
          }
      } else {
        mbar_arrive(&kv_full[buf]);
      }
    }
  } else {
    // =============================================================== warpgroups 0, 1: MMAs + softmax on the fragments
    // the warpgroup index through a lane-0 shuffle, so that the compiler knows it is warp-uniform: the key-tile loop
    // then builds its wgmma descriptors with about 20 fewer instructions (2 fewer register-to-uniform moves), for 8-16
    // more once per CTA
    const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0), wq = warp & 3, tig = tid & 127;
    if (wg >= nwg) return;
    // accumulator fragment coordinates: rows fr and fr + 8 of the warpgroup's 64, columns 8i + fc, 8i + fc + 1
    const int fr = 16 * wq + (lane >> 2), fc = 2 * (lane & 3);
    // bias:  idx(i, j) = base_i - koff_j  (grl_geometry.h rel_index); table copy c holds T shifted right by c entries
    // held as one 64-bit register pair: each bias pointer below is then a single 32-bit-index multiply-add from it
    // (left as a uniform parameter plus a 64-bit index, every address costs a chain of 64-bit adds and shifts)
    const float* bias_h = a.bias + (size_t)h * 4 * a.rows_pad;
    asm("mov.b64 %0, %0;" : "+l"(bias_h));
    // What the thread's two rows need per tile (bias base, mask region) and at the end (output element offset) is kept
    // in shared memory and read back when used: registers are the budget of two CTAs per SM.
    int2* row_s = reinterpret_cast<int2*>(smem + S::OFF_ROWS) + 2 * tid;            // base_i[2], q_rid[2]
    long long* dst_s = reinterpret_cast<long long*>(smem + S::OFF_DST) + 2 * tid;  // output offsets, -1: row >= Nq
    {
      int v[4];
#pragma unroll
      for (int j = 0; j < 2; ++j) {  // rows past Nq take query 0's bias and mask row (their Q rows are zero)
        const int qi = qt * kQT + 64 * wg + fr + 8 * j;
        const Tok tq = locate(a.gq, wr, wc, qi < Nq ? qi : 0);
        v[j] = (tq.ih + a.gk.wh - 1) * Wt + tq.iw + a.gk.ww - 1;
        v[2 + j] = region_id(a.gq, tq.r, tq.c);
        dst_s[j] = qi >= Nq ? -1ll
                   : a.o_dense ? (((long long)bw * a.heads + h) * Nq + qi) * kDP
                               : ((long long)(b * a.gq.H + tq.y) * a.gq.W + tq.x) * a.ldo + a.o_off + h * kDP;
      }
      row_s[0] = make_int2(v[0], v[1]);
      row_s[1] = make_int2(v[2], v[3]);
    }
    const bool need_mask = a.use_mask && (wr == nwh - 1 || wc == nww - 1);
    // ones-column: when head_dim < 32 the projection epilogue sets column 31 of every V row to 1, so O[:, 31] =
    // sum_j P_ij is the softmax denominator -- accumulated by the tensor core from the very P it multiplies with V,
    // and rescaled together with the other columns.
    constexpr bool ones = (VAR & 2) != 0;
    // the lazy-rescale decision is shared by 32 consecutive rows: warps 0-1 and 2-3 of the warpgroup (named barriers 1-4)
    const int pair_bar = 1 + 2 * wg + (wq >> 1);

    float oacc[16];
#pragma unroll
    for (int e = 0; e < 16; ++e) oacc[e] = 0.f;
    float m_ref[2] = {0.f, 0.f}, l_run[2] = {0.f, 0.f};

    for (int t = 0; t < ntiles; ++t) {
      const int buf = t % NS, k0 = t * KT;
      mbar_wait(&kv_full[buf], (t / NS) & 1);
      float s[32];
      const int2 rb = row_s[0];  // the region ids are read when the mask needs them
      const int base_i[2] = {rb.x, rb.y};
      // ---- the bias of this tile (log2 domain) is the accumulator's initial value, so that S_t = bias + Q K_t^T comes
      // out of the MMA without a second set of registers; s[4i + 2j + e] = row fr + 8j, column 8i + fc + e
      if ((KW > 0) && (k0 + KT <= Nk)) {
        // keys kj = k0 + 8i + fc, kj + 1 (kj even) are adjacent in one key row: table entries e0 = base - koff(kj), e0 - 1.
        // k0 % 64 == 0 and KW % 8 == 0, so koff(kj) = koff(k0 + fc) + R(i) Wt + C(i) with compile-time R, C.  Key rows
        // R and R + 2 lie 2 Wt entries apart, an even distance, so they read the same table copy: one pointer per row j
        // and key-row parity, the other key rows 2 Wt entries further, the columns at immediate offsets.
        constexpr int KWS = KW > 0 ? KW : 8;
        constexpr int NR = KWS >= 64 ? 1 : KT / KWS;  // key rows in the tile
        const int e00 = (k0 / KWS) * Wt + (k0 % KWS) + fc;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const float* pr[2];
#pragma unroll
          for (int r = 0; r < (NR < 2 ? NR : 2); ++r) {
            const int er = base_i[j] - e00 - r * Wt;  // e0 of key row r's first pair in this tile
            const int cpy = (er + 1) & 1;  // copy in which T[e0 - 1], T[e0] start at an even (8-byte aligned) position
            pr[r] = bias_h + (cpy * (a.rows_pad + 1) + er - 1);
          }
#pragma unroll
          for (int i = 0; i < KT / 8; ++i) {
            // KWS >= 64: the tile lies inside one key row (k0 % KWS + 63 < KWS); else k0 % KWS == 0
            const int R = KWS >= 64 ? 0 : 8 * i / KWS, C = KWS >= 64 ? 8 * i : 8 * i % KWS;
            const float2 bb = __ldg(reinterpret_cast<const float2*>(pr[R & 1] - (R >> 1) * (2 * Wt) - C));
            s[4 * i + 2 * j] = bb.y;
            s[4 * i + 2 * j + 1] = bb.x;
          }
        }
      } else {
        const float* prow[2] = {bias_h + base_i[0], bias_h + base_i[1]};  // T[base_j - koff] = prow[j][-koff]
#pragma unroll
        for (int i = 0; i < KT / 8; ++i) {
          const int2 ko = *reinterpret_cast<const int2*>(koff_s + buf * KT + 8 * i + fc);
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            s[4 * i + 2 * j] = __ldg(prow[j] - ko.x);
            s[4 * i + 2 * j + 1] = __ldg(prow[j] - ko.y);
          }
        }
      }
      {  // ---- S_t = bias + Q K_t^T
        const uint32_t q_sa = smem_u32(Qs) + wg * (64 * 64), k_sa = smem_u32(Ks + buf * S::KV_BYTES);
        wgmma_fence_regs(s);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kDP / 16; ++k) {
          const uint64_t ad = gmma_desc(q_sa + k * 32, 16, 512, SWZ_64B);
          const uint64_t bd = gmma_desc(k_sa + k * 32, 16, 512, SWZ_64B);
          if (fmt == FMT_BF16) wgmma_n64_bf16(s, ad, bd, true);
          else wgmma_n64_f16(s, ad, bd, true);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(s);
      }

      if (need_mask) {
        const int2 rq = row_s[1];
        const int q_rid[2] = {rq.x, rq.y};
#pragma unroll
        for (int i = 0; i < KT / 8; ++i) {
          const int2 rr = *reinterpret_cast<const int2*>(krid_s + buf * KT + 8 * i + fc);
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            if (rr.x != q_rid[j]) s[4 * i + 2 * j] += kMaskLog2;
            if (rr.y != q_rid[j]) s[4 * i + 2 * j + 1] += kMaskLog2;
          }
        }
      }
      if (k0 + KT > Nk) {
#pragma unroll
        for (int i = 0; i < KT / 8; ++i)
#pragma unroll
          for (int e = 0; e < 4; ++e)
            if (k0 + 8 * i + fc + (e & 1) >= Nk) s[4 * i + e] = -INFINITY;
      }
      float mx[2];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        float m0 = s[2 * j], m1 = s[2 * j + 1];
#pragma unroll
        for (int i = 1; i < KT / 8; ++i) m0 = fmaxf(m0, s[4 * i + 2 * j]), m1 = fmaxf(m1, s[4 * i + 2 * j + 1]);
        m0 = fmaxf(m0, m1);
        m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1));
        mx[j] = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
      }
      // Lazy rescale: the reference m_ref moves only when the tile maximum of some row of the 32-row group outgrew it by
      // more than 2^kTau (and on the first tile); P = exp2(x - m_ref) <= 2^kTau stays far inside the fp16 range.
      if (t == 0) {
        m_ref[0] = mx[0], m_ref[1] = mx[1];
      } else if (pair_any(mx[0] - m_ref[0] > kTau || mx[1] - m_ref[1] > kTau, pair_bar)) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const float delta = fmaxf(mx[j] - m_ref[j], 0.f);
          m_ref[j] += delta;
          const float corr = ex2(-delta);
          l_run[j] *= corr;
#pragma unroll
          for (int i = 0; i < kDP / 8; ++i) oacc[4 * i + 2 * j] *= corr, oacc[4 * i + 2 * j + 1] *= corr;
        }
      }
      // ---- P_t, rounded to the operand format, packed straight into the A fragments of the P V product (k-step kk:
      // column blocks 2kk and 2kk + 1)
      uint32_t pa[KT / 16][4];
#pragma unroll
      for (int i = 0; i < KT / 8; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const uint32_t u = pack16(ex2(s[4 * i + 2 * j] - m_ref[j]), ex2(s[4 * i + 2 * j + 1] - m_ref[j]), fmt);
          pa[i >> 1][2 * (i & 1) + j] = u;
          if (!ones) {  // the denominator is the sum of the ROUNDED P that the MMA multiplies with V
            const float2 f = unpack16(u, fmt);
            l_run[j] += f.x + f.y;
          }
        }
      {  // ---- O += P_t V_t
        const uint32_t v_sa = smem_u32(Vs + buf * S::KV_BYTES);
        wgmma_fence_regs(oacc);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < KT / 16; ++kk) {
          const uint64_t bd = gmma_desc(v_sa + kk * 1024, 16, 512, SWZ_64B);
          if (fmt == FMT_BF16) wgmma_rs_n32t_bf16(oacc, pa[kk], bd);
          else wgmma_rs_n32t_f16(oacc, pa[kk], bd);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(oacc);
      }
      // stage t (K / V / metadata) is no longer read: its P V has completed, and that product needed every warp's P
      // fragment, so every warp is past its metadata reads.  (Keeping P_t V_t in flight under S_{t+1} would hold P and
      // the next bias live together, beyond the 96 registers of two CTAs per SM.)
      if (tig == 0) mbar_arrive(&kv_empty[buf]);
    }
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      float den;
      if (ones) {
        den = __shfl_sync(0xffffffffu, oacc[13 + 2 * j], lane | 3);  // O[:, 31]: block 3, column 6 + 1 of lane 4r + 3
      } else {
        den = l_run[j];
        den += __shfl_xor_sync(0xffffffffu, den, 1);
        den += __shfl_xor_sync(0xffffffffu, den, 2);
      }
      const float inv = 1.0f / den;
      const long long off = dst_s[j];
      if (off >= 0) {
        __nv_bfloat16* dst = static_cast<__nv_bfloat16*>(a.out) + off;
#pragma unroll
        for (int i = 0; i < kDP / 8; ++i)
          *reinterpret_cast<uint32_t*>(dst + 8 * i + fc) =
              pack16(oacc[4 * i + 2 * j] * inv, oacc[4 * i + 2 * j + 1] * inv, fmt);
      }
    }
  }
}

template <int KT, int KW, int VAR>
static int launch_attn_var(const AttnMaps& tm, const GrlTcAttn& a, unsigned nblk, cudaStream_t st) {
  auto kern = attn_tc_kernel<KT, KW, VAR>;
  // the attribute is per device: a process that drives several GPUs configures each one once
  static bool configured[kMaxDevices] = {false};
  int dev = 0;
  GRL_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= kMaxDevices || !configured[dev]) {
    GRL_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, AttnSmem<KT, kAttnStages>::TOTAL));
    if (dev >= 0 && dev < kMaxDevices) configured[dev] = true;
  }
  kern<<<nblk, kAttnThreads, AttnSmem<KT, kAttnStages>::TOTAL, st>>>(tm, a);
  GRL_LAUNCH_CHECK("attn_tc_kernel");
  return GRL_OK;
}

template <int KT, int KW>
static int launch_attn_one(const AttnMaps& tm, const GrlTcAttn& a, unsigned nblk, cudaStream_t st) {
  switch ((a.fmt == FMT_BF16 ? 1 : 0) | (a.ones_col ? 2 : 0)) {
    case 0: return launch_attn_var<KT, KW, 0>(tm, a, nblk, st);
    case 1: return launch_attn_var<KT, KW, 1>(tm, a, nblk, st);
    case 2: return launch_attn_var<KT, KW, 2>(tm, a, nblk, st);
    default: return launch_attn_var<KT, KW, 3>(tm, a, nblk, st);
  }
}

// Tokens per TMA box for a window of width ww rolled by sw: the largest power of two <= 64 dividing gcd(ww, sw) (ww if the
// grid is not rolled horizontally).  0 = no usable box (runs shorter than 8 tokens = 512 bytes, the 64-byte-swizzle repeat).
static int attn_tma_box_tokens(const GrlGrid& g) {
  int d = g.ww;
  if (g.sw > 0) {
    int x = g.ww, y = g.sw;
    while (y) {
      const int t = x % y;
      x = y, y = t;
    }
    d = x;
  }
  int bw = 64;
  while (bw > 1 && d % bw) bw >>= 1;
  return bw >= 8 ? bw : 0;
}

// (B * H * W tokens, ld) 16-bit tensor map with {32 channels, box tokens} boxes; false: no usable map (box 0 then)
static bool token_map(CUtensorMap* m, const void* base, long long ld, long long tokens, int box, int fmt) {
  EncodeTiledFn fn = encode_tiled_fn();
  if (!fn || box <= 0 || (reinterpret_cast<uintptr_t>(base) & 15) || (ld * 2) % 16) return false;
  const cuuint64_t dims[2] = {(cuuint64_t)ld, (cuuint64_t)tokens};
  const cuuint64_t str[1] = {(cuuint64_t)ld * 2};
  const cuuint32_t boxd[2] = {(cuuint32_t)kDP, (cuuint32_t)box};
  const cuuint32_t ones[2] = {1, 1};
  return fn(m, fmt == FMT_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base),
            dims, str, boxd, ones, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace tc
}  // namespace grl

using namespace grl;
using namespace grl::tc;

extern "C" {

int grl_tc_attn_box_tokens(GrlGrid g) {
  if (check_grid(g, "attn_box_tokens") != GRL_OK) return 0;
  return attn_tma_box_tokens(g);
}

int grl_tc_attn_variant(int set) {
  static int variant = -1;
  if (variant < 0) {
    // default 5: TMA boxes wherever the geometry has them; GRL_ATTN_SPLIT=0 gathers every operand row by row
    const char* e = getenv("GRL_ATTN_SPLIT");
    variant = (e && atoi(e) == 0) ? 0 : 5;
  }
  const int prev = variant;
  if (set == 0 || set == 5) variant = set;
  return prev;
}

int grl_tc_attn(const GrlTcAttn* p, void* stream) {
  GRL_REQUIRE(p != nullptr, "tc_attn: null problem");
  if (!grl_device_ok()) return fail(GRL_ERR_ARCH, "tc_attn: wgmma kernels need an sm_90 device");
  const GrlTcAttn& a = *p;
  if (check_fmt(a.fmt)) return GRL_ERR_INVALID;
  GRL_REQUIRE((a.ldq % 8) == 0 && (a.ldk % 8) == 0 && (a.v_dense || (a.ldv % 8) == 0) &&
                  (a.o_dense || (a.ldo % 8) == 0) && (a.q_off % 8) == 0 && (a.k_off % 8) == 0 &&
                  (a.v_off % 8) == 0 && (a.o_off % 8) == 0,
              "tc_attn: pitches and offsets must be multiples of 8 elements (16 bytes)");
  GRL_REQUIRE(a.rows == (a.gq.wh + a.gk.wh - 1) * (a.gq.ww + a.gk.ww - 1), "tc_attn: bias table has %d rows, expected %d",
              a.rows, (a.gq.wh + a.gk.wh - 1) * (a.gq.ww + a.gk.ww - 1));
  const cudaStream_t st = (cudaStream_t)stream;
  if (a.B == 0) return GRL_OK;
  int rc;
  if ((rc = check_grid(a.gq, "attn_tc(q grid)")) != GRL_OK) return rc;
  if ((rc = check_grid(a.gk, "attn_tc(k grid)")) != GRL_OK) return rc;
  GRL_REQUIRE(a.gq.H / a.gq.wh == a.gk.H / a.gk.wh && a.gq.W / a.gq.ww == a.gk.W / a.gk.ww,
              "attn_tc: query and key grids have different window counts");
  GRL_REQUIRE(a.heads >= 1 && a.heads <= 8, "attn_tc: heads=%d unsupported", a.heads);
  GRL_REQUIRE(a.rows_pad % 4 == 0 && a.rows_pad >= a.rows + 4, "attn_tc: bias table pitch %d too small for %d rows", a.rows_pad,
              a.rows);
  const int Nq = a.gq.wh * a.gq.ww;
  const long long nblk = (long long)a.B * (a.gq.H / a.gq.wh) * (a.gq.W / a.gq.ww) * a.heads * ceil_div(Nq, kQT);
  GRL_REQUIRE(nblk < (1ll << 31), "attn_tc: grid too large");
  AttnMaps tm;
  memset(&tm, 0, sizeof(tm));
  if (grl_tc_attn_variant(-1) == 5) {
    const long long nq = (long long)a.B * a.gq.H * a.gq.W, nk = (long long)a.B * a.gk.H * a.gk.W;
    tm.box_q = attn_tma_box_tokens(a.gq);
    tm.box_k = attn_tma_box_tokens(a.gk);
    if (!token_map(&tm.q, a.q, a.ldq, nq, tm.box_q, a.fmt)) tm.box_q = 0;
    if (!token_map(&tm.k, a.k, a.ldk, nk, tm.box_k, a.fmt) ||
        (!a.v_dense && !token_map(&tm.v, a.v, a.ldv, nk, tm.box_k, a.fmt)))
      tm.box_k = 0;
  }
  // 64 keys per tile: one m64n64 S fragment per warpgroup, 2 CTAs / SM
  switch (a.gk.ww) {
    case 8: return launch_attn_one<64, 8>(tm, a, (unsigned)nblk, st);
    case 16: return launch_attn_one<64, 16>(tm, a, (unsigned)nblk, st);
    case 32: return launch_attn_one<64, 32>(tm, a, (unsigned)nblk, st);
    case 64: return launch_attn_one<64, 64>(tm, a, (unsigned)nblk, st);
    case 128: return launch_attn_one<64, 128>(tm, a, (unsigned)nblk, st);
    default: return launch_attn_one<64, 0>(tm, a, (unsigned)nblk, st);
  }
}

}  // extern "C"
