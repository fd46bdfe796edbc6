// ops_f32.cu -- the fp32 exact-parity path: every operator of one GRL block as a hand-written CUDA
// kernel with fp32 storage, fp32 FMA accumulation and accurate (non-approx) transcendentals.
// This path is what the <= 1e-3 max-abs gate of BASELINE.json is checked on; the bf16 wgmma path
// (gemm_tc.cu / attn_tc.cu) is the throughput path and is gated on PSNR.
//
// Reference semantics cited per kernel (paths relative to the reference root).
#include <string.h>

#include "grl_common.cuh"

namespace grl {

struct GemmArgs {
  const float* x;
  long long ldx;
  const float* w;  // (N, K) row-major
  const float* b;
  const float* res;
  long long ldr;
  float* y;
  long long ldy;
  long long M;
  int N, K;
  int act;
  float slope;
  int H, W, Cin;  // conv only
};

struct AttnArgs {
  GrlGrid gq, gk;  // query / key token grids (same number of windows)
  const float* q;
  long long ldq;
  int q_off;  // channel offset of head 0 in a token row
  const float* k;
  long long ldk;
  int k_off;
  const float* v;
  long long ldv;
  int v_off;
  int v_dense;  // V is the dense (B_, heads, Nk, d) X1 buffer
  float* out;
  long long ldo;
  int o_off;
  int o_dense;  // write dense (B_, heads, Nq, d)
  int B, heads, d;
  const float* logit_scale;  // (heads)
  const float* bias;         // (heads, rows)
  int rows;
  int use_mask;
};

// =====================================================================================
// bias table: out[h, r] = 16 * sigmoid( W2[h,:] . relu(W1 t_r + b1) )
// (AffineTransform.forward mixed_attn_block_efficient.py:41-47; CPB_MLP mixed_attn_block.py:24-31).
// sigmoid and the index gather commute, so the table is activated once per block instead of once per
// score element.
// =====================================================================================
constexpr int kMaxHeads = 8;

__global__ void bias_table_kernel(const float* __restrict__ table, int rows, const float* __restrict__ w1,
                                  const float* __restrict__ b1, const float* __restrict__ w2, int hidden, int heads,
                                  float mul, int copies, int rows_pad, float* __restrict__ out) {
  extern __shared__ float sm[];  // w1 (hidden*2) | b1 (hidden) | w2 (heads*hidden)
  float* s_w1 = sm;
  float* s_b1 = sm + 2 * hidden;
  float* s_w2 = s_b1 + hidden;
  for (int i = threadIdx.x; i < 2 * hidden; i += blockDim.x) s_w1[i] = w1[i];
  for (int i = threadIdx.x; i < hidden; i += blockDim.x) s_b1[i] = b1[i];
  for (int i = threadIdx.x; i < heads * hidden; i += blockDim.x) s_w2[i] = w2[i];
  __syncthreads();
  int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  float t0 = table[2 * r], t1 = table[2 * r + 1];
  float acc[kMaxHeads];
#pragma unroll
  for (int h = 0; h < kMaxHeads; ++h) acc[h] = 0.f;
  for (int k = 0; k < hidden; ++k) {
    float hk = fmaf(s_w1[2 * k + 1], t1, fmaf(s_w1[2 * k], t0, s_b1[k]));
    hk = fmaxf(hk, 0.f);
#pragma unroll
    for (int h = 0; h < kMaxHeads; ++h)
      if (h < heads) acc[h] = fmaf(s_w2[h * hidden + k], hk, acc[h]);
  }
#pragma unroll
  for (int h = 0; h < kMaxHeads; ++h)
    if (h < heads) {
      const float val = (16.f / (1.f + expf(-acc[h]))) * mul;
      for (int c = 0; c < copies; ++c) out[((size_t)h * copies + c) * rows_pad + r + c] = val;  // copy c: shifted by c
    }
}

// =====================================================================================
// AffineTransform.forward on a materialised attention map (API-compat operator; the fused attention
// kernels never materialise the map).  mixed_attn_block_efficient.py:36-58.
// =====================================================================================
__global__ void affine_kernel(float* __restrict__ attn, long long total, int heads, int n1, int n2,
                              const float* __restrict__ logit_scale, const float* __restrict__ bias, int rows,
                              const long long* __restrict__ index, const float* __restrict__ mask, int nW) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  long long per = (long long)n1 * n2;
  long long ij = i % per;
  long long bh = i / per;
  int h = (int)(bh % heads);
  long long b_ = bh / heads;
  float scale = expf(fminf(logit_scale[h], 4.605170185988092f));
  float v = attn[i] * scale + bias[(size_t)h * rows + index[ij]];
  if (mask) v += mask[(b_ % nW) * per + ij];
  attn[i] = v;
}

// =====================================================================================
// Tiled fp32 GEMM  y = act(A w^T + b) (+ res), with A either a plain row-major matrix (nn.Linear) or
// the on-the-fly im2col view of a channels-last image (3x3 conv, pad 1):
//   A[m, tap*Cin + c] = x[b, y+ky, x+kx, c]   (zero outside the image)
// 64x64x16 tiles, 256 threads, 4x4 outputs per thread.
// =====================================================================================

constexpr int BM = 64, BN = 64, BK = 16;

template <bool CONV>
__global__ void __launch_bounds__(256) gemm_f32_kernel(GemmArgs a) {
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const long long m0 = (long long)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;
  const int lk = tid & 15;   // k inside the tile handled by this thread when loading
  const int lr = tid >> 4;   // row (0..15), + 16*p

  // conv: per-row pixel coordinates of the 4 rows this thread loads
  int py[4], px[4];
  long long pb[4];
  if (CONV) {
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      long long m = m0 + lr + 16 * p;
      long long hw = (long long)a.H * a.W;
      long long bb = m / hw;
      int rem = (int)(m - bb * hw);
      py[p] = rem / a.W;
      px[p] = rem - py[p] * a.W;
      pb[p] = bb;
    }
  }

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < a.K; k0 += BK) {
    const int k = k0 + lk;
    int tap = 0, c = 0, ky = 0, kx = 0;
    if (CONV) {
      tap = k / a.Cin;
      c = k - tap * a.Cin;
      ky = tap / 3 - 1;
      kx = tap - (tap / 3) * 3 - 1;
    }
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const int r = lr + 16 * p;
      const long long m = m0 + r;
      float v = 0.f;
      if (m < a.M && k < a.K) {
        if (CONV) {
          int yy = py[p] + ky, xx = px[p] + kx;
          if (yy >= 0 && yy < a.H && xx >= 0 && xx < a.W)
            v = __ldg(a.x + ((pb[p] * a.H + yy) * a.W + xx) * a.Cin + c);
        } else {
          v = __ldg(a.x + m * a.ldx + k);
        }
      }
      As[lk][r] = v;
      const int n = n0 + r;
      Bs[lk][r] = (n < a.N && k < a.K) ? __ldg(a.w + (long long)n * a.K + k) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      const float4 av = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
      const float4 bv = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
      const float ar[4] = {av.x, av.y, av.z, av.w};
      const float br[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ar[i], br[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const long long m = m0 + ty * 4 + i;
    if (m >= a.M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= a.N) continue;
      float v = acc[i][j] + (a.b ? a.b[n] : 0.f);
      v = apply_act(v, a.act, a.slope);
      if (a.res) v += a.res[m * a.ldr + n];
      a.y[m * a.ldy + n] = v;
    }
  }
}

// =====================================================================================
// AvgPool2d(df) / MaxPool2d(df) on channels-last data (AnchorLinear, mixed_attn_block.py:723-726,:733).
// =====================================================================================
template <bool MAX>
__global__ void pool_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int H, int W, int C, int df) {
  const int Ho = H / df, Wo = W / df;
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long total = (long long)B * Ho * Wo * C;
  if (i >= total) return;
  int c = (int)(i % C);
  long long t = i / C;
  int xo = (int)(t % Wo);
  t /= Wo;
  int yo = (int)(t % Ho);
  int b = (int)(t / Ho);
  float s = MAX ? -INFINITY : 0.f;
  for (int dy = 0; dy < df; ++dy)
    for (int dx = 0; dx < df; ++dx) {
      const float v = x[(((long long)b * H + yo * df + dy) * W + xo * df + dx) * C + c];
      if (MAX)
        s = (v > s || v != v) ? v : s;  // a NaN propagates, as in torch's max_pool2d
      else
        s += v;
    }
  y[i] = MAX ? s : s / (float)(df * df);
}

// =====================================================================================
// out = x + res_scale * LN(u) (+ cab_y * gate[b])     one warp per token row
// (mixed_attn_block_efficient.py:543-554; LayerNorm eps 1e-5, biased variance).
// =====================================================================================
__global__ void ln_residual_kernel(const float* __restrict__ x, const float* __restrict__ u,
                                   const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                   float res_scale, const float* __restrict__ cab_y,
                                   const float* __restrict__ cab_gate, long long L, float* __restrict__ out,
                                   long long M, int C) {
  const int warps = blockDim.x >> 5;
  long long m = (long long)blockIdx.x * warps + (threadIdx.x >> 5);
  if (m >= M) return;
  const int lane = threadIdx.x & 31;
  const float* ur = u + m * C;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += ur[c];
  const float mean = warp_sum(s) / (float)C;
  float v = 0.f;
  for (int c = lane; c < C; c += 32) {
    float d = ur[c] - mean;
    v = fmaf(d, d, v);
  }
  const float rstd = 1.0f / sqrtf(warp_sum(v) / (float)C + eps);
  const long long b = m / L;
  for (int c = lane; c < C; c += 32) {
    float r = ((ur[c] - mean) * rstd * gamma[c] + beta[c]) * res_scale;
    if (x) r += x[m * C + c];
    if (cab_y) r += cab_y[m * C + c] * cab_gate[b * C + c];
    out[m * C + c] = r;
  }
}

// =====================================================================================
// ChannelAttention (mixed_attn_block.py:948-967): deterministic two-stage mean over L, then the
// squeeze/excite MLP.  partial: (B, chunks, C)
// =====================================================================================
constexpr int kPoolRows = 256;

__global__ void channel_partial_kernel(const float* __restrict__ y, long long L, int C, float* __restrict__ partial,
                                       int chunks) {
  const int b = blockIdx.y, ch = blockIdx.x;
  const long long r0 = (long long)ch * kPoolRows;
  const long long r1 = min(L, r0 + kPoolRows);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float s = 0.f;
    for (long long r = r0; r < r1; ++r) s += y[((long long)b * L + r) * C + c];
    partial[((long long)b * chunks + ch) * C + c] = s;
  }
}

__global__ void channel_gate_kernel(const float* __restrict__ partial, int chunks, long long L, int C,
                                    const float* __restrict__ w1, const float* __restrict__ b1,
                                    const float* __restrict__ w2, const float* __restrict__ b2, int R,
                                    float* __restrict__ gate) {
  extern __shared__ float sm[];  // mean[C] | hid[R]
  float* s_mean = sm;
  float* s_hid = sm + C;
  const int b = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float s = 0.f;
    for (int k = 0; k < chunks; ++k) s += partial[((long long)b * chunks + k) * C + c];
    s_mean[c] = s / (float)L;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int r = warp; r < R; r += nw) {
    float s = 0.f;
    for (int c = lane; c < C; c += 32) s = fmaf(w1[(long long)r * C + c], s_mean[c], s);
    s = warp_sum(s);
    if (lane == 0) s_hid[r] = fmaxf(s + b1[r], 0.f);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float s = b2[c];
    for (int r = 0; r < R; ++r) s = fmaf(w2[(long long)c * R + r], s_hid[r], s);
    gate[(long long)b * C + c] = 1.f / (1.f + expf(-s));
  }
}

// =====================================================================================
// Fused cosine attention (fp32, flash-style, one query row per thread).
//   Attention.attn + AffineTransform: mixed_attn_block_efficient.py:36-58,:77-94
//   roll/partition/merge addressing: :139-163 (window), :234-267 (stripe); ops.py:36-73
// One kernel serves the three uses:
//   window:        Q,K,V = window tokens                          -> token grid
//   stripe pass 1: Q = anchors, K,V = stripe tokens               -> dense X1 (B_, heads, N2, d)
//   stripe pass 2: Q = stripe tokens, K = anchors, V = dense X1   -> token grid
// =====================================================================================

constexpr int kQT = 128;  // queries per CTA (one per thread)
constexpr int kKT = 32;   // keys per smem tile

template <int D>
__global__ void __launch_bounds__(kQT) attn_f32_kernel(AttnArgs a) {
  __shared__ float ks[kKT][D];
  __shared__ float vs[kKT][D];
  __shared__ int k_ih[kKT], k_iw[kKT], k_rid[kKT];

  const int Nq = a.gq.wh * a.gq.ww, Nk = a.gk.wh * a.gk.ww;
  const int nqt = (Nq + kQT - 1) / kQT;
  const int nww = a.gq.W / a.gq.ww;  // windows per row (same for both grids)
  const int nW = (a.gq.H / a.gq.wh) * nww;
  int bid = blockIdx.x;
  const int qt = bid % nqt;
  bid /= nqt;
  const int h = bid % a.heads;
  const int bw = bid / a.heads;
  const int b = bw / nW, w = bw - b * nW;
  const int wr = w / nww, wc = w - wr * nww;
  const int d = a.d;
  const int tid = threadIdx.x;

  // ---- this thread's query row
  const int qi = qt * kQT + tid;
  const bool q_ok = qi < Nq;
  float q[D], o[D];
  Tok tq = locate(a.gq, wr, wc, q_ok ? qi : 0);
  const int q_rid = region_id(a.gq, tq.r, tq.c);
  {
    const float* qp = a.q + ((long long)(b * a.gq.H + tq.y) * a.gq.W + tq.x) * a.ldq + a.q_off + h * d;
    float ss = 0.f;
#pragma unroll
    for (int e = 0; e < D; ++e) {
      q[e] = (e < d) ? qp[e] : 0.f;
      ss = fmaf(q[e], q[e], ss);
      o[e] = 0.f;
    }
    const float inv = 1.0f / fmaxf(sqrtf(ss), 1e-12f);  // F.normalize eps
#pragma unroll
    for (int e = 0; e < D; ++e) q[e] *= inv;
  }
  const float scale = expf(fminf(a.logit_scale[h], 4.605170185988092f));  // clamp(max=ln 100).exp()
  const float* bias = a.bias + (size_t)h * a.rows;
  float m_run = -INFINITY, l_run = 0.f;

  for (int k0 = 0; k0 < Nk; k0 += kKT) {
    __syncthreads();  // previous tile fully consumed
    // ---- stage K / V tile
    for (int idx = tid; idx < kKT * D; idx += kQT) {
      const int j = idx / D, e = idx - j * D;
      const int kj = k0 + j;
      float kv = 0.f, vv = 0.f;
      if (kj < Nk && e < d) {
        Tok tk = locate(a.gk, wr, wc, kj);
        const long long tok = (long long)(b * a.gk.H + tk.y) * a.gk.W + tk.x;
        kv = a.k[tok * a.ldk + a.k_off + h * d + e];
        vv = a.v_dense ? a.v[(((long long)bw * a.heads + h) * Nk + kj) * d + e]
                       : a.v[tok * a.ldv + a.v_off + h * d + e];
      }
      ks[j][e] = kv;
      vs[j][e] = vv;
    }
    if (tid < kKT) {
      const int kj = k0 + tid;
      Tok tk = locate(a.gk, wr, wc, kj < Nk ? kj : 0);
      k_ih[tid] = tk.ih;
      k_iw[tid] = tk.iw;
      k_rid[tid] = region_id(a.gk, tk.r, tk.c);
    }
    __syncthreads();
    if (tid < kKT) {  // F.normalize(k)
      float ss = 0.f;
#pragma unroll
      for (int e = 0; e < D; ++e) ss = fmaf(ks[tid][e], ks[tid][e], ss);
      const float inv = 1.0f / fmaxf(sqrtf(ss), 1e-12f);
#pragma unroll
      for (int e = 0; e < D; ++e) ks[tid][e] *= inv;
    }
    __syncthreads();

    // ---- logits of this tile
    float lg[kKT];
    float m_tile = -INFINITY;
#pragma unroll
    for (int j = 0; j < kKT; ++j) {
      float s = 0.f;
#pragma unroll
      for (int e = 0; e < D; ++e) s = fmaf(q[e], ks[j][e], s);
      const int ridx = rel_index(tq.ih, tq.iw, k_ih[j], k_iw[j], a.gq.ww, a.gk.wh, a.gk.ww);
      float v = s * scale + __ldg(bias + ridx);
      if (a.use_mask && q_rid != k_rid[j]) v += -100.0f;
      if (k0 + j >= Nk) v = -INFINITY;
      lg[j] = v;
      m_tile = fmaxf(m_tile, v);
    }
    const float m_new = fmaxf(m_run, m_tile);
    const float corr = expf(m_run - m_new);  // exp(-inf) = 0 on the first tile
    l_run *= corr;
#pragma unroll
    for (int e = 0; e < D; ++e) o[e] *= corr;
#pragma unroll
    for (int j = 0; j < kKT; ++j) {
      const float p = expf(lg[j] - m_new);
      l_run += p;
#pragma unroll
      for (int e = 0; e < D; ++e) o[e] = fmaf(p, vs[j][e], o[e]);
    }
    m_run = m_new;
  }

  if (!q_ok) return;
  const float inv_l = 1.0f / l_run;
  float* op = a.o_dense ? a.out + (((long long)bw * a.heads + h) * Nq + qi) * d
                        : a.out + ((long long)(b * a.gq.H + tq.y) * a.gq.W + tq.x) * a.ldo + a.o_off + h * d;
#pragma unroll
  for (int e = 0; e < D; ++e)
    if (e < d) op[e] = o[e] * inv_l;
}

// -------------------------------------------------------------------------------------
// host side
// -------------------------------------------------------------------------------------
static int launch_bias_table(const float* table, int rows, const float* w1, const float* b1, const float* w2, int hidden,
                             int heads, float mul, int copies, int rows_pad, float* out, cudaStream_t st) {
  GRL_REQUIRE(copies >= 1 && copies <= 4 && rows_pad >= rows + copies - 1, "bias_table: bad copies / pitch");
  GRL_REQUIRE(heads >= 1 && heads <= kMaxHeads, "bias_table: heads=%d unsupported (max %d)", heads, kMaxHeads);
  GRL_REQUIRE(rows > 0 && hidden > 0, "bias_table: empty");
  size_t smem = sizeof(float) * (size_t)(3 + heads) * hidden;
  GRL_REQUIRE(smem <= 48 * 1024, "bias_table: hidden=%d too large", hidden);
  bias_table_kernel<<<ceil_div(rows, 128), 128, smem, st>>>(table, rows, w1, b1, w2, hidden, heads, mul, copies, rows_pad, out);
  GRL_LAUNCH_CHECK("bias_table_kernel");
  return GRL_OK;
}

static int launch_gemm(const GemmArgs& a, bool conv, cudaStream_t st) {
  if (a.M == 0 || a.N == 0) return GRL_OK;
  GRL_REQUIRE(a.K > 0, "gemm: K must be positive");
  dim3 grid(ceil_div(a.M, BM), ceil_div(a.N, BN));
  GRL_REQUIRE(grid.y <= 65535, "gemm: N too large");
  if (conv)
    gemm_f32_kernel<true><<<grid, 256, 0, st>>>(a);
  else
    gemm_f32_kernel<false><<<grid, 256, 0, st>>>(a);
  GRL_LAUNCH_CHECK("gemm_f32_kernel");
  return GRL_OK;
}

int channel_gate_from_partial(const float* partial, int chunks, int B, long long L, int C, const float* w1, const float* b1,
                              const float* w2, const float* b2, int R, float* gate, cudaStream_t st) {
  if (B == 0) return GRL_OK;
  channel_gate_kernel<<<B, 256, sizeof(float) * (C + R), st>>>(partial, chunks, L, C, w1, b1, w2, b2, R, gate);
  GRL_LAUNCH_CHECK("channel_gate_kernel");
  return GRL_OK;
}

// the window attention and both passes of the stripe attention
static int launch_attn(const AttnArgs& a, cudaStream_t st) {
  if (a.B == 0) return GRL_OK;
  int rc;
  if ((rc = check_grid(a.gq, "attn(q grid)")) != GRL_OK) return rc;
  if ((rc = check_grid(a.gk, "attn(k grid)")) != GRL_OK) return rc;
  GRL_REQUIRE(a.gq.H / a.gq.wh == a.gk.H / a.gk.wh && a.gq.W / a.gq.ww == a.gk.W / a.gk.ww,
              "attn: query and key grids have different window counts");
  GRL_REQUIRE(a.d >= 1 && a.d <= 64, "attn: head_dim %d unsupported (1..64)", a.d);
  GRL_REQUIRE(a.heads >= 1 && a.heads <= kMaxHeads, "attn: heads=%d unsupported", a.heads);
  const int Nq = a.gq.wh * a.gq.ww;
  const long long nblk = (long long)a.B * windows_per_image(a.gq) * a.heads * ceil_div(Nq, kQT);
  GRL_REQUIRE(nblk < (1ll << 31), "attn: grid too large");
  if (a.d <= 16)
    attn_f32_kernel<16><<<(unsigned)nblk, kQT, 0, st>>>(a);
  else if (a.d <= 32)
    attn_f32_kernel<32><<<(unsigned)nblk, kQT, 0, st>>>(a);
  else
    attn_f32_kernel<64><<<(unsigned)nblk, kQT, 0, st>>>(a);
  GRL_LAUNCH_CHECK("attn_f32_kernel");
  return GRL_OK;
}

}  // namespace grl

using namespace grl;

extern "C" {

int grl_bias_table_f32(const float* table, int rows, const float* w1, const float* b1, const float* w2, int hidden,
                       int heads, float* out, void* stream) {
  return launch_bias_table(table, rows, w1, b1, w2, hidden, heads, 1.0f, 1, rows, out, (cudaStream_t)stream);
}

int grl_tc_bias_table4(const float* table, int rows, const float* w1, const float* b1, const float* w2, int hidden,
                       int heads, float mul, int rows_pad, float* out, void* stream) {
  GRL_REQUIRE(rows_pad % 4 == 0 && rows_pad >= rows + 4, "tc_bias_table4: rows_pad must be a multiple of 4 and >= rows + 4");
  return launch_bias_table(table, rows, w1, b1, w2, hidden, heads, mul, 4, rows_pad, out, (cudaStream_t)stream);
}

int grl_affine_f32(float* attn, int64_t B_, int heads, int n1, int n2, const float* logit_scale, const float* bias,
                   int rows, const int64_t* index, const float* mask, int nW, void* stream) {
  long long total = B_ * heads * n1 * n2;
  if (total == 0) return GRL_OK;
  GRL_REQUIRE(!mask || (nW > 0 && B_ % nW == 0), "affine: batch %lld not a multiple of nW=%d", (long long)B_, nW);
  affine_kernel<<<ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(attn, total, heads, n1, n2, logit_scale, bias, rows,
                                                                       (const long long*)index, mask, nW > 0 ? nW : 1);
  GRL_LAUNCH_CHECK("affine_kernel");
  return GRL_OK;
}

int grl_linear_f32(const float* x, int64_t ldx, const float* w, const float* b, const float* res, int64_t ldr,
                   float* y, int64_t ldy, int64_t M, int N, int K, int act, float slope, void* stream) {
  GRL_REQUIRE(M >= 0 && N >= 0 && K > 0 && ldx >= K && ldy >= N, "linear: bad shape M=%lld N=%d K=%d", (long long)M, N,
              K);
  GemmArgs a = {x, ldx, w, b, res, ldr, y, ldy, M, N, K, act, slope, 0, 0, 0};
  return launch_gemm(a, false, (cudaStream_t)stream);
}

int grl_conv3x3_f32(const float* x, const float* w, const float* b, const float* res, float* y, int B, int H, int W,
                    int Cin, int Cout, int act, float slope, void* stream) {
  GRL_REQUIRE(B >= 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0, "conv3x3: bad shape");
  GemmArgs a = {x, 0, w, b, res, Cout, y, Cout, (long long)B * H * W, Cout, 9 * Cin, act, slope, H, W, Cin};
  return launch_gemm(a, true, (cudaStream_t)stream);
}

static int launch_pool(const float* x, float* y, int B, int H, int W, int C, int df, bool max, cudaStream_t st) {
  GRL_REQUIRE(df >= 1 && H % df == 0 && W % df == 0, "pool: %dx%d not divisible by %d", H, W, df);
  long long total = (long long)B * (H / df) * (W / df) * C;
  if (total == 0) return GRL_OK;
  if (max)
    pool_kernel<true><<<ceil_div(total, 256), 256, 0, st>>>(x, y, B, H, W, C, df);
  else
    pool_kernel<false><<<ceil_div(total, 256), 256, 0, st>>>(x, y, B, H, W, C, df);
  GRL_LAUNCH_CHECK("pool_kernel");
  return GRL_OK;
}

int grl_avgpool_f32(const float* x, float* y, int B, int H, int W, int C, int df, void* stream) {
  return launch_pool(x, y, B, H, W, C, df, false, (cudaStream_t)stream);
}

int grl_maxpool_f32(const float* x, float* y, int B, int H, int W, int C, int df, void* stream) {
  return launch_pool(x, y, B, H, W, C, df, true, (cudaStream_t)stream);
}

int grl_ln_residual_f32(const float* x, const float* u, const float* gamma, const float* beta, float eps,
                        float res_scale, const float* cab_y, const float* cab_gate, int64_t L, float* out, int64_t M,
                        int C, void* stream) {
  if (M == 0) return GRL_OK;
  GRL_REQUIRE((cab_y == nullptr) == (cab_gate == nullptr), "ln_residual: cab_y and cab_gate go together");
  GRL_REQUIRE(L > 0 && M % L == 0, "ln_residual: M=%lld not a multiple of L=%lld", (long long)M, (long long)L);
  ln_residual_kernel<<<ceil_div(M, 8), 256, 0, (cudaStream_t)stream>>>(x, u, gamma, beta, eps, res_scale, cab_y, cab_gate, L,
                                                                      out, M, C);
  GRL_LAUNCH_CHECK("ln_residual_kernel");
  return GRL_OK;
}

size_t grl_channel_gate_workspace(int B, int64_t L, int C) {
  return sizeof(float) * (size_t)B * ceil_div(L, kPoolRows) * C;
}

int grl_channel_gate_f32(const float* y, int B, int64_t L, int C, const float* w1, const float* b1, const float* w2,
                         const float* b2, int R, float* gate, void* workspace, size_t workspace_bytes, void* stream) {
  if (B == 0) return GRL_OK;
  GRL_REQUIRE(L > 0 && C > 0 && R > 0, "channel_gate: empty");
  const size_t need = grl_channel_gate_workspace(B, L, C);
  if (workspace_bytes < need) return fail(GRL_ERR_WORKSPACE, "channel_gate: workspace %zu < %zu", workspace_bytes, need);
  const cudaStream_t st = (cudaStream_t)stream;
  const int chunks = ceil_div(L, kPoolRows);
  channel_partial_kernel<<<dim3(chunks, B), 256, 0, st>>>(y, L, C, (float*)workspace, chunks);
  GRL_LAUNCH_CHECK("channel_partial_kernel");
  channel_gate_kernel<<<B, 256, sizeof(float) * (C + R), st>>>((const float*)workspace, chunks, L, C, w1, b1, w2, b2, R, gate);
  GRL_LAUNCH_CHECK("channel_gate_kernel");
  return GRL_OK;
}

int grl_window_attn_f32(const float* qkv, int64_t ld_qkv, float* out, int64_t ld_out, int B, GrlGrid grid, int heads,
                        int d, const float* logit_scale, const float* bias, int use_mask, void* stream) {
  AttnArgs a;
  memset(&a, 0, sizeof(a));
  const int c = heads * d;
  a.gq = grid;
  a.gk = grid;
  a.q = qkv, a.ldq = ld_qkv, a.q_off = 0;
  a.k = qkv, a.ldk = ld_qkv, a.k_off = c;
  a.v = qkv, a.ldv = ld_qkv, a.v_off = 2 * c;
  a.out = out, a.ldo = ld_out, a.o_off = 0;
  a.B = B, a.heads = heads, a.d = d;
  a.logit_scale = logit_scale;
  a.bias = bias;
  a.rows = (2 * grid.wh - 1) * (2 * grid.ww - 1);
  a.use_mask = use_mask;
  return launch_attn(a, (cudaStream_t)stream);
}

size_t grl_stripe_attn_workspace(int B, GrlGrid tok, GrlGrid anc, int heads, int d) {
  (void)tok;
  return sizeof(float) * (size_t)B * anc.H * anc.W * heads * d;
}

int grl_stripe_attn_f32(const float* qkv, int64_t ld_qkv, const float* anchor, int64_t ld_anchor, float* out,
                        int64_t ld_out, int B, GrlGrid tok, GrlGrid anc, int heads, int d, const float* logit_scale1,
                        const float* bias1, const float* logit_scale2, const float* bias2, int use_mask,
                        void* workspace, size_t workspace_bytes, void* stream) {
  const size_t need = grl_stripe_attn_workspace(B, tok, anc, heads, d);
  if (workspace_bytes < need) return fail(GRL_ERR_WORKSPACE, "stripe_attn: workspace %zu < %zu", workspace_bytes, need);
  const int c = heads * d;
  const int rows = (tok.wh + anc.wh - 1) * (tok.ww + anc.ww - 1);
  float* x1 = (float*)workspace;
  AttnArgs a;
  memset(&a, 0, sizeof(a));
  // pass 1: anchors attend to the stripe's tokens (a2w)   efficient.py:256-258
  a.gq = anc, a.gk = tok;
  a.q = anchor, a.ldq = ld_anchor, a.q_off = 0;
  a.k = qkv, a.ldk = ld_qkv, a.k_off = c;
  a.v = qkv, a.ldv = ld_qkv, a.v_off = 2 * c;
  a.out = x1, a.o_dense = 1;
  a.B = B, a.heads = heads, a.d = d;
  a.logit_scale = logit_scale1, a.bias = bias1, a.rows = rows, a.use_mask = use_mask;
  int rc = launch_attn(a, (cudaStream_t)stream);
  if (rc != GRL_OK) return rc;
  // pass 2: tokens attend to the anchors, values = X1 (w2a)   efficient.py:259
  memset(&a, 0, sizeof(a));
  a.gq = tok, a.gk = anc;
  a.q = qkv, a.ldq = ld_qkv, a.q_off = 0;
  a.k = anchor, a.ldk = ld_anchor, a.k_off = 0;
  a.v = x1, a.v_dense = 1;
  a.out = out, a.ldo = ld_out, a.o_off = 0;
  a.B = B, a.heads = heads, a.d = d;
  a.logit_scale = logit_scale2, a.bias = bias2, a.rows = rows, a.use_mask = use_mask;
  return launch_attn(a, (cudaStream_t)stream);
}

}  // extern "C"
