/* grl_b200.h -- C ABI of libgrl_b200.so: the H100 (sm_90a) implementation of GRL's forward hot path.
 *
 * The reference (ofsoundof/GRL-Image-Restoration) is pure Python/ATen: it has no FFI, plugin or
 * operator registry for this path.  Its boundary is the nn.Module contract (SURVEY.md section 8b);
 * every entry point below therefore cites the reference *Python interface* it replaces
 * (paths relative to the reference root) and INTEGRATION.md shows the ctypes binding a maintainer
 * adds.  Conventions for every function:
 *   - plain pointers + sizes only; all data pointers are DEVICE pointers unless the name ends in
 *     _host; `stream` is a cudaStream_t passed as void*;
 *   - no allocation, no synchronisation; re-entrant per stream.  Process-wide state is limited to: the
 *     per-thread error string, an atomic launch counter (grl_launch_count), the attention operand-load
 *     selector (grl_tc_attn_variant, initialised from GRL_ATTN_SPLIT) and the per-device "shared-memory
 *     attribute set" flags.  None of it depends on the data of a call;
 *   - returns 0 on success, a negative GrlStatus otherwise; grl_last_error() gives the message
 *     (the Python wrappers raise RuntimeError -- same behaviour as a failing ATen call).
 * Activations are channels-last: a (B, L, C) token tensor is the same memory as (B, H, W, C).
 */
#ifndef GRL_B200_H_
#define GRL_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GRL_B200_ABI_VERSION 6

typedef enum {
  GRL_OK = 0,
  GRL_ERR_INVALID = -1,   /* bad argument / unsupported shape */
  GRL_ERR_CUDA = -2,      /* a CUDA runtime/driver call failed */
  GRL_ERR_WORKSPACE = -3, /* workspace too small */
  GRL_ERR_ARCH = -4       /* device is not sm_90 */
} GrlStatus;

typedef enum { GRL_ACT_NONE = 0, GRL_ACT_GELU = 1, GRL_ACT_LEAKY = 2 } GrlAct;

/* One attention "level": a (H x W) token grid cut into (wh x ww) windows/stripes after a cyclic
 * roll by (-sh, -sw)  [torch.roll + window_partition: mixed_attn_block_efficient.py:139-147,
 * :234-247; models/common/ops.py:36-54]. */
typedef struct {
  int32_t H, W;   /* grid size (tokens, or anchors = tokens / df) */
  int32_t wh, ww; /* window / stripe size on this grid */
  int32_t sh, sw; /* cyclic shift on this grid (0 = none) */
} GrlGrid;

const char* grl_last_error(void);
int grl_abi_version(void);
/* number of kernels this library has launched since it was loaded (bench.py's gpu_launches) */
uint64_t grl_launch_count(void);
/* 1 if the current device is compute capability 9.x */
int grl_device_ok(void);

/* ---- geometry, host side (bit-exact restatement of models/common/ops.py; used by tests and by the
 * Python surface to honour the reference's table/index/mask arguments) ------------------------- */
/* get_relative_position_index_simple (ops.py:352-375): out is (n1, n2) int64, row-major.
 * window_to_anchor != 0: n1 = wh*ww, n2 = (wh/df)*(ww/df); else transposed roles. */
int grl_rel_index_host(int wh, int ww, int df, int window_to_anchor, int64_t* out);
/* calculate_mask / calculate_mask_all (ops.py:112-157): out is (nW, n1, n2) fp32 of 0 / -100. */
int grl_shift_mask_host(int H, int W, int wh, int ww, int sh, int sw, int df, int window_to_anchor, float* out);
/* get_relative_coords_table_all (ops.py:225-271), pretrained size 0: out is ((wh+awh-1)*(ww+aww-1), 2) fp32 */
int grl_coords_table_host(int wh, int ww, int df, float* out);
/* torch.roll(-shift) + window_partition (ops.py:36-53, efficient.py:141-143,:236-241) as a gather map: out is
 * (nW, wh*ww) int32, the flat index y*W + x (un-rolled image) of token n of window w -- the addressing every attention
 * kernel folds into its loads and stores. */
int grl_token_map_host(GrlGrid g, int32_t* out);
/* Tokens per TMA box of the attention kernel for this grid (csrc/attn_tc.cu): runs of that many
 * tokens starting at multiples of it are contiguous in memory for every window.  0 = no box form (gather kernel). */
int grl_tc_attn_box_tokens(GrlGrid g);

/* ---- fp32 operators (exact-parity path; every one is a hand-written sm_90a kernel) ---------- */

/* AffineTransform bias: out[h, r] = 16*sigmoid(CPB_MLP(table[r]))  for r < rows
 * (mixed_attn_block_efficient.py:41-47 with the gather commuted out; mixed_attn_block.py:24-31).
 * table (rows,2); w1 (hidden,2); b1 (hidden); w2 (heads,hidden); out (heads, rows). */
int grl_bias_table_f32(const float* table, int rows, const float* w1, const float* b1, const float* w2,
                       int hidden, int heads, float* out, void* stream);

/* AffineTransform.forward on a materialised map (mixed_attn_block_efficient.py:36-58):
 * attn (B_, heads, n1, n2) in place: attn*exp(min(logit_scale,ln100)) + bias[h, index[i,j]] + mask[b_%nW,i,j].
 * bias = output of grl_bias_table_f32; index (n1,n2) int64; mask (nW,n1,n2) or NULL. */
int grl_affine_f32(float* attn, int64_t B_, int heads, int n1, int n2, const float* logit_scale,
                   const float* bias, int rows, const int64_t* index, const float* mask, int nW, void* stream);

/* y[m, n] = act(sum_k x[m*ldx + k] * w[n*K + k] + b[n]) (+ res[m*ldr + n]);  nn.Linear / QKVProjection /
 * AnchorLinear.reduction / Mlp.fc1,fc2 / MixedAttention.proj (mixed_attn_block.py:661-676,:714-736;
 * swin_v1_block.py:37-43; mixed_attn_block_efficient.py:379). b, res may be NULL. */
int grl_linear_f32(const float* x, int64_t ldx, const float* w, const float* b, const float* res, int64_t ldr,
                   float* y, int64_t ldy, int64_t M, int N, int K, int act, float slope, void* stream);

/* 3x3 / stride 1 / pad 1 convolution on channels-last data (nn.Conv2d in CAB mixed_attn_block.py:973-977,
 * TransformerStage.conv grl.py:136,:168, conv_first / conv_after_body / upsampler heads grl.py:293,:348-379).
 * x (B,H,W,Cin); w packed (Cout, 9*Cin) with k = (ky*3+kx)*Cin + c; y (B,H,W,Cout); res optional (B,H,W,Cout). */
int grl_conv3x3_f32(const float* x, const float* w, const float* b, const float* res, float* y, int B, int H, int W,
                    int Cin, int Cout, int act, float slope, void* stream);

/* AvgPool2d(df, df) on channels-last data (AnchorLinear.pooling, mixed_attn_block.py:725,:733). */
int grl_avgpool_f32(const float* x, float* y, int B, int H, int W, int C, int df, void* stream);
/* MaxPool2d(df, df) on channels-last data (AnchorLinear.pooling with pooling_mode "maxpool", mixed_attn_block.py:724). */
int grl_maxpool_f32(const float* x, float* y, int B, int H, int W, int C, int df, void* stream);
/* Patch rows of a channels-last image x (B, H, W, C) at row pitch ldx, for the convolutional anchor projections
 * (nn.Conv2d(C, C/2, k, stride, pad) and PatchMerging, mixed_attn_block.py:679-711,:745-770; the reference runs them with
 * torch's conv2d / cat + Linear): y (B*Ho*Wo, ldy), Ho = (H + 2 pad - k) / stride + 1,
 * y[(b,yo,xo), tap*C + c] = x[b, yo*stride - pad + ky, xo*stride - pad + kx, c] (0 outside), 0 for k*k*C <= col < ldy;
 * tap = ky*k + kx when row_major (nn.Conv2d's weight order), kx*k + ky otherwise (PatchMerging's x0..x3 order). */
int grl_anchor_gather_f32(const float* x, int64_t ldx, int B, int H, int W, int C, int ksize, int stride, int pad,
                          int row_major, float* y, int ldy, void* stream);

/* out = (x ? x : 0) + res_scale * LayerNorm(u; gamma, beta, eps) (+ cab_y * cab_gate[b, c])
 * (post-norm residual, mixed_attn_block_efficient.py:543-554; norm_start/norm_end grl.py:494,:501 with x = NULL).
 * Rows M = B*L; cab_y (M,C) and cab_gate (B,C) optional (both or none). */
int grl_ln_residual_f32(const float* x, const float* u, const float* gamma, const float* beta, float eps,
                        float res_scale, const float* cab_y, const float* cab_gate, int64_t L, float* out,
                        int64_t M, int C, void* stream);

/* ChannelAttention gate (mixed_attn_block.py:948-967): gate[b,c] = sigmoid(W2 relu(W1 mean_L(y[b]) + b1) + b2).
 * y (B,L,C); w1 (R,C); w2 (C,R); workspace >= grl_channel_gate_workspace(B,L,C) bytes. */
size_t grl_channel_gate_workspace(int B, int64_t L, int C);
int grl_channel_gate_f32(const float* y, int B, int64_t L, int C, const float* w1, const float* b1, const float* w2,
                         const float* b2, int R, float* gate, void* workspace, size_t workspace_bytes, void* stream);

/* WindowAttention.forward (mixed_attn_block_efficient.py:128-165) fused: roll + partition + cosine attention
 * + learned scale + relative-position bias + shift mask + softmax + AV + merge + reverse roll.
 * qkv: token rows of `ld_qkv` floats; the window half starts at qkv and is laid out (3, heads, d).
 * out: token rows of `ld_out` floats, channel = head*d + e.  bias (heads, rows) from grl_bias_table_f32 with
 * rows = (2wh-1)(2ww-1).  use_mask: apply the region-id shift mask (mask argument not None in the reference). */
int grl_window_attn_f32(const float* qkv, int64_t ld_qkv, float* out, int64_t ld_out, int B, GrlGrid grid, int heads,
                        int d, const float* logit_scale, const float* bias, int use_mask, void* stream);

/* AnchorStripeAttention.forward (mixed_attn_block_efficient.py:215-270) fused: two chained attentions
 * X1 = softmax(a k^T) v (anchors attend to the stripe), Y = softmax(q a^T) X1.
 * qkv: stripe half (3, heads, d) per token; anchor (B, H/df, W/df, heads*d) rows of `ld_anchor` floats;
 * tok = stripe grid on tokens, anc = the same stripes on the anchor grid; bias1/scale1 = attn_transform1
 * (a2w index), bias2/scale2 = attn_transform2 (w2a index).  workspace >= grl_stripe_attn_workspace bytes. */
size_t grl_stripe_attn_workspace(int B, GrlGrid tok, GrlGrid anc, int heads, int d);
int grl_stripe_attn_f32(const float* qkv, int64_t ld_qkv, const float* anchor, int64_t ld_anchor, float* out,
                        int64_t ld_out, int B, GrlGrid tok, GrlGrid anc, int heads, int d, const float* logit_scale1,
                        const float* bias1, const float* logit_scale2, const float* bias2, int use_mask,
                        void* workspace, size_t workspace_bytes, void* stream);

/* ---- bf16 tensor-core operators (throughput path: wgmma + TMA, sm_90a only) ----------------
 * Activations are bf16 with channel pitches padded to a multiple of 64; attention heads live in 32-wide "slots"
 * (head_dim zero-padded to 32).  The residual stream, LayerNorm, softmax statistics and all accumulators stay fp32. */

/* grl_bias_table_f32 scaled by `mul` (log2(e) for the exp2-domain softmax of grl_tc_attn) and written as FOUR
 * copies, copy c shifted right by c entries: out[(h*4 + c)*rows_pad + r + c] = bias[h][r].  `out` (heads, 4, rows_pad)
 * must be zero-initialised; rows_pad % 4 == 0, rows_pad >= rows + 4.  The attention kernel reads runs of four
 * consecutive table entries as one aligned 16-byte load from the copy that matches the run's alignment. */
int grl_tc_bias_table4(const float* table, int rows, const float* w1, const float* b1, const float* w2, int hidden,
                       int heads, float mul, int rows_pad, float* out, void* stream);

/* `fmt` selects the 16-bit operand format everywhere below: 0 = fp16 (default: 11-bit mantissa, saturating
 * converts; needed for the 0.01 dB PSNR gate), 1 = bf16.  Both run wgmma at the same rate. */

/* fp32 (M, C) rows of pitch ldx -> 16-bit (M, Cpad) zero-padded; and back (16-bit rows of pitch ldx, column offset). */
int grl_tc_pack16(const float* x, int64_t ldx, void* y16, int64_t M, int C, int Cpad, int fmt, void* stream);
int grl_tc_unpack16(const void* x16, int64_t ldx, int x_off, float* y, int64_t ldy, int64_t M, int C, int fmt, void* stream);
/* Network input in one pass: check_image_size (reflect pad on the bottom / right up to (Hp, Wp); zero pad when the pad
 * exceeds the image, as grl.py:485-488 falls back) + (x - mean) * img_range (grl.py:510-511) + bchw -> channels-last +
 * 16-bit pack.  x (B, 1 <= Cin <= 8, H, W) fp32 -> y16 (B, Hp, Wp, Cpad), zero in [Cin, Cpad); y32 (may be NULL): the
 * fp32 channels-last copy (B, Hp, Wp, Cin) the no-upsampler heads add back (grl.py:540-547).  mean4 (may be NULL: zero
 * mean): max(4, Cin) HOST floats, i.e. exactly 4 for Cin <= 4 and Cin for Cin in 5..8 (the 6-channel dual-pixel input);
 * entries past Cin are not used. */
int grl_tc_head_pack(const float* x, int B, int Cin, int H, int W, int Hp, int Wp, const float* mean4, float range, void* y16,
                     int Cpad, float* y32, int fmt, void* stream);
/* grl_tc_head_pack of the demosaiced image, with the demosaic fused in: cfa4 (B, 4, h, w) fp32 packed RGGB planes are the
 * network input dm_matlab(cfa4) (utils/utils_mosaic.py:36-111; engines/base.py:127-128) of size (H, W) = (2h, 2w), Cin = 3.
 * Each padded pixel is the demosaic at the source pixel check_image_size maps it to (zero pad as in grl_tc_head_pack), so
 * the full-resolution RGB image is never written.  y32 as in grl_tc_head_pack.  h, w >= 2. */
int grl_tc_head_pack_rggb(const float* cfa4, int B, int h, int w, int Hp, int Wp, const float* mean4, float range, void* y16,
                          int Cpad, float* y32, int fmt, void* stream);
/* AvgPool2d(df) on 16-bit channels-last data (AnchorLinear.pooling, mixed_attn_block.py:725). */
int grl_tc_avgpool16(const void* x16, void* y16, int B, int H, int W, int Cpad, int df, int fmt, void* stream);
/* MaxPool2d(df) on 16-bit channels-last data (AnchorLinear.pooling with pooling_mode "maxpool", mixed_attn_block.py:724). */
int grl_tc_maxpool16(const void* x16, void* y16, int B, int H, int W, int Cpad, int df, int fmt, void* stream);
/* grl_anchor_gather_f32 on 16-bit operands (either format: the values are copied): the K operand of the anchor
 * projection's grl_tc_gemm, ldy a multiple of 64. */
int grl_tc_anchor_gather16(const void* x16, int64_t ldx, int B, int H, int W, int C, int ksize, int stride, int pad,
                           int row_major, void* y16, int ldy, void* stream);
/* Per-slot multipliers of the packed qkv layout [win q|k|v][stripe q|k|v] x heads: exp(min(logit_scale, ln100))*log2(e)
 * on window q, stripe q (attn_transform2) and stripe k (attn_transform1); 1 on the other q/k slots; 0 on v slots
 * (mixed_attn_block_efficient.py:39). out: (3*hw + 3*hs) floats. */
int grl_tc_slot_scale(const float* ls_window, const float* ls_stripe1, const float* ls_stripe2, int heads_w, int heads_s,
                      float* out, void* stream);
/* ChannelAttention gate from bf16 CAB features y (B, L, ld) (mixed_attn_block.py:948-967). */
size_t grl_tc_channel_gate_workspace(int B, int64_t L, int C);
int grl_tc_channel_gate(const void* y16, int64_t ld, int fmt, int B, int64_t L, int C, const float* w1, const float* b1,
                        const float* w2, const float* b2, int R, float* gate, void* workspace, size_t workspace_bytes,
                        void* stream);

/* Tensor-core GEMM / implicit-GEMM 3x3 conv with a fused epilogue.  x: bf16 (M, kpad) or (B, H, W, kpad) when taps == 9;
 * w: bf16 (npad, taps*kpad) K-major (conv: k = tap*kpad + c, tap = ky*3+kx); bias: (npad) fp32, zero in the pad.
 *   epi 0  y = act(acc + b) (+ res_f32)           -> out_bf16 (n_store cols) and/or out_f32 (n_real cols)
 *          nn.Linear / nn.Conv2d of Mlp.fc1, CAB, TransformerStage.conv, conv_first/after_body/upsampler heads
 *   epi 1  per 32-wide slot: (acc + b) * slot_scale / max(||.||2, 1e-12) (slot_scale <= 0: untouched) -> out_bf16
 *          QKVProjection / AnchorLinear.reduction fused with F.normalize + logit scale (efficient.py:39,:85)
 *   epi 2  out = res_f32 + res_scale * LayerNorm(acc + b) (+ cab_y * cab_gate[token / L]) -> out_f32 + out_bf16
 *          MixedAttention.proj + norm1 + CAB add, Mlp.fc2 + norm2 (efficient.py:543-554); needs npad <= 256. */
typedef struct {
  int32_t fmt; /* 0 = fp16, 1 = bf16 */
  const void* x;
  const void* w;
  const float* bias;
  int64_t M;
  int32_t B, H, W;
  int32_t kpad, npad, taps, epi;
  int32_t n_store, n_real;
  void* out_bf16;
  int64_t ldo_bf16;
  float* out_f32;
  int64_t ldo_f32;
  const float* res_f32;
  int64_t ldr;
  int32_t act;
  float slope;
  const float* slot_scale;
  int32_t C;
  const float* gamma;
  const float* beta;
  float eps, res_scale;
  const void* cab_y;
  int64_t ld_caby;
  const float* cab_gate;
  int64_t L;
  /* head / tail fusion (taps == 9 only; zero = off).
   * ps_r > 0: PixelShuffle(ps_r) folded into the 16-bit store (models/common/upsample.py:6-30): w rows must be packed so
   *   that output column n' = q * (n_store / r^2) + c holds torch channel c * r^2 + q; out_bf16 is (B, H r, W r, ldo_bf16).
   * out_nchw: final image planes (B, n_real / nchw_r^2, Hc, Wc) fp32 = value * post_scale + post_shift[c]: x / img_range +
   *   mean, the crop to (Hc, Wc) and bhwc -> bchw (grl.py:549-551) folded into the store; nchw_r > 1 additionally folds
   *   UpsampleOneStep's PixelShuffle (upsample.py:33-50, torch channel order). */
  int32_t ps_r;
  float* out_nchw;
  int32_t nchw_r, Hc, Wc;
  float post_scale;
  float post_shift[4];
} GrlTcGemm;
int grl_tc_gemm(const GrlTcGemm* p, void* stream);

/* The launch path grl_tc_gemm takes for problem p, from the same host-side selection, without a device: validates p
 * like grl_tc_gemm (pointers are only tested for NULL, never dereferenced) and fills *out. */
typedef struct {
  int32_t bn;       /* N tile width: 64, 128, 192 or 256 */
  int32_t epi_mode; /* 0 = 16-bit outputs only, 1 = fp32 staging (whole row in one tile), 2 = direct per-row stores */
  int32_t conv;     /* 1 = implicit-GEMM 3x3 conv (taps == 9) */
  int32_t n_tiles;  /* N tiles of one row tile */
  int32_t nk_total; /* 64-wide k chunks through the 4-stage operand ring: taps * kpad / 64 */
  int64_t grid;     /* CTAs: row tiles (conv: 8 x 16 pixel patches of every image) x n_tiles */
} GrlTcGemmPath;
int grl_tc_gemm_path(const GrlTcGemm* p, GrlTcGemmPath* out);

/* Fused cosine attention over packed bf16 head slots: out = softmax2(q k^T + bias + mask) v, one call per
 * WindowAttention.forward and two per AnchorStripeAttention.forward (efficient.py:128-165,:215-270).
 * q/k/v: bf16 token rows (pitch ld*, element offset *_off of head 0's slot); v_dense/o_dense: the (B_, heads, N, 32)
 * intermediate X1 of the stripe attention; bias: (heads, 4, rows_pad) fp32 from grl_tc_bias_table4(.., log2 e, ..). */
typedef struct {
  int32_t fmt; /* 0 = fp16, 1 = bf16 */
  GrlGrid gq, gk;
  const void* q;
  int64_t ldq;
  int32_t q_off;
  const void* k;
  int64_t ldk;
  int32_t k_off;
  const void* v;
  int64_t ldv;
  int32_t v_off;
  int32_t v_dense;
  void* out;
  int64_t ldo;
  int32_t o_off;
  int32_t o_dense;
  int32_t B, heads;
  const float* bias; /* (heads, 4, rows_pad) from grl_tc_bias_table4 */
  int32_t rows;
  int32_t rows_pad;
  int32_t use_mask;
  int32_t ones_col; /* 1: column 31 of every V row is 1.0 (head_dim < 32) -> the row sum comes out of the P V MMA */
} GrlTcAttn;
int grl_tc_attn(const GrlTcAttn* p, void* stream);

/* How grl_tc_attn loads its operands: 5 (default) = Q and the K / V tiles as TMA boxes of the (B, H, W, C) tensors for
 * every geometry whose rolled window rows split into runs of >= 8 contiguous tokens (grl_tc_attn_box_tokens > 0), row
 * gathers with cp.async for the rest; 0 = row gathers everywhere.  Initial value: environment variable GRL_ATTN_SPLIT
 * (unset = 5).  Returns the previous value; anything but 0 / 5 only queries.  Both compute the same function. */
int grl_tc_attn_variant(int variant);


/* ---- validation metric (SURVEY.md 8f row 3) -------------------------------------------------- */
/* Per-image PSNR of the reference's validation step in one fused pass: tensor_round (utils/utils_image.py:30-33) of
 * both images, `border` pixels shaved on every side (engines/base.py:265-267, utils_image.py:8-11), mean squared error
 * over (C, H, W) and -10 log10 (utils/metrics/psnr.py:44-48).  restored / target: (B, C, H, W) fp32, C <= 4.
 * psnr_y (may be NULL): the same on the luma of MATLAB's rgb2ycbcr rounded to 8 bit (utils_image.py:43-80) when C == 3,
 * else a copy of psnr_rgb.  The error is accumulated exactly (integers), so the result does not depend on the launch
 * geometry.  workspace: 16 * B bytes of device memory (zeroed by the call). */
int grl_psnr_f32(const float* restored, const float* target, int B, int C, int H, int W, int border, void* workspace,
                 size_t workspace_bytes, float* psnr_rgb, float* psnr_y, void* stream);
/* Every metric entry point below has a _u8 sibling that takes 8-bit images, restored / target (B, H, W, C) uint8 (note the
 * argument order B, H, W, C), as they come out of grl_f32_to_u8 or an image decoder: the bytes are the 8-bit integers
 * tensor_round gives, so the result equals that of the _f32 entry point on grl_u8_to_f32 of the same images bit for bit.
 * Shapes, workspaces and outputs are those of the _f32 entry point. */
int grl_psnr_u8(const uint8_t* restored, const uint8_t* target, int B, int H, int W, int C, int border, void* workspace,
                size_t workspace_bytes, float* psnr_rgb, float* psnr_y, void* stream);

/* Per-image PSNR-B of the JPEG test commands (PeakSignalNoiseRatioBlock.update, utils/metrics/psnrb.py:141-163) on
 * tensor_round'ed images, no shave: per channel 10 log10(1 / (mse + bef)) with the blocking-effect factor bef of the
 * RESTORED image (psnrb.py:22-101, its normalisers H * (W // 8 - 1) etc. as written there, not the counts of the summed
 * positions), averaged in dB over the channels.  restored / target: (B, C, H, W) fp32, C = 1 or 3, H, W >= 16.
 * psnrb_y (may be NULL): the same on the luma of grl_psnr_f32 for C == 3, else a copy of psnrb_rgb.  Both outputs are
 * float64.  The sums are exact integers, so the result does not depend on the launch geometry.
 * workspace >= grl_psnrb_workspace(B) bytes of device memory (zeroed by the call). */
size_t grl_psnrb_workspace(int B);
int grl_psnrb_f32(const float* restored, const float* target, int B, int C, int H, int W, void* workspace,
                  size_t workspace_bytes, double* psnrb_rgb, double* psnrb_y, void* stream);
int grl_psnrb_u8(const uint8_t* restored, const uint8_t* target, int B, int H, int W, int C, void* workspace,
                 size_t workspace_bytes, double* psnrb_rgb, double* psnrb_y, void* stream);

/* Per-image SSIM of the validation step (StructuralSimilarityIndexMeasure.update, utils/metrics/ssim.py:167-193 ->
 * ssim / _ssim, ssim.py:36-85, after engines/base.py:255-268): both images tensor_round'ed, `border` pixels shaved, local
 * statistics under the 11-tap Gaussian window of gaussian(11, 1.5) (ssim.py:17-24) with zero padding and no
 * renormalisation at the border, C1 = 1e-4, C2 = 9e-4, the mean of the map over channels and pixels.  restored / target:
 * (B, C, H, W) fp32, C == 1 or 3, 2 * border < min(H, W).  ssim_y (may be NULL): the same on the luma of grl_psnr_f32 for
 * C == 3, else a copy of ssim_rgb.  Both outputs are float64 (B,).  Arithmetic is float64 on the exact 8-bit integers and
 * separable (csrc/grl_ssim.h); partial sums are combined in a fixed order, so two calls give the same bits and an image
 * scores the same alone and in a batch.  map_rgb (B, C, H - 2 border, W - 2 border) and map_y (B, 1, ...; written for
 * C == 3 only) receive the float64 SSIM map when not NULL.  workspace >= grl_ssim_workspace(...) bytes of device memory
 * (0 for a shape the call refuses). */
size_t grl_ssim_workspace(int B, int C, int H, int W, int border);
int grl_ssim_f32(const float* restored, const float* target, int B, int C, int H, int W, int border, void* workspace,
                 size_t workspace_bytes, double* ssim_rgb, double* ssim_y, double* map_rgb, double* map_y, void* stream);
int grl_ssim_u8(const uint8_t* restored, const uint8_t* target, int B, int H, int W, int C, int border, void* workspace,
                size_t workspace_bytes, double* ssim_rgb, double* ssim_y, double* map_rgb, double* map_y, void* stream);
/* The 11 normalised float64 window taps (gaussian(11, 1.5), ssim.py:17-24); HOST pointer. */
int grl_ssim_taps_host(double* taps11);
/* grl_ssim_f32 on the CPU from the same closed form, HOST pointers; its maps equal the kernel's bit for bit.  Allocates
 * host scratch of 8 planes of float64. */
int grl_ssim_host(const float* restored, const float* target, int B, int C, int H, int W, int border, double* ssim_rgb,
                  double* ssim_y, double* map_rgb, double* map_y);

/* ---- NIQE features of the blind-SR test command (NaturalImageQualityEvaluator.update, utils/metrics/niqe.py:566-576) --
 * restored: (B, C = 3, H, W) fp32; the score is the multivariate-Gaussian distance of the features to the caller's
 * pristine model (metrics.niqe, batched torch float64).  The crop keeps (Hc, Wc) = 96 * floor((H - 2 border, W - 2 border)
 * / 96) from the top left of the border-cropped image; both need at least 96 pixels.
 * window49: HOST pointer to the 7 x 7 float64 gaussian_window of niqe_pris_params.npz.  tables: DEVICE (4, 9801) float64:
 * gam = 0.2 : 0.001 : 10 as np.arange builds it, r_gam = G(2/g)^2 / (G(1/g) G(3/g)) with 1/g computed first,
 * sqrt(G(1/g) / G(3/g)) and G(2/g) / G(1/g).  feats: (B, nbw * nbh, 36) float64, row iw * nbh + ih, 18 features of the
 * 96 x 96 block at scale 1 then 18 of the 48 x 48 block at scale 2.  The stage entry points are the pieces
 * grl_niqe_features_f32 runs, one kernel each (csrc/niqe.cu). */
size_t grl_niqe_workspace(int B, int H, int W, int border);
int grl_niqe_features_f32(const float* restored, int B, int C, int H, int W, int border, const double* window49,
                          const double* tables, void* workspace, size_t workspace_bytes, double* feats, void* stream);
int grl_niqe_features_u8(const uint8_t* restored, int B, int H, int W, int C, int border, const double* window49,
                         const double* tables, void* workspace, size_t workspace_bytes, double* feats, void* stream);
/* The rounded luma (an integer in [16, 235] as fp32) of n 8-bit RGB triples rgb (n, 3); HOST pointers (csrc/grl_niqe.h). */
int grl_niqe_luma_host(const uint8_t* rgb, int64_t n, float* y);
/* The 8 fp32 taps of the x0.5 antialiased bicubic resize (niqe.py:169-238); HOST pointer. */
int grl_niqe_half_taps_host(float* w8);
/* luma + crops: y (B, Hc, Wc). */
int grl_niqe_luma_f32(const float* restored, int B, int C, int H, int W, int border, float* y, void* stream);
int grl_niqe_luma_u8(const uint8_t* restored, int B, int H, int W, int C, int border, float* y, void* stream);
/* MSCN of img (B, H, W) -> out (B, H, W) (niqe.py:447-455). */
int grl_niqe_mscn_f32(const float* img, int B, int H, int W, const double* window49, float* out, void* stream);
/* 255 * imresize(img / 255, 0.5) (niqe.py:470-471): img (B, H, W), H and W even; tmp (B, H/2, W); out (B, H/2, W/2). */
int grl_niqe_half_f32(const float* img, int B, int H, int W, float* tmp, float* out, void* stream);
/* Features of the MSCN images mscn1 (B, 96 nbh, 96 nbw) and mscn2 (B, 48 nbh, 48 nbw). */
int grl_niqe_feat_f32(const float* mscn1, const float* mscn2, int B, int nbh, int nbw, const double* tables, double* feats,
                      void* stream);

/* ---- LPIPS of the perceptual metric collection (LearnedPerceptualImagePatchSimilarity.update, utils/metrics/lpips.py:24-42
 * -> lpips.LPIPS(net="vgg").forward(img1, img2, normalize=True), version 0.1) -- the pieces specific to LPIPS; the 13
 * VGG16 convolutions run on grl_conv3x3_f32 (metrics.lpips).  csrc/lpips.cu. */
/* The trunk input of both images at once: restored / target (B, C = 3, H, W) fp32, tensor_round'ed inside, or their bytes
 * (B, H, W, 3) uint8; `border` pixels shaved on every side (engines/base.py:264-266) -> out (2B, Hc, Wc, 3) channels-last
 * fp32, restored images at rows 0..B-1 and targets at B..2B-1, each value 2 x - 1, minus shift, over scale in fp32 in
 * that order (csrc/grl_lpips.h).  The two entry points give the same bits for an image and u8_to_f32 of it. */
int grl_lpips_head_f32(const float* restored, const float* target, int B, int C, int H, int W, int border, float* out,
                       void* stream);
int grl_lpips_head_u8(const uint8_t* restored, const uint8_t* target, int B, int H, int W, int C, int border, float* out,
                      void* stream);
/* The head's value for n 8-bit RGB triples rgb (n, 3) -> out (n, 3) fp32; HOST pointers. */
int grl_lpips_head_host(const uint8_t* rgb, int64_t n, float* out);
/* MaxPool2d(2, 2) with floor sizes (VGG16 features 4, 9, 16, 23): x (N, H, W, C) -> y (N, H/2, W/2, C) channels-last fp32,
 * equal to torch.max_pool2d bit for bit, NaN propagated. */
int grl_maxpool2_f32(const float* x, int N, int H, int W, int C, float* y, void* stream);
/* One tap's distance (lpips.LPIPS.forward: normalize_tensor, squared difference, lin k, spatial_average): tap (2B, h, w, C)
 * fp32, images 0..B-1 against B..2B-1, C a multiple of 32 up to 512; lin_w (C) fp32 -> res (B) float64, the mean over the
 * h w pixels of sum_c lin_w[c] (f0_c / (|f0| + 1e-10) - f1_c / (|f1| + 1e-10))^2.  Per-pixel arithmetic is fp32; the mean
 * is float64 in a fixed order, so two calls give the same bits and an image's value does not depend on its batch.
 * workspace >= grl_lpips_workspace(B, h, w) bytes of device memory. */
size_t grl_lpips_workspace(int B, int h, int w);
int grl_lpips_layer_f32(const float* tap, int B, int h, int w, int C, const float* lin_w, void* workspace,
                        size_t workspace_bytes, double* res, void* stream);

/* ---- x8 self-ensemble (geometric test-time augmentation) ----------------------------------------
 * The 8 views are augment_img_tensor4(img, mode) (utils/utils_bsr/utils_image.py:444-460).  Group A = modes 0, 2, 4, 6
 * (the view keeps (H, W)), group B = modes 1, 3, 5, 7 (the view is (W, H)); inside a group view i is mode 2*i + group. */
/* Host expansion of the view maps: inverse == 0: out (H', W') int32 = flat index sy*W + sx of the source pixel of every
 * view position ((H', W') = (W, H) for group B); inverse != 0: out (H, W) int32 = flat index py*W' + px of the view
 * position that holds each image pixel (the map that undoes the view). */
int grl_d8_index_host(int mode, int H, int W, int inverse, int32_t* out);
/* augment_img_tensor4(x, mode) for the 4 modes of one group in one pass: x (B, C, H, W) fp32 -> views (4B, C, H', W'),
 * view-major (view i of image b is index i*B + b). */
int grl_ens_gather_f32(const float* x, int B, int C, int H, int W, int group, float* views, void* stream);
/* The self-ensemble average: y[b] = 0.125 * (V_0 + V_1 + ... + V_7), summed in mode order in fp32, where V_m is view m's
 * network output mapped back by the inverse of augment_img_tensor4(., m).  ya: group A outputs (4B, C, Hs, Ws); yb: group B
 * outputs (4B, C, Ws, Hs), both view-major (they may be the two halves of one tensor when Hs == Ws); y (B, C, Hs, Ws). */
int grl_ens_merge_f32(const float* ya, const float* yb, int B, int C, int Hs, int Ws, float* y, void* stream);

/* ---- demosaicking (the dm task's input, engines/base.py:127-128) ----------------------------------
 * dm_matlab (utils/utils_mosaic.py:36-111): packed RGGB planes cfa4 (B, 4, h, w) fp32 (R, G at (even, odd), G at (odd,
 * even), B; data/datasets/restoration_dm.py:33) -> RGB (B, 3, 2h, 2w) fp32.  The mosaic is reflect-padded by 2 and
 * correlated with the four 5 x 5 filters; each channel keeps the raw mosaic value at its native sites and takes one
 * filter's response at the others (utils_mosaic.py:97-109).  Every response is summed in the fixed tap order of
 * csrc/grl_demosaic.h, so the host expansion and both kernels agree bit for bit.  h, w >= 2. */
/* Host evaluation (tests): cfa4 and out are HOST pointers. */
int grl_demosaic_host(const float* cfa4, int B, int h, int w, float* out);
int grl_demosaic_f32(const float* cfa4, int B, int h, int w, float* out, void* stream);

/* ---- 8-bit images (the datasets' to_tensor and the validation step's tensor_round, csrc/grl_image_u8.h) -------------
 * The 8-bit grid at both ends of the pipeline, as two layout transposes: 8-bit HWC pixels, as image decoders give them,
 * and fp32 CHW planes, as the network and the metrics take them.  1 <= C <= 8 (the 6-channel dual-pixel input). */
/* src (B, H, W, C) uint8 -> dst (B, C, H, W) fp32 = k / 255, correctly rounded: transforms.functional.to_tensor of every
 * dataset (data/datasets/restoration_sr.py:114-115), i.e. torch's img.float().div(255) on the CPU. */
int grl_u8_to_f32(const uint8_t* src, int B, int H, int W, int C, float* dst, void* stream);
/* src (B, C, H, W) fp32 -> dst (B, H, W, C) uint8 = rint(clamp(v, 0, 1) * 255), ties to even: tensor_round
 * (utils/utils_image.py:30-33) times 255, the bytes of a saved image.  NaN, which torch leaves undefined, gives 0. */
int grl_f32_to_u8(const float* src, int B, int C, int H, int W, uint8_t* dst, void* stream);
/* The same two maps on the CPU from the same closed forms (tests); HOST pointers, any C >= 1. */
int grl_u8_to_f32_host(const uint8_t* src, int B, int H, int W, int C, float* dst);
int grl_f32_to_u8_host(const float* src, int B, int C, int H, int W, uint8_t* dst);

/* ---- lists of differently sized images (GRL.forward_list, csrc/image_list.cu) -----------------------------------------
 * The reference forward takes one (B, C, H, W) tensor, so a test set of differently sized images runs as a loop of B = 1
 * forwards.  A forward's arithmetic depends only on the padded size, so images that check_image_size pads to the same
 * (Hp, Wp) can share one forward: these two calls move such a group in and out of that batch.
 * A GrlImageRef describes one image of a list; `data` is a DEVICE pointer, the array of GrlImageRef is a HOST array that
 * the call copies into kernel parameters (no device copy).  Every ref of one call has the same kind.
 *   GRL_IMAGE_F32  (C, H, W) fp32 planes
 *   GRL_IMAGE_U8   (H, W, C) uint8 pixels, as image decoders give them (k / 255 of grl_u8_to_f32 on the way in, round8 of
 *                  grl_f32_to_u8 on the way out)
 *   GRL_IMAGE_RGGB (4, H, W) fp32 packed RGGB planes of a (2H, 2W) image, demosaiced as by grl_demosaic_f32 (gather only;
 *                  C = 3, H, W >= 2) */
typedef enum { GRL_IMAGE_F32 = 0, GRL_IMAGE_U8 = 1, GRL_IMAGE_RGGB = 2 } GrlImageKind;
typedef struct {
  void* data;
  int32_t H, W; /* the image's size (RGGB: of the packed planes) */
  int32_t kind; /* GrlImageKind */
} GrlImageRef;
/* check_image_size (grl.py:479-489) of every image of the list into one padded batch: out (n, C, Hp, Wp) fp32, image i
 * (size H x W <= Hp x Wp, demosaiced first for RGGB) reflect-padded on the bottom / right, or zero-padded on both axes
 * when Hp - H >= H or Wp - W >= W (F.pad raises and the reference falls back to constant padding, grl.py:485-488).
 * Image i of the batch equals check_image_size(x_i[None])[0] bit for bit when (Hp, Wp) is x_i's padded size.
 * 1 <= C <= 8. */
int grl_list_gather(const GrlImageRef* images, int n, int C, int Hp, int Wp, float* out, void* stream);
/* The crop of the reference's forward (grl.py:549-551) for every image of a batch: y (n, C, Hy, Wy) fp32 -> image i's
 * top-left (H, W) <= (Hy, Wy) corner, written to images[i].data as fp32 planes or as the uint8 pixels of grl_f32_to_u8.
 * 1 <= C <= 8; kind GRL_IMAGE_F32 or GRL_IMAGE_U8. */
int grl_list_crop(const float* y, int n, int C, int Hy, int Wy, const GrlImageRef* images, void* stream);

/* ---- tiled inference over a list of images (tiling.forward_tile_list, csrc/image_list.cu, csrc/grl_tiles.h) ------------
 * BaseEngine.forward_tile (engines/base.py:90-116) restores one image as t x t tiles, t = min(tile, H, W), at the origins
 * range(0, H - t, stride) + [H - t], stride = t - overlap (the same on W), sums each tile's output into E, counts into W
 * and returns E / W.  Every tile is restored on its own and a forward's result depends only on the padded size, so the
 * tiles of a whole list of images can share forwards: these three calls cut the tiles into a padded batch and blend the
 * batch's outputs into each image's accumulator, bit for bit as the per-image loop does.  Tile k of an image is tile
 * (row k / n_cols, column k % n_cols) of its origin grid, row-major: forward_tile's order. */
/* One tile of a list: the t x t window at (y0, x0) of image src, in the frame the network sees (RGGB: the demosaiced
 * (2H, 2W) frame). */
typedef struct {
  GrlImageRef src;
  int32_t y0, x0, t;
} GrlTileRef;
/* check_image_size (grl.py:479-489) of every tile's window into one padded batch: out (n, C, Hp, Wp) fp32, tile i's
 * window reflect-padded on the bottom / right, or zero-padded on both axes when Hp - t >= t or Wp - t >= t, as for the
 * whole images of grl_list_gather.  With Hp = Wp = t it is a plain cut.  Every source has the same kind; RGGB windows
 * are read from the demosaic of the whole frame (grl_demosaic_f32), as forward_tile demosaics before cutting.
 * 1 <= C <= 8, t <= min(Hp, Wp). */
int grl_tile_gather(const GrlTileRef* tiles, int n, int C, int Hp, int Wp, float* out, void* stream);
/* The blend state of one image of the list. */
typedef struct {
  float* E;         /* (C, H*scale, W*scale) fp32 accumulator, zeroed before the image's first tile */
  uint8_t* out_u8;  /* grl_tile_finish: NULL -> E / count in place in E; else (H*scale, W*scale, C) uint8 round8(E / count) */
  int32_t H, W;     /* the image's size in the network's frame */
  int32_t t, overlap;
  int32_t k0, k1;   /* grl_tile_accumulate: the image's tiles [k0, k1) are in this batch ... */
  int32_t slot;     /* ... tile k0 at batch index slot, the rest after it in order */
} GrlTileImage;
/* Adds the outputs of the tiles a batch holds to their images' accumulators: y (n, C, Hy, Wy) fp32 is the forward's
 * output of a grl_tile_gather batch; tile k's output is the top-left (t*scale)^2 of y[slot + k - k0].  At every output
 * pixel the covering tiles are added in origin order, each as E = E + o, which is what the reference's slice add_ gives;
 * a later batch continues where an earlier one stopped, so the image's tiles must reach it in order. */
int grl_tile_accumulate(const float* y, int n, int C, int Hy, int Wy, int scale, const GrlTileImage* images, int m,
                        void* stream);
/* E / W of the reference once an image's last tile is accumulated: E / count with IEEE division, count = the number of
 * tiles covering the pixel, written to E (out_u8 NULL on every image) or as uint8 pixels (on every image). */
int grl_tile_finish(const GrlTileImage* images, int m, int C, int scale, void* stream);
/* Host expansion of the coverage (tests): out (size*scale, 2) int32 = the first and last tile, in origin order, that cover
 * output row Y of an axis of `size` samples tiled with side `tile` and `overlap` (the covering tiles are that run). */
int grl_tile_cover_host(int size, int tile, int overlap, int scale, int32_t* out);

/* ---- JPEG round trip (the JPEG test command's degraded input, csrc/jpeg.cu, csrc/grl_jpeg.h) ---------------------------
 * JPEGDataset.jpeg_compress (data/datasets/restoration_jpeg.py:62-79): cv2.imencode(".jpg", img, [IMWRITE_JPEG_QUALITY,
 * quality]) then cv2.imdecode, i.e. libjpeg's default baseline encode (colour: YCbCr 4:2:0; islow DCT) and default decode
 * (islow IDCT, fancy upsampling).  Entropy coding is lossless, so the decoded pixels are integer arithmetic on 8 x 8 blocks,
 * reproduced here byte for byte.  Images are (H, W, C) uint8, C = 1 (gray, one component) or 3 (RGB in, RGB out, as the
 * dataset hands them to to_tensor); 1 <= quality <= 100. */
/* Bytes of device workspace grl_jpeg_roundtrip_u8 needs for this list: H * W + 2 * ceil(H/2) * ceil(W/2) per colour image,
 * 0 for gray. */
size_t grl_jpeg_workspace(const GrlImageRef* images, int n, int C);
/* The round trip of every image of a list: src[i] -> dst[i], both GRL_IMAGE_U8 refs of the same size (a batch is a list
 * of refs into it).  Two kernels per kJpegPerLaunch (80) images, one for gray. */
int grl_jpeg_roundtrip_u8(const GrlImageRef* src, const GrlImageRef* dst, int n, int C, int quality, void* workspace,
                          size_t workspace_bytes, void* stream);
/* The same for one image on the CPU from the same closed forms (tests); HOST pointers.  Allocates host scratch of
 * 1.5 planes for colour. */
int grl_jpeg_roundtrip_host(const uint8_t* src, int H, int W, int C, int quality, uint8_t* dst);
/* tables (2, 64) int32: the luma and chroma quantisation tables of jpeg_set_quality(quality, force_baseline = TRUE), natural
 * (row-major) order; HOST pointer. */
int grl_jpeg_quant_tables_host(int quality, int32_t* tables);

/* ---- Seeded AWGN (the denoising test command's noisy input, csrc/awgn.cu, csrc/grl_awgn.h) -----------------------------
 * DnDataset.__getitem__, validation branch (data/datasets/restoration_dn.py:134-143): noise =
 * np.random.RandomState(key).normal(0, scale, (C, H, W)) with key the 8 uint32 words of sha256 of the image's name, then
 * img_gt + torch.from_numpy(noise).float() in float32.  MT19937, init_by_array and the legacy polar Gaussian are exact;
 * log(r2) is correctly rounded on the device (csrc/grl_awgn.h states the consequence). */
/* src[i] (H, W, C) uint8 GRL_IMAGE_U8 -> dst[i] (C, H, W) fp32 GRL_IMAGE_F32 = k / 255 + (float)(scale * N_i), both of one
 * size, C in {1, 3}, C * H * W < 2^31; keys: HOST array (n, 8) uint32, the RandomState(key) of image i;
 * scale = noise_sigma / 255 (>= 0, finite).  One CTA per image, kAwgnPerLaunch (64) images per launch; no workspace. */
int grl_awgn_u8(const GrlImageRef* src, const GrlImageRef* dst, const uint32_t* keys, int n, int C, double scale,
                void* stream);
/* The noise alone on the CPU from the same closed forms, log from libm as numpy's (tests): out[count] float64 =
 * RandomState(key).normal(0, scale, count); HOST pointers. */
int grl_awgn_noise_host(const uint32_t* key, int64_t count, double scale, double* out);
/* The device's double-double log (awgn_log_cr) evaluated on the CPU (tests): out[i] = log(x[i]), x[i] positive normal. */
int grl_awgn_log_host(const double* x, int64_t n, double* out);

/* ---- Dataset-side inputs of the dm and gray JPEG test commands (csrc/dataset_u8.cu, csrc/grl_dataset_u8.h) ------------
 * Bayer mosaic: DemosaicDataset.__getitem__ (data/datasets/restoration_dm.py:33-37), to_tensor(mosaic_CFA_Bayer(img)[1])
 * (utils/utils_mosaic.py:124-147).  MATLAB luma: rgb2ycbcr_np(img, y_only=True) (utils/utils_image.py:143-190), the clean
 * image of the gray JPEG command on LIVE1 / BSDS500 / Urban100 (data/datasets/base_image.py:233-241).  Both exact. */
/* src[i] (H, W, 3) uint8 GRL_IMAGE_U8 -> dst[i] (4, H / 2, W / 2) fp32 GRL_IMAGE_RGGB (H, W of the dst ref are the planes'),
 * planes R, G (even rows), G (odd rows), B of k / 255; an odd last row / column is dropped.  kDatasetPerLaunch (128)
 * images per launch; no workspace. */
int grl_mosaic_u8(const GrlImageRef* src, const GrlImageRef* dst, int n, void* stream);
/* src[i] (H, W, 3) uint8 GRL_IMAGE_U8 -> dst[i] (H, W, 1) uint8 GRL_IMAGE_U8: the luma byte of every pixel. */
int grl_luma_u8(const GrlImageRef* src, const GrlImageRef* dst, int n, void* stream);
/* The same closed forms on the CPU (tests); HOST pointers.  mosaic: one (H, W, 3) image -> out (4, H / 2, W / 2) fp32.
 * luma: n RGB pixels (n, 3) -> out (n) bytes. */
int grl_mosaic_host(const uint8_t* img, int H, int W, float* out);
int grl_luma_host(const uint8_t* rgb, int64_t n, uint8_t* out);

/* ---- Bicubic downscale (the SR test command's LR input made from the HR image, csrc/resize.cu, csrc/grl_resize.h) -------
 * The SR dataset's online LR (data/datasets/restoration_sr.py:127-141, the load_lr False branch): imresize(modcrop(img_gt)
 * / 255, 1 / s), MATLAB's bicubic imresize with antialiasing (utils/matlab_functions.py:92-188), weights and indices of
 * calculate_weights_indices (:20-88).  s in {2, 3, 4}; output ceil(H / s) x ceil(W / s), float32, neither rounded to 8 bits
 * nor clipped.  Every output has the same T = 4s taps, each rounded once to float32 from double; the H pass runs first
 * and stores float32, each pass sums its products in float64 in tap order and rounds once (csrc/grl_resize.h).  Indices
 * past an edge mirror with the edge sample repeated; a side of one sample pads with that sample.  A side of 2 .. 3, 2 .. 5
 * or 2 .. 6 samples for s = 2, 3, 4 is shorter than a pad length, where the reference's symmetric copy fails: refused. */
/* x (B, C, H, W) fp32 -> y (B, C, ceil(H / s), ceil(W / s)) fp32, 1 <= C <= 8.  One kernel per kResizePerLaunch (64)
 * images; no workspace. */
int grl_imresize_f32(const float* x, int B, int C, int H, int W, int s, float* y, void* stream);
/* src[i] (H, W, C) uint8 GRL_IMAGE_U8 (k / 255 at the load, as to_tensor) -> dst[i] (C, ceil(H / s), ceil(W / s)) fp32
 * GRL_IMAGE_F32 (H, W of the dst ref are the output's), C in {1, 3}. */
int grl_imresize_u8_list(const GrlImageRef* src, const GrlImageRef* dst, int n, int C, int s, void* stream);
/* The taps and geometry of a side of length n on the CPU (tests); HOST pointers: taps[16] (the first T used), geometry[5]
 * = {T, c, out, pad_s, pad_e}: output o reads inputs s o + c + k (0-based), k < T; out = ceil(n / s); pad_s, pad_e the
 * reference's sym_len_s, sym_len_e.  Refuses the n the device entries refuse. */
int grl_imresize_taps_host(int n, int s, float* taps, int32_t* geometry);
/* grl_imresize_f32 on the CPU from the same closed forms (tests); HOST pointers.  Equal to the device bit for bit. */
int grl_imresize_f32_host(const float* x, int B, int C, int H, int W, int s, float* y);

#ifdef __cplusplus
}
#endif
#endif /* GRL_B200_H_ */
