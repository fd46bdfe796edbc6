// ops_f32.h -- launcher declarations of the fp32 exact-parity kernels (ops_f32.cu).
#pragma once
#include <cuda_runtime.h>

#include "../../include/grl_b200.h"

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

int launch_bias_table(const float* table, int rows, const float* w1, const float* b1, const float* w2, int hidden,
                      int heads, float mul, int copies, int rows_pad, float* out, cudaStream_t st);
int launch_affine(float* attn, long long B_, int heads, int n1, int n2, const float* logit_scale, const float* bias,
                  int rows, const long long* index, const float* mask, int nW, cudaStream_t st);
int launch_gemm(const GemmArgs& a, bool conv, cudaStream_t st);
int launch_avgpool(const float* x, float* y, int B, int H, int W, int C, int df, cudaStream_t st);
int launch_ln_residual(const float* x, const float* u, const float* gamma, const float* beta, float eps,
                       float res_scale, const float* cab_y, const float* cab_gate, long long L, float* out,
                       long long M, int C, cudaStream_t st);
size_t channel_gate_ws(int B, long long L, int C);
int launch_channel_gate(const float* y, int B, long long L, int C, const float* w1, const float* b1, const float* w2,
                        const float* b2, int R, float* gate, void* ws, size_t ws_bytes, cudaStream_t st);
int launch_channel_gate_from_partial(const float* partial, int chunks, int B, long long L, int C, const float* w1,
                                     const float* b1, const float* w2, const float* b2, int R, float* gate,
                                     cudaStream_t st);
int check_grid(const GrlGrid& g, const char* what);
int launch_attn(const AttnArgs& a, cudaStream_t st);
// fused tensor_round + shave + squared-error reduction (RGB and luma) -> per-image PSNR (metric.cu)
int launch_psnr(const float* restored, const float* target, int B, int C, int H, int W, int border,
                unsigned long long* workspace, float* psnr_rgb, float* psnr_y, cudaStream_t st);
// PSNR-B: exact integer sums of the error and of the restored image's block-boundary differences -> per image (metric.cu)
size_t psnrb_workspace(int B);
int launch_psnrb(const float* restored, const float* target, int B, int C, int H, int W, unsigned long long* workspace,
                 double* psnrb_rgb, double* psnrb_y, cudaStream_t st);
// SSIM, RGB and luma, one tile kernel + a finalize (metric.cu, grl_ssim.h); ssim_host is the same computation on the CPU
size_t ssim_workspace(int B, int C, int H, int W, int border);
int launch_ssim(const float* restored, const float* target, int B, int C, int H, int W, int border, void* workspace,
                size_t workspace_bytes, double* ssim_rgb, double* ssim_y, double* map_rgb, double* map_y, cudaStream_t st);
void ssim_taps(double* t11);
int ssim_host(const float* restored, const float* target, int B, int C, int H, int W, int border, double* ssim_rgb,
              double* ssim_y, double* map_rgb, double* map_y);
// NIQE features: luma, MSCN, x0.5 resize, per-block AGGD features (niqe.cu)
void niqe_half_taps(float* w8);
size_t niqe_ws(int B, int H, int W, int border);
int launch_niqe_luma(const float* x, int B, int C, int H, int W, int border, float* y, cudaStream_t st);
int launch_niqe_mscn(const float* in, int B, int H, int W, const double* window49, float* out, cudaStream_t st);
int launch_niqe_half(const float* in, int B, int H, int W, float* tmp, float* out, cudaStream_t st);
int launch_niqe_feat(const float* m1, const float* m2, int B, int nbh, int nbw, const double* tables, double* feats,
                     cudaStream_t st);
int launch_niqe_features(const float* x, int B, int C, int H, int W, int border, const double* window49, const double* tables,
                         void* ws, size_t ws_bytes, double* feats, cudaStream_t st);
// x8 self-ensemble: the 4 views of one group, and the ordered average of the 8 mapped-back outputs (ensemble.cu)
int launch_ens_gather(const float* x, int B, int C, int H, int W, int group, float* views, cudaStream_t st);
int launch_ens_merge(const float* ya, const float* yb, int B, int C, int Hs, int Ws, float* y, cudaStream_t st);
// dm_matlab: packed RGGB planes (B, 4, h, w) -> RGB (B, 3, 2h, 2w) (demosaic.cu)
int launch_demosaic(const float* cfa4, int B, int h, int w, float* out, cudaStream_t st);

}  // namespace grl
