// Internal (C++) interfaces between the kernel files and the engine.
#pragma once
#include "common.cuh"
#include "bn_stats.cuh"

namespace ddn {

struct ConvGeom {
  int N, Hin, Win, Cin;   // gather source (NHWC)
  int Hout, Wout, Cout;   // destination (NHWC)
  int KH, KW;
  int stride;             // destination -> source coordinate multiplier
  int ups;                // source up-sampling (transposed conv); 1 for forward
  int pad, dil;
  int cin_log2;
};

// conv_simt.cu
int conv_geom_init(ConvGeom* g, int N, int Hin, int Win, int Cin, int Hout, int Wout, int Cout,
                   int KH, int KW, int stride, int ups, int pad, int dil);
int launch_pack_weights(const float* w, float* wp, int Cout, int Cin, int CinP, int KH, int KW, int dgrad, cudaStream_t st);
int launch_unpack_wgrad(const float* dwp, float* dw, int Cout, int Cin, int CinP, int KH, int KW, cudaStream_t st);
int launch_conv_gather_f32(const float* in, const float* wp, const float* addend, float* out, const ConvGeom& g, cudaStream_t st);
int launch_conv_wgrad_f32(const float* in, const float* dy, float* dwp, const ConvGeom& g, cudaStream_t st);

// bn.cu -- NHWC tensors viewed as [M = N*H*W][C]; G BatchNorm groups of M/G consecutive rows each (bn_stats.cuh)
bool bn_c_supported(int C);                       // the channel counts the BatchNorm kernels take
size_t bn_accum_bytes(int C);                     // BnAccum storage for C channels (acc + ticket), zero-filled by the owner
BnAccum bn_accum_at(void* base, int C);
// column sums of x -> mean / invstd [G][C] (+ running statistics): one launch, finalized by the last CTA
int launch_bn_stats(const float* x, int64_t M, int C, int G, BnAccum acc, float* mean, float* invstd,
                    float* running_mean, float* running_var, float momentum, float eps, cudaStream_t st);
// mean/invstd of EVERY BatchNorm from the running statistics in one launch (eval mode): `segs` lists (offset into the
// buffer array, offset into the stats array, C) per BatchNorm; stats layout per BN = [G][C] mean then [G][C] invstd
struct BnEvalSeg { int64_t rm_off, rv_off, stat_off; int C; };
int launch_bn_eval_stats_all(const float* buffers, float* stats_base, const BnEvalSeg* segs, int n_segs, int G, float eps, cudaStream_t st);
int launch_bn_eval_stats(const float* running_mean, const float* running_var, int C, int G, float eps,
                         float* mean, float* invstd, cudaStream_t st);
// eval-mode BN folded to y = x*scale + shift (scale = gamma/sqrt(rv+eps), shift = beta - rm*scale)
int launch_bn_fold(const float* running_mean, const float* running_var, const float* gamma, const float* beta, int C, float eps,
                   float* scale, float* shift, cudaStream_t st);
// y = relu?( (x-mean)*invstd*gamma+beta + res ); res = r (fp32) or r_hi + r_lo (bf16 planes), optionally itself
// batch-normalised (the downsample branch: (r-rmean)*rinvstd*rgamma+rbeta).  Outputs: fp32 `y` and / or bf16 planes.
struct BnApplyArgs {
  const float* x; const float* mean; const float* invstd; const float* gamma; const float* beta;
  const float* r; const __nv_bfloat16* r_hi; const __nv_bfloat16* r_lo;
  const float* rmean; const float* rinvstd; const float* rgamma; const float* rbeta;
  float* y; __nv_bfloat16* hi; __nv_bfloat16* lo;
  int64_t M; int C; int relu; int G;
};
int launch_bn_apply(const BnApplyArgs& a, cudaStream_t st);
// backward of y = relu?(bn(x) + res): g = dy*(y>0); sums -> dgamma,dbeta; dx (fp32 and / or planes); optional g_out (= d res).
// ReLU mask source: `y` (fp32) or `y_hi` (bf16 plane of y); with relu set and both null the mask is recomputed as
// bn(x) > 0 (valid when the forward had no residual).
struct BnBwdArgs {
  const float* dy; const float* x; const float* mean; const float* invstd; const float* gamma; const float* beta;
  const float* y; const __nv_bfloat16* y_hi;
  float* dx; __nv_bfloat16* dx_hi; __nv_bfloat16* dx_lo; float* g_out;
  float* dgamma; float* dbeta;
  BnAccum acc; float* sums;       // workspace: accumulator (zero) and [G][2][C] floats
  int64_t M; int C; int relu; int training; int G;
  int sums_ready;                 // the column sums are in `sums` already (written by a conv epilogue): skip that pass
};
int launch_bn_backward(const BnBwdArgs& a, cudaStream_t st);

// stem: conv1 raw [N,Hc,Wc,64] -> bn+relu+maxpool3x3/2 -> y [N,Hp,Wp,64] (fp32 and / or planes), argmax uint8
int launch_stem_bn_relu_pool(const float* x, const float* mean, const float* invstd, const float* gamma, const float* beta,
                             float* y, uint8_t* argmax, __nv_bfloat16* y_hi, __nv_bfloat16* y_lo,
                             int N, int Hc, int Wc, int C, int G, cudaStream_t st);
// dy_pool [N,Hp,Wp,C] -> g [N,Hc,Wc,C] = d(relu out) * (bn(x) > 0)   (pre-BN-backward gradient)
int launch_stem_pool_relu_backward(const float* dy_pool, const uint8_t* argmax, const float* x, const float* mean,
                                   const float* invstd, const float* gamma, const float* beta, float* g,
                                   int N, int Hc, int Wc, int C, int G, cudaStream_t st);

// head.cu
int launch_nchw_to_nhwc4(const float* x, float* y, int N, int H, int W, cudaStream_t st);
// feat [N*Mimg][C]: fp32 (`feat`) or bf16 planes (feat = hi + lo) when feat == nullptr
// low [N, D, Mimg] (NCHW, read by the upsample) and optionally low_nhwc [N, Mimg, D] (read by the fused loss)
int launch_fc_forward(const float* feat, const __nv_bfloat16* feat_hi, const __nv_bfloat16* feat_lo, const float* w, const float* bias,
                      float* low, float* low_nhwc, int64_t Mimg, int N, int C, int D, cudaStream_t st);
int launch_add_lowres_nhwc(const float* dlow_nhwc, float* dlow, int64_t Mimg, int N, int D, int accumulate, cudaStream_t st);
// part: fc_part_floats(C, D) floats of scratch (per-slot partial sums of dw / dbias, added in a fixed order)
size_t fc_part_floats(int C, int D);
int launch_fc_backward(const float* dlow, const float* feat, const __nv_bfloat16* feat_hi, const __nv_bfloat16* feat_lo, const float* w,
                       float* dfeat, float* dw, float* dbias, float* part, int64_t Mimg, int N, int C, int D, cudaStream_t st);
int launch_upsample_fwd(const float* x, float* y, int NC, int h, int w, int H, int W, cudaStream_t st);
int launch_upsample_bwd(const float* dy, float* dx, int NC, int h, int w, int H, int W, cudaStream_t st);
int launch_upsample_unit_fwd(const float* x, float* y, int N, int D, int h, int w, int H, int W, cudaStream_t st);
int launch_upsample_unit_bwd(const float* x, const float* dy, float* dx, float* g, int N, int D, int h, int w, int H, int W, cudaStream_t st);
int launch_fill_zero(void* p, size_t bytes, cudaStream_t st);

}  // namespace ddn
