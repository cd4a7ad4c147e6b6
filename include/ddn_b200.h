/* ddn_b200.h -- C ABI of the H100-native dense-descriptor training path.
 *
 * One shared library (libddn_b200.so, sm_90a only) exports everything below with C linkage:
 * plain pointers and sizes, no torch / C++ types.  All pointers are DEVICE pointers unless the
 * name ends in _host; `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).
 * Every function returns 0 on success, a negative DDN_E* code on a contract violation and a
 * positive cudaError_t when the CUDA runtime reports one; ddn_last_error() gives the text.
 * Nothing here allocates device memory: the caller owns every buffer (workspace sizes are
 * queried first) -- the host side above this boundary uses torch only as the allocator.
 *
 * The reference has no native code on this path (SURVEY.md 2c); each entry point replaces the
 * PyTorch-1.1 -> ATen -> cuDNN call sequence of the reference Python cited next to it
 * (paths relative to the reference root; PSD = external/pytorch-segmentation-detection).
 */
#ifndef DDN_B200_H_
#define DDN_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DDN_ABI_VERSION 3

enum {
  DDN_OK = 0,
  DDN_EINVAL = -1,     /* bad shape / flag / null pointer            */
  DDN_EWORKSPACE = -2, /* workspace too small                         */
  DDN_EUNSUPPORTED = -3
};

/* Arithmetic used by the convolution contractions. */
enum {
  DDN_PRECISION_FP32_SIMT = 0, /* fp32 FFMA on CUDA cores (bit-for-bit class of the fp32 oracle)        */
  DDN_PRECISION_BF16X3 = 1,    /* wgmma, operands split hi+lo bf16, 3 MMAs, fp32 accumulate            */
  DDN_PRECISION_BF16 = 2       /* wgmma, single bf16 pass ("fast mode"; fails the 1e-3 descriptor gate)   */
};

int ddn_abi_version(void);
/* Data-parallel hosts: leave `n` SMs (0..64; default 0, or $DDN_RESERVED_SMS) free of the persistent tensor-core kernels so that a
 * concurrent collective (the NCCL all-reduce a ddn_grad_bucket_fn callback starts inside ddn_resnet34_8s_backward) has SMs to run on.
 * No reference counterpart: the reference is single-GPU (dense_correspondence/training/training.py:254-256). */
int ddn_set_reserved_sms(int n);
const char* ddn_last_error(void);

/* ------------------------------------------------------------------------------------------
 * Parameter layout of Resnet34_8s(num_classes=D)
 *   PSD/pytorch_segmentation_detection/models/resnet_dilated.py:283-322
 *   PSD/vision/torchvision/models/resnet.py:112-229 (names, shapes, order of named_parameters())
 * Learnable parameters live in ONE flat fp32 array, BatchNorm running statistics in a second one;
 * entry i of the tables gives the reference state-dict key (without the leading "resnet34_8s."),
 * its shape and its element offset in the flat array.
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  char name[64];
  int32_t ndim;
  int32_t shape[4];
  int64_t offset; /* elements */
  int64_t numel;
} ddn_tensor_entry;

/* Fills up to `cap` entries, returns the number of learnable tensors (110). */
int ddn_resnet34_8s_param_table(int D, ddn_tensor_entry* out, int cap);
/* Running mean / running var entries (72 = 36 BN x 2), same convention. */
int ddn_resnet34_8s_buffer_table(ddn_tensor_entry* out, int cap);
int64_t ddn_resnet34_8s_param_count(int D);
int64_t ddn_resnet34_8s_buffer_count(void);

/* ------------------------------------------------------------------------------------------
 * Backbone forward / backward.
 *   forward  replaces Resnet34_8s.forward            (resnet_dilated.py:310-322)
 *                     ResNet.forward / BasicBlock    (resnet.py:231-265, :53-69)
 *            as called by DenseCorrespondenceNetwork.forward
 *                     (dense_correspondence/network/dense_correspondence_network.py:239-263)
 *   backward replaces the autograd backward of the same (dense_correspondence/training/training.py:345)
 *
 * x  [B,3,H,W] fp32 NCHW (already mean/std normalised), y [B,D,H,W] fp32 NCHW contiguous.
 * H, W multiples of 8 (the trunk runs at H/8 x W/8).  1 <= D <= 32.
 * mode DDN_MODE_TRAIN: BatchNorm uses the statistics of THIS call's images (biased variance) and updates
 *   running_mean/var in `buffers` with `momentum` and the unbiased variance, exactly like
 *   nn.BatchNorm2d in train(); the activations needed by backward are kept in `workspace`.
 * mode DDN_MODE_INFER: BatchNorm uses `buffers` (folded into the conv epilogues); nothing is kept.
 * mode DDN_MODE_EVAL_SAVE: BatchNorm uses `buffers` (frozen statistics) and the activations are kept, so that
 *   ddn_resnet34_8s_backward can differentiate an eval()-mode network like autograd does for the reference.
 * bn_groups G (1 or 2): the batch is G consecutive groups of B/G images, each normalised by its OWN batch
 *   statistics -- G = 2 runs the reference's two forward calls of a step (image A batch, image B batch:
 *   dense_correspondence/training/training.py:329-333) as one launch sequence; running statistics are updated
 *   group 0 first, then group 1, as the two calls would.
 * The same `workspace` (untouched in between) must be handed to ddn_resnet34_8s_backward (same mode / bn_groups),
 * which OVERWRITES grads[0 .. param_count) with dL/dparams for the cotangent dy [B,D,H,W].
 * on_bucket (may be NULL) is called on the HOST, in order, each time a contiguous range of `grads` is final --
 *   i.e. right after the last kernel writing grads[offset, offset+numel) has been enqueued on `stream` -- so that a
 *   data-parallel caller can start the all-reduce of that range while the rest of the backward still runs
 *   (4 ranges, last layers first; ddn_resnet34_8s_grad_buckets lists them).
 * ------------------------------------------------------------------------------------------ */
enum { DDN_MODE_INFER = 0, DDN_MODE_TRAIN = 1, DDN_MODE_EVAL_SAVE = 2 };

size_t ddn_resnet34_8s_workspace_bytes(int B, int H, int W, int D, int mode, int precision);

int ddn_resnet34_8s_forward(const float* x, const float* params, float* buffers, float* y,
                            void* workspace, size_t workspace_bytes,
                            int B, int H, int W, int D,
                            int mode, int bn_groups, float momentum, float eps, int precision,
                            float* low_nhwc_out /* optional [B, H/8*W/8, D]: the low-resolution descriptor map y is upsampled from */,
                            void* stream);

typedef void (*ddn_grad_bucket_fn)(void* user, int bucket, int64_t offset, int64_t numel);

/* dy [B,D,H,W] and / or dlow_nhwc [B, H/8*W/8, D] (the cotangent of low_nhwc_out, produced by the loss kernels that are fused
 * with the upsample): either may be NULL, not both. */
int ddn_resnet34_8s_backward(const float* dy, const float* dlow_nhwc, const float* params, float* grads,
                             void* workspace, size_t workspace_bytes,
                             int B, int H, int W, int D, int mode, int bn_groups, float eps, int precision,
                             ddn_grad_bucket_fn on_bucket, void* user, void* stream);

/* offsets[0..3] = first element of gradient bucket 0..3 (in completion order), offsets[4] = param_count; returns 4.
 * Bucket i covers [offsets[i], offsets[i-1]) for i > 0 and [offsets[0], param_count) for i = 0. */
int ddn_resnet34_8s_grad_buckets(int D, int64_t* offsets, int cap);

/* Optional cache of the tensor-core weight packs (bf16 hi/lo, forward and data-gradient layouts of every conv).
 * The caller owns `cache` (ddn_resnet34_8s_weight_cache_bytes(D) bytes of device memory) and bumps `version` whenever the
 * parameter array changed (optimizer step, load_state_dict); forward/backward calls made with the same `params` pointer and
 * `precision` then pack each conv once per version instead of once per call.  cache == NULL switches it off. */
size_t ddn_resnet34_8s_weight_cache_bytes(int D);
int ddn_resnet34_8s_set_weight_cache(void* cache, size_t bytes, const float* params, uint64_t version, int precision);

/* ------------------------------------------------------------------------------------------
 * The same entry points for a backbone chosen by id, as the reference picks it by name
 * (dense_correspondence/network/dense_correspondence_network.py:360-383):
 *   DDN_ARCH_RESNET34_8S  Resnet34_8s, BasicBlock [3, 4, 6, 3]   (the ddn_resnet34_8s_* functions above)
 *   DDN_ARCH_RESNET50_8S  Resnet50_8s, Bottleneck [3, 4, 6, 3], 2048-channel trunk, fc = Conv2d(2048, D, 1)
 *                         (PSD/pytorch_segmentation_detection/models/resnet_dilated.py:399-435, resnet.py:72-109)
 * Arguments and results are those of the ddn_resnet34_8s_* function of the same suffix; table names are the state-dict keys
 * without the leading "resnet50_8s." (320 entries: 161 learnable tensors, 106 running statistics, 53 num_batches_tracked).
 * An unknown arch returns DDN_EINVAL (0 from the size queries).  ddn_resnet34_8s_set_weight_cache serves every architecture.
 * ------------------------------------------------------------------------------------------ */
enum { DDN_ARCH_RESNET34_8S = 0, DDN_ARCH_RESNET50_8S = 1 };

int ddn_net_param_table(int arch, int D, ddn_tensor_entry* out, int cap);
int ddn_net_buffer_table(int arch, ddn_tensor_entry* out, int cap);
int64_t ddn_net_param_count(int arch, int D);
int64_t ddn_net_buffer_count(int arch);
size_t ddn_net_workspace_bytes(int arch, int B, int H, int W, int D, int mode, int precision);
int ddn_net_forward(int arch, const float* x, const float* params, float* buffers, float* y,
                    void* workspace, size_t workspace_bytes,
                    int B, int H, int W, int D,
                    int mode, int bn_groups, float momentum, float eps, int precision,
                    float* low_nhwc_out, void* stream);
int ddn_net_backward(int arch, const float* dy, const float* dlow_nhwc, const float* params, float* grads,
                     void* workspace, size_t workspace_bytes,
                     int B, int H, int W, int D, int mode, int bn_groups, float eps, int precision,
                     ddn_grad_bucket_fn on_bucket, void* user, void* stream);
/* 4 buckets for both architectures: layer4 + fc, layer3, layer2, layer1 + stem. */
int ddn_net_grad_buckets(int arch, int D, int64_t* offsets, int cap);

/* The three calls above with a `flags` argument (0 = exactly the calls above).
 *   DDN_NET_UNIT_DESCRIPTORS: y is written with unit-length descriptors, y[:, p] = x / ||x|| for the bilinear upsample x of
 *   every pixel p -- the reference's `normalize` option (dense_correspondence/network/dense_correspondence_network.py:256-259)
 *   applied to each image on its own.  low_nhwc_out stays the un-normalised map.  The backward then takes dy through the
 *   normalisation's Jacobian (dy - y (y.dy)) / ||x|| before the upsample's adjoint; dlow_nhwc is added as it is (the loss
 *   kernels with DDN_LOWRES_UNIT already applied the Jacobian).  No epsilon: a pixel whose upsampled descriptor is zero gets
 *   NaN, as x / ||x|| does in fp32.  Forward and backward of one step take the same flags, and the workspace is sized by
 *   ddn_net_workspace_bytes_v2 with them (a backward with the flag needs B*D*H*W more floats). */
enum { DDN_NET_UNIT_DESCRIPTORS = 1 };
size_t ddn_net_workspace_bytes_v2(int arch, int B, int H, int W, int D, int mode, int precision, int flags);
int ddn_net_forward_v2(int arch, const float* x, const float* params, float* buffers, float* y,
                       void* workspace, size_t workspace_bytes,
                       int B, int H, int W, int D,
                       int mode, int bn_groups, float momentum, float eps, int precision,
                       float* low_nhwc_out, int flags, void* stream);
int ddn_net_backward_v2(int arch, const float* dy, const float* dlow_nhwc, const float* params, float* grads,
                        void* workspace, size_t workspace_bytes,
                        int B, int H, int W, int D, int mode, int bn_groups, float eps, int precision, int flags,
                        ddn_grad_bucket_fn on_bucket, void* user, void* stream);
size_t ddn_net_weight_cache_bytes(int arch, int D);

/* ------------------------------------------------------------------------------------------
 * Pixelwise contrastive loss.
 * Descriptor images are addressed with explicit strides so the reference's strided view
 *   process_network_output: [N,D,H,W].view(N,D,W*H).permute(0,2,1)
 *   (dense_correspondence_network.py:303-319)
 * is consumed in place: element (image b, pixel p, channel c) = base[b*stride_b + p*stride_p + c*stride_c].
 *
 * A "term" is one list of index pairs scored one way:
 *   kind DDN_TERM_MATCH    sum_i ||A[a_i]-B[b_i]||^2                 pixelwise_contrastive_loss.py:131-167
 *   kind DDN_TERM_HINGE    sum_j max(0, M-||A[a_j]-B[b_j]||)^2       :170-213, :271-304
 *   kind DDN_TERM_HINGE_INV    max(0, ||.||-M)^2   (invert=True)     :204-208
 *   flag DDN_TERM_PIXEL_WEIGHT multiplies l_j by min(||uv(gt_b[j/k]) - uv(b_j)||, M_pixel)/M_pixel,
 *        k = n / n_gt                                                :215-269, :307-352
 * Per (image pair, term) the forward produces the fp64 sum and the number of non-zero hinge
 * values ("hard negatives", :210-211) without any host synchronisation.
 * ------------------------------------------------------------------------------------------ */
enum { DDN_TERM_MATCH = 0, DDN_TERM_HINGE = 1, DDN_TERM_HINGE_INV = 2 };
enum { DDN_TERM_PIXEL_WEIGHT = 1 };

typedef struct {
  const int64_t* idx_a; /* [B, n] flat pixel indices into image A (n = u + W*v)                */
  const int64_t* idx_b; /* [B, n]                                                               */
  const int64_t* gt_b;  /* [B, n_gt] matches_b, only read when DDN_TERM_PIXEL_WEIGHT is set      */
  int64_t n;
  int64_t n_gt;
  int32_t kind;
  int32_t flags;
  float margin;  /* M_descriptor of this term */
  float m_pixel; /* M_pixel                   */
  /* Ragged batches (real SpartanDataset samples have a different number of matches per pair: num_matching_attempts is
   * only an upper bound, dense_correspondence/dataset/spartan_dataset_masked.py:652-660,841-858): rows are padded to n
   * (n_gt) with -1 and len[b] (len_gt[b]) gives pair b's true count.  DEVICE pointers [B], NULL = every pair has n (n_gt). */
  const int64_t* len;
  const int64_t* len_gt;
} ddn_loss_term;

#define DDN_MAX_TERMS 8

/* sums  [B, n_terms] fp64, counts [B, n_terms] int64 (both written, not accumulated). */
int ddn_contrastive_terms_forward(const float* pred_a, const float* pred_b,
                                  int64_t stride_b, int64_t stride_p, int64_t stride_c,
                                  int B, int64_t P, int D, int image_width,
                                  const ddn_loss_term* terms_host, int n_terms,
                                  double* sums, int64_t* counts, void* stream);

/* dpred_a/b += sum_t coef[b,t] * d(term_t sum of pair b)/dpred   (scatter-add; caller zero-fills).
 * coef [B, n_terms] fp32 lives on the device so the scale 1/max(#hard,1) never visits the host. */
int ddn_contrastive_terms_backward(const float* pred_a, const float* pred_b,
                                   int64_t stride_b, int64_t stride_p, int64_t stride_c,
                                   int B, int64_t P, int D, int image_width,
                                   const ddn_loss_term* terms_host, int n_terms,
                                   const float* coef, const float* upstream /* device scalar or NULL */,
                                   float* dpred_a, float* dpred_b, void* stream);

/* The same two entry points FUSED WITH THE BILINEAR UPSAMPLE that produced the descriptor images
 * (nn.functional.upsample_bilinear, resnet_dilated.py:320): low_a / low_b [B, h*w, D] are the low-resolution maps
 * (`low_nhwc_out` of ddn_resnet34_8s_forward), index tensors still address the H x W image.  Each descriptor is blended from
 * its 4 low-resolution cells (identical fp32 arithmetic to ddn_upsample_bilinear_forward), so sums / counts equal those of
 * the entry points above on the upsampled image; the backward scatters into d(low) [B, h*w, D] (caller zero-fills), which
 * ddn_resnet34_8s_backward takes as `dlow_nhwc` -- the full-resolution image and its gradient are never touched.  The scatter
 * accumulates in fp64 so that its result does not depend on the order in which pairs arrive: `scratch` = 2 * B*h*w*D doubles
 * (any contents; 16-byte aligned) holds that accumulator, which is then added to dlow_a / dlow_b. */
int ddn_contrastive_terms_forward_lowres(const float* low_a, const float* low_b, int B, int h, int w, int H, int W, int D,
                                         const ddn_loss_term* terms_host, int n_terms,
                                         double* sums, int64_t* counts, void* stream);
int ddn_contrastive_terms_backward_lowres(const float* low_a, const float* low_b, int B, int h, int w, int H, int W, int D,
                                          const ddn_loss_term* terms_host, int n_terms,
                                          const float* coef, const float* upstream,
                                          float* dlow_a, float* dlow_b, double* scratch, void* stream);

/* The same two with a `flags` argument (0 = exactly the calls above).
 *   DDN_LOWRES_UNIT: every sampled descriptor is the blend x normalised to unit length, y = x / ||x|| (the images are the
 *   DDN_NET_UNIT_DESCRIPTORS output of the network), in every term kind; the backward applies (g - y (y.g)) / ||x|| to each
 *   side's gradient before the scatter.  A zero blend gives NaN descriptors (no epsilon). */
enum { DDN_LOWRES_UNIT = 1 };
int ddn_contrastive_terms_forward_lowres_v2(const float* low_a, const float* low_b, int B, int h, int w, int H, int W, int D,
                                            const ddn_loss_term* terms_host, int n_terms,
                                            double* sums, int64_t* counts, int flags, void* stream);
int ddn_contrastive_terms_backward_lowres_v2(const float* low_a, const float* low_b, int B, int h, int w, int H, int W, int D,
                                             const ddn_loss_term* terms_host, int n_terms,
                                             const float* coef, const float* upstream,
                                             float* dlow_a, float* dlow_b, double* scratch, int flags, void* stream);

/* loss_composer.get_within_scene_loss (dense_correspondence/loss_functions/loss_composer.py:70-143)
 * evaluated on the device from the sums/counts of terms ordered {match, masked, background[, blind]}:
 *   five [5] fp32 = (loss, match_loss, masked_scaled, background_scaled, blind_scaled), mean over B pairs
 *   coef [B, n_terms] fp32 = d(loss)/d(term sum) for the backward above (already divided by B, times upstream). */
typedef struct {
  float match_loss_weight;
  float non_match_loss_weight;
  int32_t scale_by_hard_negatives;
  int32_t has_blind;
  int64_t n_match, n_masked, n_background, n_blind;
  /* ragged batches: per-pair true counts, DEVICE pointers [B] (NULL = the n_* above for every pair) */
  const int64_t* len_match; const int64_t* len_masked; const int64_t* len_background; const int64_t* len_blind;
} ddn_within_scene_cfg;

int ddn_within_scene_compose(const double* sums, const int64_t* counts, int B, int n_terms,
                             const ddn_within_scene_cfg* cfg_host, float* five, float* coef, void* stream);

/* loss_composer.get_loss for a batch whose pairs have different SpartanDatasetDataType values: every pair gets its own
 * type's formula, evaluated on the device from the sums/counts of the five terms
 *   {match, masked, background, blind@M_masked, blind@M_background}
 * (the last two read the same blind index tensors; the caller routes them with per-pair lengths: term 3 gets the blind
 * count of the within-scene-type pairs and 0 for the others, term 4 the reverse).
 *   SINGLE_OBJECT_WITHIN_SCENE, MULTI_OBJECT, SYNTHETIC_MULTI_OBJECT: get_within_scene_loss (loss_composer.py:70-143),
 *     exactly as ddn_within_scene_compose with the blind term; the blind term is reported, never optimised.
 *   DIFFERENT_OBJECT: get_different_object_loss (:168-191): blind = sum / max(#hard, 1) (scale_by_hard_negatives_
 *     DIFFERENT_OBJECT) or sum / max(len_blind, 1); the pair's five values are (blind, 0, 0, 0, blind).
 * pair_type [B] int32 DEVICE array; types are validated by the caller (SINGLE_OBJECT_ACROSS_SCENE has no loss upstream).
 * five [5] fp32 = mean over B of the per-pair five values, summed in fp64 in a fixed order;
 * coef [B, 5] fp32 = d(loss)/d(term sum), already divided by B.  n_terms must be 5. */
typedef struct {
  float match_loss_weight;
  float non_match_loss_weight;
  int32_t scale_by_hard_negatives;
  int32_t scale_by_hard_negatives_different_object;
  int64_t n_match, n_masked, n_background, n_blind;
  /* per-pair true counts, DEVICE pointers [B] (NULL = the n_* above for every pair); len_blind is the unrouted blind count */
  const int64_t* len_match; const int64_t* len_masked; const int64_t* len_background; const int64_t* len_blind;
} ddn_pair_type_cfg;

int ddn_pair_type_compose(const double* sums, const int64_t* counts, int B, int n_terms, const ddn_pair_type_cfg* cfg_host,
                          const int32_t* pair_type, float* five, float* coef, void* stream);

/* ------------------------------------------------------------------------------------------
 * Host-buffer entry point (pageable or pinned host memory in, host memory out); it stages through
 * device memory it allocates itself and synchronises before returning.
 * ddn_within_scene_loss_host == loss_composer.get_loss(...) for SINGLE_OBJECT_WITHIN_SCENE on
 * descriptor images held on the host; used by the C smoke test and INTEGRATION.md's ctypes stub.
 * ------------------------------------------------------------------------------------------ */
int ddn_within_scene_loss_host(const float* pred_a_host, const float* pred_b_host, /* [B,D,H*W] NCHW */
                               int B, int H, int W, int D,
                               const int64_t* matches_a_host, const int64_t* matches_b_host, int64_t n_match,
                               const int64_t* masked_a_host, const int64_t* masked_b_host, int64_t n_masked,
                               const int64_t* background_a_host, const int64_t* background_b_host, int64_t n_background,
                               float m_masked, float m_background,
                               float match_loss_weight, float non_match_loss_weight, int scale_by_hard_negatives,
                               float* five_host /* [5] */);

/* ------------------------------------------------------------------------------------------
 * Single-operator entry points (unit tests, and the building blocks the two network calls use).
 * Activations are NHWC fp32 inside the library; conv weights arrive in the reference's
 * [Cout, Cin, kh, kw] layout and are repacked on the device.
 * ------------------------------------------------------------------------------------------ */
/* y[N,Ho,Wo,Cout] = conv2d(x[N,H,W,Cin], w[Cout,Cin,k,k], stride, pad, dilation), no bias -- nn.Conv2d (resnet.py:36,136,210) */
int ddn_conv2d_forward(const float* x_nhwc, const float* w_oihw, float* y_nhwc,
                       int N, int H, int W, int Cin, int Cout, int k, int stride, int pad, int dil,
                       int precision, void* workspace, size_t workspace_bytes, void* stream);
size_t ddn_conv2d_workspace_bytes(int N, int H, int W, int Cin, int Cout, int k, int stride, int pad, int dil, int precision);
/* dx (may be NULL) and dw[Cout,Cin,k,k] (overwritten) for the cotangent dy[N,Ho,Wo,Cout]. */
int ddn_conv2d_backward(const float* x_nhwc, const float* w_oihw, const float* dy_nhwc,
                        float* dx_nhwc, float* dw_oihw,
                        int N, int H, int W, int Cin, int Cout, int k, int stride, int pad, int dil,
                        int precision, void* workspace, size_t workspace_bytes, void* stream);

/* Training-mode BatchNorm2d + optional residual + optional ReLU on NHWC (resnet.py:57-67):
 *   y = relu?( (x-mean)/sqrt(var+eps)*gamma + beta + residual? ); mean/var of this batch (biased);
 *   save_mean/save_invstd [C] written; running stats updated when running_mean != NULL. */
int ddn_batchnorm_forward(const float* x, const float* gamma, const float* beta, const float* residual,
                          float* y, float* save_mean, float* save_invstd,
                          float* running_mean, float* running_var,
                          int64_t M, int C, int relu, int training, float momentum, float eps,
                          void* workspace, size_t workspace_bytes, void* stream);
/* g = dy * (y>0 if relu); dx, dgamma, dbeta; d_residual (= g, may be NULL). */
int ddn_batchnorm_backward(const float* dy, const float* x, const float* y, const float* gamma,
                           const float* save_mean, const float* save_invstd,
                           float* dx, float* dgamma, float* dbeta, float* d_residual,
                           int64_t M, int C, int relu, void* workspace, size_t workspace_bytes, void* stream);
/* 0 for a C the BatchNorm kernels do not take: they need 4 <= C <= 1024 with 256 % (C/4) == 0, or a multiple of 1024 up to 4096. */
size_t ddn_batchnorm_workspace_bytes(int64_t M, int C);

/* Tensor-core convolutions with the fused epilogues the network runs (resnet.py:53-69 conv -> BatchNorm -> [+ residual] -> ReLU),
 * one operator at a time.  precision BF16X3 or BF16 only (FP32_SIMT has no fused epilogues: DDN_EUNSUPPORTED), shapes as
 * ddn_conv2d_forward's tensor-core path; every argument is checked before anything is launched.  bn_groups G (1 or 2, dividing N):
 * images [g*N/G, (g+1)*N/G) form BatchNorm group g.  One workspace query serves all three. */
size_t ddn_conv2d_fused_workspace_bytes(int N, int H, int W, int Cin, int Cout, int k, int stride, int pad, int dil, int precision);
/* Training forward: raw[N,Ho,Wo,Cout] = conv2d(x, w) and the batch statistics of raw per group, mean / invstd [G][Cout]
 * (biased variance, invstd = 1/sqrt(var+eps)); running_mean / running_var [Cout] (both or neither) are updated group 0 first,
 * then group 1, with `momentum` and the unbiased variance, like nn.BatchNorm2d in train().
 * Cin = 3, k = 7, stride 2, pad 3 is the stem (resnet.py:127): x is then NCHW [N,3,H,W], the network's input layout, and the
 * conv runs as the 7x7/2 patch GEMM. */
int ddn_conv2d_bn_stats_forward(const float* x_nhwc, const float* w_oihw, float* raw_nhwc, float* mean, float* invstd,
                                float* running_mean, float* running_var,
                                int N, int H, int W, int Cin, int Cout, int k, int stride, int pad, int dil,
                                int bn_groups, float momentum, float eps, int precision,
                                void* workspace, size_t workspace_bytes, void* stream);
/* Inference forward, eval-mode BatchNorm folded in: y = relu?(conv2d(x, w) * scale + shift + addend), scale = gamma /
 * sqrt(running_var + eps), shift = beta - running_mean * scale; addend [N,Ho,Wo,Cout] fp32 may be NULL.  Outputs (at least one):
 * fp32 y, and / or the bf16 operand planes y_hi = bf16(y), y_lo = bf16(y - y_hi) (y_lo written in BF16X3 only; may be NULL). */
int ddn_conv2d_folded_forward(const float* x_nhwc, const float* w_oihw, const float* gamma, const float* beta,
                              const float* running_mean, const float* running_var, const float* addend_nhwc,
                              float* y_nhwc, void* y_hi_bf16, void* y_lo_bf16,
                              int N, int H, int W, int Cin, int Cout, int k, int stride, int pad, int dil, int relu, float eps,
                              int precision, void* workspace, size_t workspace_bytes, void* stream);
/* Data gradient dx[N,H,W,Cin] = conv2d_input(dy[N,Ho,Wo,Cout], w) + addend (may be NULL), together with the column sums of the
 * BatchNorm backward that consumes dx: that BatchNorm's output is y = relu(bn(raw) [+ residual]) with raw [N,H,W,Cin] and
 * mean / invstd [G][Cin]; g = dx * (y > 0), the mask read from the bf16 hi plane of y (y_hi, blocks with a residual) or, when
 * y_hi is NULL, recomputed from raw, gamma and beta.  sums [G][2][Cin] = (sum g, sum g * xhat) per group, dbeta = sum over
 * groups of sum g, dgamma = of sum g * xhat. */
int ddn_conv2d_backward_data_bn_stats(const float* w_oihw, const float* dy_nhwc, const float* addend_nhwc,
                                      const float* raw_nhwc, const float* mean, const float* invstd, const float* gamma,
                                      const float* beta, const void* y_hi_bf16,
                                      float* dx_nhwc, float* dgamma, float* dbeta, float* sums,
                                      int N, int H, int W, int Cin, int Cout, int k, int stride, int pad, int dil,
                                      int bn_groups, int precision, void* workspace, size_t workspace_bytes, void* stream);

/* The stem after conv1 (resnet.py:231-235: bn1 -> ReLU -> max-pool 3x3/2 pad 1), one operator at a time, with the kernels and the
 * wiring the network runs.  raw [N,Hc,Wc,64] is conv1's output, mean / invstd [G][64] bn1's statistics per BatchNorm group
 * (G = 1 or 2 dividing N: image n is in group n / (N/G)), gamma / beta [64]; Hp = (Hc-1)/2+1, Wp = (Wc-1)/2+1.
 * Every argument is checked before anything is launched.
 * Forward: y [N,Hp,Wp,64] = maxpool(relu(bn(raw))) as fp32 y and / or the bf16 planes y_hi = bf16(y), y_lo = bf16(y - y_hi)
 * (y_lo may be NULL; the network writes it in BF16X3 only); argmax [N,Hp,Wp,64] uint8 = the window-local r*3+s of the first
 * maximum in row-major scan order (a window whose every element is 0 after the ReLU: its first in-bounds element). */
int ddn_stem_pool_forward(const float* raw, const float* mean, const float* invstd, const float* gamma, const float* beta,
                          float* y, void* y_hi_bf16, void* y_lo_bf16, void* argmax_u8, int N, int Hc, int Wc, int G, void* stream);
/* Backward of the whole stem for the image x [N,3,H,W] (NCHW), Hc = (H-1)/2+1, Wc = (W-1)/2+1: dy_pool [N,Hp,Wp,64] -> the pool /
 * ReLU backward g = scatter(dy_pool, argmax) * (bn(raw) > 0) -> bn1's backward (`training`: batch statistics; else frozen ones,
 * dx = gamma * invstd * g) -> dgamma, dbeta [64] and dw_conv1 [64,3,7,7] (overwritten).  BF16X3 / BF16: the weight gradient
 * runs on the tensor cores over the 7x7/2 patch planes of x and the bf16 planes of d raw; FP32_SIMT: the fp32 CUDA-core
 * kernels over the NHWC4 image.  Optional outputs (NULL: not written): g_out and dx_bn [N,Hc,Wc,64] (the fp32 d raw), and on
 * the tensor cores the bf16 planes of d raw the weight gradient reads, dx_hi = bf16(dx) and (BF16X3 only) dx_lo = bf16(dx - dx_hi). */
size_t ddn_stem_workspace_bytes(int N, int H, int W, int precision);
int ddn_stem_backward(const float* x_nchw, const float* raw, const float* mean, const float* invstd, const float* gamma,
                      const float* beta, const void* argmax_u8, const float* dy_pool, float* g_out, float* dx_bn,
                      void* dx_hi_bf16, void* dx_lo_bf16, float* dgamma, float* dbeta, float* dw_conv1,
                      int N, int H, int W, int G, int training, int precision, void* workspace, size_t workspace_bytes, void* stream);

/* Bilinear align_corners=True resize of planar maps [N*C, h, w] -> [N*C, H, W]
 * (nn.functional.upsample_bilinear, resnet_dilated.py:320) and its adjoint. */
int ddn_upsample_bilinear_forward(const float* x, float* y, int NC, int h, int w, int H, int W, void* stream);
int ddn_upsample_bilinear_backward(const float* dy, float* dx, int NC, int h, int w, int H, int W, void* stream);
/* The same resize of N images of D maps [N, D, h, w] -> [N, D, H, W] with every output pixel's D-vector normalised to unit
 * length (y = x / ||x||, the network's DDN_NET_UNIT_DESCRIPTORS output; 1 <= D <= 32; a zero vector gives NaN), and its
 * adjoint: dx [N, D, h, w] = upsample^T((dy - y (y.dy)) / ||x||), with `scratch` N*D*H*W floats for the middle term. */
int ddn_upsample_bilinear_unit_forward(const float* x, float* y, int N, int D, int h, int w, int H, int W, void* stream);
int ddn_upsample_bilinear_unit_backward(const float* x, const float* dy, float* dx, float* scratch, int N, int D, int h, int w,
                                        int H, int W, void* stream);

/* The scoring layer fc = nn.Conv2d(C, D, 1) with bias (resnet_dilated.py:298 for C = 512, :414 for C = 2048) on the trunk's
 * channels-last features, and its backward.  feat [N*Mimg, C] fp32, or its bf16 operand planes (feat = hi + lo; feat_lo may be
 * NULL: hi alone) -- exactly one of the two; w [D, C], bias [D]; low / dlow [N, D, Mimg] (the planar map the upsample reads);
 * low_nhwc (optional) [N*Mimg, D].  1 <= D <= 32, C a multiple of 512; feat, feat_hi, feat_lo and dfeat 16-byte aligned.
 * The backward overwrites dfeat [N*Mimg, C], dw [D, C] and dbias [D]; its workspace (ddn_fc_workspace_bytes, 0 for an
 * unsupported C, D) holds per-slot partial sums that are added in a fixed order, so the result is the same on every run.
 * Every argument is checked before anything is launched. */
size_t ddn_fc_workspace_bytes(int C, int D);
int ddn_fc_forward(const float* feat, const void* feat_hi_bf16, const void* feat_lo_bf16, const float* w, const float* bias,
                   float* low, float* low_nhwc, int64_t Mimg, int N, int C, int D, void* stream);
int ddn_fc_backward(const float* dlow, const float* feat, const void* feat_hi_bf16, const void* feat_lo_bf16, const float* w,
                    float* dfeat, float* dw, float* dbias, int64_t Mimg, int N, int C, int D,
                    void* workspace, size_t workspace_bytes, void* stream);

/* Data-parallel helpers on the flat gradient: g *= scale (after an all-reduce SUM over ranks). */
int ddn_scale_inplace(float* g, int64_t n, float scale, void* stream);

/* Batched best-match search: for each of Q query descriptors [Q,D] find the pixel of the descriptor image res_b
 * (element (p, c) at p*stride_p + c*stride_c, p = u + W*v) with the smallest L2 distance -- the device-side equivalent of
 * DenseCorrespondenceNetwork.find_best_match (dense_correspondence/network/dense_correspondence_network.py:488-525), first
 * minimum on ties like numpy.argmin.  best_uv [Q,2] int64 = (u, v), best_diff [Q] = that distance; norm_diffs (optional)
 * [Q, H*W] = the full distance maps.  mask_b (optional, [H*W] fp32, 1 inside / 0 outside the object mask): additionally
 * the best match restricted to the mask, argmin(norm_diffs + (1 - mask_b) * 1e6) like
 * dense_correspondence/evaluation/evaluation.py:1052-1059 -> best_uv_masked [Q,2], best_diff_masked [Q] (the masked
 * minimum itself, +1e6 outside).  scratch: 2 x Q x 8 bytes. */
int ddn_find_best_match(const float* res_b, int64_t stride_p, int64_t stride_c, int H, int W, int D,
                        const float* queries, int Q, int64_t* best_uv, float* best_diff, float* norm_diffs,
                        const float* mask_b, int64_t* best_uv_masked, float* best_diff_masked,
                        void* scratch, void* stream);

/* Per-match evaluation statistics == DenseCorrespondenceEvaluation.compute_descriptor_match_statistics
 * (dense_correspondence/evaluation/evaluation.py:1006-1178) for Q ground-truth matches over N image pairs in one call,
 * with no host synchronisation.  Query i belongs to pair[i] (int64 [Q], 0 <= pair < N); uv_a [Q,2], uv_b [Q,2] int64 (u, v)
 * pixels, uv_b already clipped and rounded as clip_pixel_to_image_size_and_round (evaluation.py:603-607) does it.
 *   res_a, res_b   descriptor images [N,H,W,D] fp32, element (n, v, u, c) at n*s[0] + v*s[1] + u*s[2] + c*s[3] with the
 *                  strides strides_*_host[4] (elements), e.g. the permuted view forward_single_image_tensor returns; 1 <= D <= 32
 *   mask_b         [N,H,W] fp32, 1 on the object, 0 elsewhere (the dataset's uint8 mask)
 *   depth_a/b      [N,H,W] fp32 raw sensor units (millimetres; divided by DEPTH_IM_SCALE = 1000.0 in float64)
 *   K_inv_host     [9] row-major HOST double: inv(K) as pinhole_projection_image_to_world computes it (numpy.linalg.inv,
 *                  dense_correspondence/correspondence_tools/correspondence_finder.py:123-144)
 *   poses_*_host   [N,16] row-major HOST doubles, camera-to-world; copied into `scratch` before this returns
 * nd(p) = sqrt(sum_c (res_b[p,c] - res_a[uv_a,c])^2) is computed in fp32 exactly as numpy does it on a contiguous float32
 * array (find_best_match, dense_correspondence/network/dense_correspondence_network.py:488-525): squares rounded, numpy's
 * pairwise summation order.  The threshold t = nd(uv_b) uses the same arithmetic; the reference computes it with
 * np.linalg.norm (a BLAS dot, evaluation.py:1070), which may differ from it in the last bits.  The masked distance
 * nd + (1 - mask_b) * 1e6, its comparison with t and its minimum are float64, as in the reference (evaluation.py:1053-1058).
 * Outputs, one row per query (column indices DDN_MS_* below):
 *   out_f32 [Q, DDN_MS_NF32], out_f64 [Q, DDN_MS_NF64], out_i64 [Q, DDN_MS_NI64]
 * A query whose pair index or pixels lie outside [0,N) x image gets NaN in every float column and -1 in every integer
 * column, and is counted in *bad_queries (DEVICE int64, overwritten); so is a query whose masked distances are all NaN
 * (NaN descriptors), which has no masked minimum.  An empty mask_b gives a NaN masked fraction (the
 * reference divides by an integer 0).  Per-block partial sums are added in a fixed order: a second call is bit-identical.
 * scratch: ddn_match_statistics_scratch_bytes(N, H, W, Q) bytes (0 for sizes outside the limits below). */
#define DDN_MS_MAX_PAIRS 65535
#define DDN_MS_MAX_QUERIES (1 << 22)
enum { DDN_MS_NORM_DIFF_DESCRIPTOR_GROUND_TRUTH = 0, DDN_MS_NORM_DIFF_DESCRIPTOR = 1, DDN_MS_NF32 = 2 };
enum {
  DDN_MS_NORM_DIFF_DESCRIPTOR_MASKED = 0,
  DDN_MS_NORM_DIFF_GROUND_TRUTH_3D = 1,
  DDN_MS_NORM_DIFF_PRED_3D = 2,
  DDN_MS_NORM_DIFF_PRED_3D_MASKED = 3,
  DDN_MS_PIXEL_MATCH_ERROR_L2 = 4,
  DDN_MS_PIXEL_MATCH_ERROR_L2_MASKED = 5,
  DDN_MS_PIXEL_MATCH_ERROR_L1 = 6,
  DDN_MS_FRACTION_CLOSER = 7,                 /* fraction_pixels_closer_than_ground_truth            */
  DDN_MS_FRACTION_CLOSER_MASKED = 8,          /* fraction_pixels_closer_than_ground_truth_masked     */
  DDN_MS_AVERAGE_L2_FALSE_POSITIVES = 9,      /* average_l2_distance_for_false_positives             */
  DDN_MS_AVERAGE_L2_FALSE_POSITIVES_MASKED = 10,
  DDN_MS_NF64 = 11
};
enum {
  DDN_MS_IS_VALID = 0,
  DDN_MS_IS_VALID_MASKED = 1,
  DDN_MS_U_PRED = 2, DDN_MS_V_PRED = 3,                 /* best match (first minimum of nd)              */
  DDN_MS_U_PRED_MASKED = 4, DDN_MS_V_PRED_MASKED = 5,   /* masked best match                             */
  DDN_MS_NUM_CLOSER = 6, DDN_MS_NUM_CLOSER_MASKED = 7,  /* pixels with nd < t, with masked nd < t        */
  DDN_MS_NUM_MASK_PIXELS = 8,                           /* nonzero pixels of mask_b                      */
  DDN_MS_NI64 = 9
};
size_t ddn_match_statistics_scratch_bytes(int N, int H, int W, int64_t Q);
int ddn_match_statistics(const float* res_a, const int64_t* strides_a_host, const float* res_b, const int64_t* strides_b_host,
                         int N, int H, int W, int D, const int64_t* pair, const int64_t* uv_a, const int64_t* uv_b, int64_t Q,
                         const float* mask_b, const float* depth_a, const float* depth_b,
                         const double* K_inv_host, const double* poses_a_host, const double* poses_b_host,
                         float* out_f32, double* out_f64, int64_t* out_i64, int64_t* bad_queries,
                         void* scratch, size_t scratch_bytes, void* stream);

/* Best match of Q query pixels over N image pairs in one launch: the across-object analysis
 * (compute_descriptor_match_statistics_no_ground_truth, dense_correspondence/evaluation/evaluation.py:977-1004), i.e.
 * find_best_match (dense_correspondence_network.py:488-525) of uv_a[q] in res_a[pair[q]] against all of res_b[pair[q]].
 *   res_a/b, strides_*_host, N, H, W, D   as ddn_match_statistics (1 <= D <= 32, element strides over (n, h, w, c))
 *   pair [Q] int64, uv_a [Q,2] int64 (u, v)   DEVICE
 * Outputs: best_uv [Q,2] int64 (u, v) and best_diff [Q] float32, the distance nd at it, computed as ddn_match_statistics
 * computes nd (bit-equal to numpy on a contiguous array); ties go to the first pixel in row-major order (np.argmin).  A
 * query whose pair or uv_a is out of range gets (-1, -1) and NaN and is counted in *bad_queries (DEVICE int64,
 * overwritten).  The result does not depend on the order in which blocks run: a second call is bit-identical.
 * scratch: ddn_best_match_batch_scratch_bytes(Q) bytes (0 for Q outside 1..DDN_BM_MAX_QUERIES). */
#define DDN_BM_MAX_QUERIES (65535 * 8)
size_t ddn_best_match_batch_scratch_bytes(int64_t Q);
int ddn_best_match_batch(const float* res_a, const int64_t* strides_a_host, const float* res_b, const int64_t* strides_b_host,
                         int N, int H, int W, int D, const int64_t* pair, const int64_t* uv_a, int64_t Q,
                         int64_t* best_uv, float* best_diff, int64_t* bad_queries, void* scratch, size_t scratch_bytes,
                         void* stream);

/* Per-image, per-channel descriptor statistics in one launch: the body of compute_descriptor_statistics
 * (dense_correspondence/evaluation/evaluation.py:2177-2219) for N images at once.
 *   res            N descriptor images, element (n, h, w, c) at res[n*s[0] + h*s[1] + w*s[2] + c*s[3]] with
 *                  s = strides_host [4] (HOST int64, elements): the NCHW network output and the [H,W,D] view of
 *                  forward_single_image_tensor both work without a copy.  1 <= D <= 32.
 *   mask           [N,H,W] contiguous DEVICE, DDN_DS_MASK_F32 (float32) or DDN_DS_MASK_U8 (uint8); nonzero = object.
 * Outputs (DEVICE): out_stats [N, DDN_DS_NSTATS, D] float32 in the order of DDN_DS_* below; out_count [N] int64, the
 * nonzero mask pixels.  min / max propagate NaN as torch.min / torch.max do; means are fp64 sums over the pixels (per
 * block, then the blocks in a fixed order by the image's last block), divided by the count and rounded once to float32,
 * so a second call is bit-identical.  An empty mask gives count 0 and NaN mask statistics; nothing is raised.
 * scratch: ddn_descriptor_statistics_scratch_bytes(N, H, W, D) bytes (0 for sizes outside the limits). */
enum { DDN_DS_MASK_F32 = 0, DDN_DS_MASK_U8 = 1 };
enum { DDN_DS_MIN = 0, DDN_DS_MAX = 1, DDN_DS_MEAN = 2, DDN_DS_MASK_MIN = 3, DDN_DS_MASK_MAX = 4, DDN_DS_MASK_MEAN = 5,
       DDN_DS_NSTATS = 6 };
#define DDN_DS_MAX_IMAGES 65535
size_t ddn_descriptor_statistics_scratch_bytes(int N, int H, int W, int D);
int ddn_descriptor_statistics(const float* res, const int64_t* strides_host, int N, int H, int W, int D, const void* mask,
                              int mask_dtype, float* out_stats, int64_t* out_count, void* scratch, size_t scratch_bytes,
                              void* stream);

/* Non-match sampling on the device: out_b[j] = flat index (u + W*v) of a pixel drawn uniformly from the nonzero pixels of
 * `mask` [H*W] fp32 (nz[floor(rand_u[j] * #nonzero)], nonzero pixels in ascending order) or, when mask is NULL or empty,
 * from the whole image (floor(rand_u*W), floor(rand_v*H)); out_a[j] = matches_a[j / non_matches_per_match] (may be NULL).
 * == create_non_correspondences (dense_correspondence/correspondence_tools/correspondence_finder.py:276-405, whose
 * "too close" perturbation is a no-op upstream) + create_non_matches / flatten_uv_tensor
 * (dense_correspondence/dataset/spartan_dataset_masked.py:841-858,1255-1264), given the same uniform numbers. */
size_t ddn_sample_non_matches_scratch_bytes(int H, int W);
int ddn_sample_non_matches(const float* mask, int H, int W, const float* rand_u, const float* rand_v, int64_t n,
                           const int64_t* matches_a, int64_t non_matches_per_match, int64_t* out_a, int64_t* out_b,
                           void* scratch, size_t scratch_bytes, void* stream);

/* Pinhole reprojection match finder for candidate pixels of image A == batch_find_pixel_correspondences
 * (dense_correspondence/correspondence_tools/correspondence_finder.py:409-619): zero-depth, field-of-view and occlusion
 * (3 mm margin) pruning, survivors in candidate order.  depth_* are fp32 [H*W] device arrays in raw sensor units
 * (millimetres, DEPTH_IM_SCALE = 1000); K [9], pose_a [16], pose_b [16] are row-major HOST doubles (camera-to-world poses).
 * out_a / out_b [n] int64 flat pixels (u + W*v; b truncated like .long()), out_u2 / out_v2 optional sub-pixel positions in B;
 * *out_count (DEVICE int64) = number of survivors. */
size_t ddn_find_pixel_correspondences_scratch_bytes(int64_t n);
int ddn_find_pixel_correspondences(const float* depth_a, const float* depth_b, int H, int W,
                                   const int64_t* candidates, int64_t n,
                                   const double* K_host, const double* pose_a_host, const double* pose_b_host,
                                   int64_t* out_a, int64_t* out_b, float* out_u2, float* out_v2, int64_t* out_count,
                                   void* scratch, size_t scratch_bytes, void* stream);

/* Within-scene training batch on the device == SpartanDataset.get_within_scene_data
 * (dense_correspondence/dataset/spartan_dataset_masked.py:646-769, SINGLE_OBJECT_WITHIN_SCENE, debug off) for B image pairs
 * at once, with every random number given as an input.  Per pair: candidates in A (from mask_a when
 * sample_matches_only_off_mask, else uniform), reprojection into B (as ddn_find_pixel_correspondences), background domain
 * randomisation of A then B (correspondence_augmentation.py:86-214, exact uint8 arithmetic), the 180-degree flip of A and B
 * with their index lists, masked / background non-matches from the flipped mask_b, blind non-matches, and
 * ToTensor + Normalize into fp32 NCHW.  A pair whose mask_a is empty while sampling on the mask is the reference's
 * return_empty_data: both images are the normalised, un-augmented image A and every count is 0.
 * Index outputs are [B, cap] int64 padded with -1 past the pair's count: cap = n_attempts (matches),
 * n_attempts * k_masked, n_attempts * k_background, H * W (blind).  counts [B, 4] int64 (matches, masked, background, blind)
 * and empty [B] uint8 are DEVICE outputs: nothing is read back, and the number of launches does not depend on B.
 * Every device array is dense in the layout given below; K [9], poses [B * 16] are row-major HOST doubles. */
#define DDN_WS_MAX_PAIRS 128          /* per-pair matrices travel as kernel parameters (168 bytes each) */
enum { DDN_WS_RANDOMIZE = 0, DDN_WS_GRADIENT, DDN_WS_VERTICAL, DDN_WS_NOISE, DDN_WS_FLIP, DDN_WS_RGB1, DDN_WS_RGB2 = 8,
       DDN_WS_PARAM_BYTES = 16 };    /* byte offsets in one image's parameter block */
typedef struct {
  int32_t B, H, W;
  int32_t sample_matches_only_off_mask, domain_randomize, use_image_b_mask_inv;
  int64_t n_attempts, k_masked, k_background;
  float mean[3], std[3];              /* Normalize, per channel */
} ddn_ws_batch_cfg;
typedef struct {
  /* [B, 2, DDN_WS_PARAM_BYTES] uint8, image A then B: decisions (0 / 1) at DDN_WS_RANDOMIZE..DDN_WS_FLIP, colours
   * rgb1 / rgb2 (0..254) at DDN_WS_RGB1 / DDN_WS_RGB2; the solid background uses rgb1 */
  const uint8_t* params;
  const uint8_t* noise;               /* [B, 2 (image), 2 (N1, N2), H, W, 3] uint8: background + N1 - N2 */
  const float *cand_u, *cand_v;       /* [B, n_attempts] uniform [0, 1) */
  const float *masked_u, *masked_v;   /* [B, n_attempts * k_masked] */
  const float *background_u, *background_v;  /* [B, n_attempts * k_background] */
  const float* blind;                 /* [B, H * W] */
} ddn_ws_batch_rand;
typedef struct {
  float *image_a, *image_b;           /* [B, 3, H, W] */
  int64_t *matches_a, *matches_b, *masked_a, *masked_b, *background_a, *background_b, *blind_a, *blind_b;
  int64_t* counts;                    /* [B, 4] */
  uint8_t* empty;                     /* [B] */
} ddn_ws_batch_out;
size_t ddn_within_scene_batch_scratch_bytes(const ddn_ws_batch_cfg* cfg);   /* 0 for a refused cfg */
int ddn_within_scene_batch(const ddn_ws_batch_cfg* cfg, const uint8_t* rgb_a, const uint8_t* rgb_b,
                           const uint8_t* mask_a, const uint8_t* mask_b, const float* depth_a, const float* depth_b,
                           const double* K_host, const double* poses_a_host, const double* poses_b_host,
                           const ddn_ws_batch_rand* rand, const ddn_ws_batch_out* out,
                           void* scratch, size_t scratch_bytes, void* stream);

/* Across-scene training batch on the device == SpartanDataset.get_across_scene_data
 * (dense_correspondence/dataset/spartan_dataset_masked.py:1056-1141, debug off), the producer of DIFFERENT_OBJECT and
 * SINGLE_OBJECT_ACROSS_SCENE pairs, for B image pairs at once with every random number given as an input.  Per pair:
 * num_samples blind pixels drawn with replacement from the nonzero pixels of mask_a and of mask_b
 * (random_sample_from_masked_image_torch, correspondence_finder.py:92-121), background domain randomisation of A then B
 * (as ddn_within_scene_batch, same parameter blocks and noise layout), the 180-degree flip of A and B with their blind
 * pixels (p -> P-1-p), and ToTensor + Normalize into fp32 NCHW.  A pair whose mask_a or mask_b is empty is the
 * reference's return_empty_data: both images are the normalised, un-augmented image A, every count is 0 and the blind
 * rows are -1.  blind_a / blind_b are [B, num_samples] int64; counts [B, 4] int64 (0, 0, 0, blind) and empty [B] uint8 are
 * DEVICE outputs: nothing is read back, and a call is 5 launches whatever B.  Every array is a dense device array. */
#define DDN_AS_MAX_PAIRS 16384        /* 2 * B compaction rows on the grid's y dimension */
typedef struct {
  int32_t B, H, W;
  int32_t domain_randomize;
  int64_t num_samples;                /* training.cross_scene_num_samples, >= 1 */
  float mean[3], std[3];              /* Normalize, per channel */
} ddn_as_batch_cfg;
typedef struct {
  const uint8_t* params;              /* [B, 2, DDN_WS_PARAM_BYTES] uint8, as ddn_ws_batch_rand.params */
  const uint8_t* noise;               /* [B, 2, 2, H, W, 3] uint8, as ddn_ws_batch_rand.noise */
  const float *blind_a, *blind_b;     /* [B, num_samples] uniform [0, 1): the draws over mask_a, mask_b */
} ddn_as_batch_rand;
typedef struct {
  float *image_a, *image_b;           /* [B, 3, H, W] */
  int64_t *blind_a, *blind_b;         /* [B, num_samples] */
  int64_t* counts;                    /* [B, 4] */
  uint8_t* empty;                     /* [B] */
} ddn_as_batch_out;
size_t ddn_across_scene_batch_scratch_bytes(const ddn_as_batch_cfg* cfg);   /* 0 for a refused cfg */
int ddn_across_scene_batch(const ddn_as_batch_cfg* cfg, const uint8_t* rgb_a, const uint8_t* rgb_b,
                           const uint8_t* mask_a, const uint8_t* mask_b, const ddn_as_batch_rand* rand,
                           const ddn_as_batch_out* out, void* scratch, size_t scratch_bytes, void* stream);

/* Synthetic multi-object training batch on the device == SpartanDataset.get_synthetic_multi_object_within_scene_data
 * (dense_correspondence/dataset/spartan_dataset_masked.py:890-1053, SYNTHETIC_MULTI_OBJECT, debug off) for B pairs at
 * once, with every random number given as an input.  A pair has two within-scene halves, scene A (images a1, a2) and scene
 * B (b1, b2); every image input is stacked [B, 2 (scene A, scene B), ...].  Per half: candidates in image 1 (from mask_1 when
 * sample_matches_only_off_mask, else uniform) and their reprojection into image 2 (as ddn_within_scene_batch, no background
 * randomisation, no flip); the sub-pixel positions in image 2 are truncated (.long()).  Merge 1 of a1 and b1 and merge 2 of
 * a2 and b2 (correspondence_augmentation.py:217-347), each with its own foreground decision: fg * m + (1 - m) * bg in uint8
 * arithmetic modulo 256; the background half keeps the matches whose image-1 (merge 1) / image-2 (merge 2) pixel is off
 * the foreground's mask.  matches = scene A's survivors then scene B's; masked / background non-matches from merged mask 2
 * = clip(fg_mask_2 + bg_mask_2, 0, 1) with the uint8 sum wrapping.  There are no blind non-matches.  The reference's four
 * early returns (mask_a1 empty: a1 twice; mask_b1 empty, or a background half fully occluded by merge 1 or 2: b1 twice)
 * give the normalised image twice, every count 0 and empty = 1.
 * Index outputs are [B, cap] int64 padded with -1: cap = 2 * n_attempts (matches), 2 * n_attempts * k_masked,
 * 2 * n_attempts * k_background, 1 (blind, always -1).  counts [B, 4] (matches, masked, background, 0) and empty [B] are
 * DEVICE outputs; a call is 15 launches whatever B.  K [9] and poses [B * 2 * 16] (image 1 / image 2 of row 2 * pair + half)
 * are row-major HOST doubles. */
#define DDN_SMO_MAX_PAIRS (DDN_WS_MAX_PAIRS / 2)   /* two reprojection matrix sets per pair travel as kernel parameters */
typedef struct {
  int32_t B, H, W;
  int32_t sample_matches_only_off_mask, use_image_b_mask_inv;
  int64_t n_attempts, k_masked, k_background;
  float mean[3], std[3];              /* Normalize, per channel */
} ddn_smo_batch_cfg;
typedef struct {
  const uint8_t* merge;               /* [B, 2] uint8: 1 = merge 1 / merge 2 puts scene B in the foreground */
  const float *cand_u, *cand_v;       /* [B, 2 (half), n_attempts] uniform [0, 1) */
  const float *masked_u, *masked_v;   /* [B, 2 * n_attempts * k_masked] */
  const float *background_u, *background_v;  /* [B, 2 * n_attempts * k_background] */
} ddn_smo_batch_rand;
typedef struct {
  float *image_a, *image_b;           /* [B, 3, H, W]: merged image 1, merged image 2 */
  int64_t *matches_a, *matches_b, *masked_a, *masked_b, *background_a, *background_b, *blind_a, *blind_b;
  int64_t* counts;                    /* [B, 4] */
  uint8_t* empty;                     /* [B] */
} ddn_smo_batch_out;
size_t ddn_synthetic_multi_object_batch_scratch_bytes(const ddn_smo_batch_cfg* cfg);   /* 0 for a refused cfg */
int ddn_synthetic_multi_object_batch(const ddn_smo_batch_cfg* cfg, const uint8_t* rgb_1, const uint8_t* rgb_2,
                                     const uint8_t* mask_1, const uint8_t* mask_2, const float* depth_1, const float* depth_2,
                                     const double* K_host, const double* poses_1_host, const double* poses_2_host,
                                     const ddn_smo_batch_rand* rand, const ddn_smo_batch_out* out,
                                     void* scratch, size_t scratch_bytes, void* stream);

/* Device-resident training frames (pdc_b200.frames.FrameStore): one launch gathers, for B pairs, frames idx_a[b] and
 * idx_b[b] of a store of F frames of H x W -- rgb uint8 [F, H, W, 3], depth uint16 [F, H, W] (millimetres), mask uint8
 * [F, H, W], contiguous -- into the producers' inputs: rgb_a / rgb_b uint8 [B, H, W, 3] and mask_a / mask_b uint8 [B, H, W]
 * copied, depth_a / depth_b float32 [B, H, W] converted exactly (both null: no depth; across-scene pairs need none).
 * The store may be in device memory or in pinned host memory (read through UVA, zero-copy); outputs are device memory.
 * idx_a_host / idx_b_host are host arrays of B int32 in [0, F); they travel as kernel parameters, so the call neither copies
 * nor synchronises.  B in [1, DDN_FRAMES_MAX_PAIRS]; every argument is checked before the launch. */
#define DDN_FRAMES_MAX_PAIRS 128
int ddn_frames_gather(const uint8_t* rgb, const uint16_t* depth, const uint8_t* mask, int64_t F, int H, int W,
                      const int32_t* idx_a_host, const int32_t* idx_b_host, int B, uint8_t* rgb_a, uint8_t* rgb_b,
                      float* depth_a, float* depth_b, uint8_t* mask_a, uint8_t* mask_b, void* stream);

/* Fused Adam step over flat arrays == torch.optim.Adam(lr, betas, eps, weight_decay) as used by
 * dense_correspondence/training/training.py:133-145,346 (L2 weight decay folded into the gradient, bias-corrected moments,
 * no amsgrad).  `step` is the 1-based step count; grads are read as grads[i]*grad_scale (1/world after a SUM all-reduce). */
int ddn_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n, int64_t step,
                  float lr, float beta1, float beta2, float eps, float weight_decay, float grad_scale, void* stream);

/* Per-kernel-class device timing (CUDA events recorded on the launching stream around each launch of the
 * convolution / loss kernels while enabled).  ddn_profile_read synchronises on the recorded events and
 * fills one entry per class that ran: work = algorithmic FLOPs (conv_*) or bytes (loss_*). */
typedef struct {
  char name[32];
  int64_t launches;
  double ms;
  double work;
} ddn_profile_entry;
int ddn_profile_enable(int on);
int ddn_profile_reset(void);
int ddn_profile_read(ddn_profile_entry* out, int cap);

/* Number of kernels this library has launched since load (bench.py's gpu_launches). */
int64_t ddn_kernel_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* DDN_B200_H_ */
