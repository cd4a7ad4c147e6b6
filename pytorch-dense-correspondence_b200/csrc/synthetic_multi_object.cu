// Synthetic multi-object training batches on the device: SpartanDataset.get_synthetic_multi_object_within_scene_data
// (dense_correspondence/dataset/spartan_dataset_masked.py:890-1053) for B pairs in one call, given its random numbers.
// Contract and layouts: include/ddn_b200.h (ddn_synthetic_multi_object_batch).
//
// Each pair has two within-scene halves (row r = 2 * pair + half; half 0 = scene A: images a1, a2; half 1 = scene B: b1, b2),
// which run as 2B rows through the within-scene kernels.  Launches (15, whatever B):  compact mask_1 (3)  ->  candidates (1)
// ->  reprojection (1)  ->  compact the survivors of merge 1 and of merge 2 (3)  ->  gather (1)  ->  merged images and merged
// mask 2 (1)  ->  compact merged mask 2 (!= 0, != 1) (3)  ->  masked, background (2).
#include "sampling.cuh"

namespace ddn {

// A candidate j of row r = 2b + h survives merge 1 unless its half is merge 1's background and its image-1 pixel lies on the
// foreground's mask_1; it survives merge 2 unless, in addition, its half is merge 2's background and its image-2 pixel lies
// on the foreground's mask_2 (prune_matches_if_occluded, correspondence_augmentation.py:291-333; merge 2 receives the pairs
// swapped, spartan_dataset_masked.py:944-949).  merge[b, i] = 1: merge i + 1 puts scene B in the foreground.
// Compaction row q = 2r + stage (stage 0: survivors of merge 1, stage 1: of merge 2).
struct SmoSurvive {
  const float* flag; const int64_t* cand; const int64_t* b_flat; const uint8_t* mask_1; const uint8_t* mask_2;
  const uint8_t* merge; int64_t n, P;
  __device__ __forceinline__ bool operator()(int64_t q, int64_t j) const {
    const int64_t r = q >> 1, b = r >> 1; const int h = (int)(r & 1), stage = (int)(q & 1);
    if (flag[r * n + j] == 0.f) return false;
    const int64_t fg = 2 * b + (1 - h);                     // the other half's masks are the foreground's
    const bool bg1 = (merge[2 * b] != 0) == (h == 0);
    if (bg1 && mask_1[fg * P + cand[r * n + j]] != 0) return false;
    if (stage == 0) return true;
    const bool bg2 = (merge[2 * b + 1] != 0) == (h == 0);
    return !(bg2 && mask_2[fg * P + b_flat[r * n + j]] != 0);
  }
};

// Which of the reference's returns pair b takes: 0 the merged batch; 1 return_empty_data with a1 twice (no candidate in
// mask_a1, :913-916); 2 with b1 twice (no candidate in mask_b1, :922-925, or a background half fully occluded by merge 1
// or merge 2, :938-941, :951-954).
struct SmoStatus {
  const int* total_1; int64_t total_stride;        // mask_1 totals of row 2b + h; NULL when the candidates are uniform
  const int* surv; int64_t surv_stride; int nblk;   // survivor totals of compaction row 2(2b + h) + stage
  const uint8_t* merge;
  __device__ __forceinline__ int operator()(int64_t b) const {
    if (total_1 && total_1[(2 * b) * total_stride] == 0) return 1;
    if (total_1 && total_1[(2 * b + 1) * total_stride] == 0) return 2;
    const int64_t h1 = merge[2 * b] ? 0 : 1, h2 = merge[2 * b + 1] ? 0 : 1;   // background halves of merge 1, 2
    if (surv[(2 * (2 * b + h1) + 0) * surv_stride + nblk] == 0) return 2;
    if (surv[(2 * (2 * b + h2) + 1) * surv_stride + nblk] == 0) return 2;
    return 0;
  }
};

struct SmoGather {
  SmoStatus st; const int* nz; const int64_t* cand; const int64_t* b_flat; int64_t n;
  int64_t* out_a; int64_t* out_b; int64_t* counts; uint8_t* empty; int64_t* blind_a; int64_t* blind_b;
};

// matches_a = flat(cat(uv_a1, uv_b1)), matches_b = flat(cat(uv_a2, uv_b2)) over the survivors of merge 2 (merge_matches,
// correspondence_augmentation.py:335-347), padded with -1 to 2 * n_attempts; blind rows [B, 1] = -1 (empty_tensor())
__global__ void __launch_bounds__(SAMP_THREADS)
smo_gather_kernel(const SmoGather g) {
  pdl_prologue();
  const int64_t b = blockIdx.y, n = g.n;
  const int status = g.st(b);
  const int LA = status ? 0 : g.st.surv[(2 * (2 * b) + 1) * g.st.surv_stride + g.st.nblk];
  const int L = status ? 0 : LA + g.st.surv[(2 * (2 * b + 1) + 1) * g.st.surv_stride + g.st.nblk];
  if (blockIdx.x == 0 && threadIdx.x < 4) {
    g.counts[b * 4 + threadIdx.x] = threadIdx.x == 0 ? L : 0;
    if (threadIdx.x == 0) { g.empty[b] = status ? 1 : 0; g.blind_a[b] = -1; g.blind_b[b] = -1; }
  }
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < 2 * n; i += (int64_t)gridDim.x * blockDim.x) {
    if (i >= L) { g.out_a[b * 2 * n + i] = -1; g.out_b[b * 2 * n + i] = -1; continue; }
    const int64_t r = 2 * b + (i < LA ? 0 : 1);
    const int j = g.nz[(2 * r + 1) * n + (i < LA ? i : i - LA)];
    g.out_a[b * 2 * n + i] = g.cand[r * n + j]; g.out_b[b * 2 * n + i] = g.b_flat[r * n + j];
  }
}

struct SmoMergeArgs {
  SmoStatus st; const uint8_t* rgb_1; const uint8_t* rgb_2; const uint8_t* mask_1; const uint8_t* mask_2;
  float* image_a; float* image_b; uint8_t* mmask_2; float mean[3], std[3]; int B; int64_t P;
};

// One thread per pixel of merged image 1 or 2 of a pair (merge_images_with_occlusions, correspondence_augmentation.py:
// 217-288): fg * m + (1 - m) * bg in uint8 arithmetic modulo 256 with the foreground's mask m, then ToTensor + Normalize.
// Merged mask 2 = clip(fg_mask_2 + bg_mask_2, 0, 1) with the uint8 sum wrapping.  An early return writes a1 or b1 twice.
__global__ void __launch_bounds__(256)
smo_merge_kernel(const SmoMergeArgs a) {
  pdl_prologue();
  const int64_t P = a.P, total = 2 * (int64_t)a.B * P;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = t / P, p = t - row * P, b = row >> 1;
    const int img = (int)(row & 1);                               // 0: merged image 1, 1: merged image 2
    const int status = a.st(b);
    const uint8_t* rgb = img ? a.rgb_2 : a.rgb_1; const uint8_t* mask = img ? a.mask_2 : a.mask_1;
    const int64_t fg = 2 * b + (a.st.merge[2 * b + img] ? 1 : 0), bg = 4 * b + 1 - fg;
    int v[3];
    if (status) {
      const uint8_t* s = a.rgb_1 + ((2 * b + (status == 2 ? 1 : 0)) * P + p) * 3;
      v[0] = s[0]; v[1] = s[1]; v[2] = s[2];
    } else {
      const int m = mask[fg * P + p];
      const uint8_t* f = rgb + (fg * P + p) * 3; const uint8_t* k = rgb + (bg * P + p) * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) v[c] = (f[c] * m + ((1 - m) & 255) * k[c]) & 255;
      if (img) a.mmask_2[b * P + p] = ((mask[fg * P + p] + mask[bg * P + p]) & 255) != 0;
    }
    if (status && img) a.mmask_2[b * P + p] = 0;
    float* out = (img ? a.image_b : a.image_a) + b * 3 * P + p;
#pragma unroll
    for (int c = 0; c < 3; ++c) out[c * P] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)v[c], 255.f), a.mean[c]), a.std[c]);
  }
}

// row 2b + set over merged mask 2 (values 0 / 1): set 0 != 0 (masked non-matches), set 1: 1 - m != 0 (background)
struct SmoSets {
  const uint8_t* m; int64_t P;
  __device__ __forceinline__ bool operator()(int64_t r, int64_t p) const {
    const uint8_t v = m[(r >> 1) * P + p];
    return (r & 1) ? v != 1 : v != 0;
  }
};

struct SmoScratch {
  int *counts_1, *nz_1, *counts_s, *nz_s, *counts_m, *nz_m;
  uint8_t* mmask_2;
  int64_t *cand, *b_flat;
  float *flag, *u2, *v2;
  size_t bytes;
};

static SmoScratch smo_layout(const ddn_smo_batch_cfg& c, char* base) {
  const int64_t R = 2 * (int64_t)c.B, P = (int64_t)c.H * c.W, n = c.n_attempts;
  const int64_t csP = compact_counts_stride(P), csN = compact_counts_stride(n);
  SmoScratch s;
  size_t off = 0;
  auto take = [&](size_t bytes) { char* p = base ? base + off : nullptr; off += align_up(bytes, 256); return p; };
  s.counts_1 = (int*)take(sizeof(int) * R * csP); s.nz_1 = (int*)take(sizeof(int) * R * P);
  s.cand = (int64_t*)take(8 * R * n); s.flag = (float*)take(4 * R * n); s.b_flat = (int64_t*)take(8 * R * n);
  s.u2 = (float*)take(4 * R * n); s.v2 = (float*)take(4 * R * n);
  s.counts_s = (int*)take(sizeof(int) * 2 * R * csN); s.nz_s = (int*)take(sizeof(int) * 2 * R * n);
  s.mmask_2 = (uint8_t*)take(c.B * P);
  s.counts_m = (int*)take(sizeof(int) * R * csP); s.nz_m = (int*)take(sizeof(int) * R * P);
  s.bytes = off + 256;
  return s;
}

static bool smo_cfg_ok(const ddn_smo_batch_cfg* c) {
  if (!c) return false;
  auto flag = [](int32_t v) { return v == 0 || v == 1; };
  const int64_t P = (int64_t)c->H * c->W;
  const int64_t kmax = c->k_masked > c->k_background ? c->k_masked : c->k_background;
  bool ok = flag(c->sample_matches_only_off_mask) && flag(c->use_image_b_mask_inv) && c->B >= 1 && c->B <= DDN_SMO_MAX_PAIRS &&
            c->H >= 1 && c->W >= 1 && P < (1ll << 30) && c->n_attempts >= 1 && c->n_attempts < (1ll << 29) &&
            c->k_masked >= 0 && c->k_background >= 0 && kmax <= (1ll << 29) / c->n_attempts;
  for (int i = 0; i < 3; ++i) ok = ok && c->std[i] != 0.f && c->std[i] == c->std[i] && c->mean[i] == c->mean[i];
  return ok;
}

}  // namespace ddn

using namespace ddn;

extern "C" size_t ddn_synthetic_multi_object_batch_scratch_bytes(const ddn_smo_batch_cfg* cfg) {
  if (!smo_cfg_ok(cfg)) return 0;
  return smo_layout(*cfg, nullptr).bytes;
}

extern "C" int ddn_synthetic_multi_object_batch(const ddn_smo_batch_cfg* cfg, const uint8_t* rgb_1, const uint8_t* rgb_2,
                                                const uint8_t* mask_1, const uint8_t* mask_2, const float* depth_1,
                                                const float* depth_2, const double* K_host, const double* poses_1_host,
                                                const double* poses_2_host, const ddn_smo_batch_rand* rand,
                                                const ddn_smo_batch_out* out, void* scratch, size_t scratch_bytes, void* stream) {
  DDN_CHECK_ARG(smo_cfg_ok(cfg), "bad synthetic multi-object configuration (B in [1, %d], H, W, n_attempts >= 1, k >= 0, "
                "flags 0/1, std != 0)", DDN_SMO_MAX_PAIRS);
  const ddn_smo_batch_cfg c = *cfg;
  const int B = c.B, H = c.H, W = c.W, R = 2 * B;
  const int64_t P = (int64_t)H * W, n = c.n_attempts, cap_m = 2 * n * c.k_masked, cap_b = 2 * n * c.k_background;
  DDN_CHECK_ARG(rgb_1 && rgb_2 && mask_1 && mask_2 && depth_1 && depth_2 && K_host && poses_1_host && poses_2_host && rand && out,
                "null argument");
  DDN_CHECK_ARG(rand->merge && rand->cand_u && rand->cand_v && (cap_m == 0 || (rand->masked_u && rand->masked_v)) &&
                (cap_b == 0 || (rand->background_u && rand->background_v)), "null random-number array");
  DDN_CHECK_ARG(out->image_a && out->image_b && out->matches_a && out->matches_b && out->blind_a && out->blind_b && out->counts &&
                out->empty && (cap_m == 0 || (out->masked_a && out->masked_b)) &&
                (cap_b == 0 || (out->background_a && out->background_b)), "null output array");
  DDN_CHECK_ARG(scratch && scratch_bytes >= smo_layout(c, nullptr).bytes, "scratch too small");
  ReprojBatch<DDN_WS_MAX_PAIRS> mats;
  for (int r = 0; r < R; ++r)
    DDN_CHECK_ARG(reproj_mats(K_host, poses_1_host + 16 * r, poses_2_host + 16 * r, mats.m[r]), "singular intrinsics");

  cudaStream_t st = (cudaStream_t)stream;
  const SmoScratch s = smo_layout(c, reinterpret_cast<char*>(align_up(reinterpret_cast<uintptr_t>(scratch), 256)));
  const int nblkP = (int)ceil_div(P, SAMP_PER_BLOCK), nblkN = (int)ceil_div(n, SAMP_PER_BLOCK);
  const int64_t csP = compact_counts_stride(P), csN = compact_counts_stride(n);
  const int wide = num_sms() * 8;
  auto blocks = [&](int64_t items) { return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(items, SAMP_THREADS), wide)); };

  // 1. candidates of both halves: from mask_a1 / mask_b1 (whose totals mark the first two early returns) or uniform
  const CompactRows c1 = {s.counts_1, s.nz_1, csP, P, nblkP};
  DDN_TRY(compact_rows(NonzeroU8{mask_1, P}, P, R, c1, st));
  SampleRows sc = {};
  if (c.sample_matches_only_off_mask) { sc.nz = s.nz_1; sc.counts = s.counts_1; sc.nz_stride = P; sc.counts_stride = csP; sc.nblk = nblkP; }
  sc.ru = rand->cand_u; sc.rv = rand->cand_v; sc.r_stride = n; sc.n = n; sc.k = 1;
  sc.out_b = s.cand; sc.out_stride = n; sc.H = H; sc.W = W;
  DDN_LAUNCH(sample_non_matches_kernel, dim3(blocks(n), R), SAMP_THREADS, 0, st, sc);

  // 2. reprojection image 1 -> image 2 of each half, then the survivors of the two merges' occlusion pruning
  DDN_LAUNCH(reproject_kernel<DDN_WS_MAX_PAIRS>, dim3(blocks(n), R), SAMP_THREADS, 0, st, depth_1, depth_2, s.cand, n, H, W, mats,
             s.flag, s.b_flat, s.u2, s.v2);
  const CompactRows cs = {s.counts_s, s.nz_s, csN, n, nblkN};
  DDN_TRY(compact_rows(SmoSurvive{s.flag, s.cand, s.b_flat, mask_1, mask_2, rand->merge, n, P}, n, 2 * R, cs, st));
  const SmoStatus status = {c.sample_matches_only_off_mask ? s.counts_1 + nblkP : nullptr, csP, s.counts_s, csN, nblkN, rand->merge};

  // 3. merged matches, counts[:, 0], empty, blind rows
  const SmoGather g = {status, s.nz_s, s.cand, s.b_flat, n, out->matches_a, out->matches_b, out->counts, out->empty,
                       out->blind_a, out->blind_b};
  DDN_LAUNCH(smo_gather_kernel, dim3(blocks(2 * n), B), SAMP_THREADS, 0, st, g);

  // 4. merged images and merged mask 2
  const SmoMergeArgs mg = {status, rgb_1, rgb_2, mask_1, mask_2, out->image_a, out->image_b, s.mmask_2,
                           {c.mean[0], c.mean[1], c.mean[2]}, {c.std[0], c.std[1], c.std[2]}, B, P};
  DDN_LAUNCH(smo_merge_kernel, blocks(2 * B * P), 256, 0, st, mg);

  // 5. masked and background non-matches from merged mask 2 (create_non_correspondences + create_non_matches)
  const CompactRows cm = {s.counts_m, s.nz_m, csP, P, nblkP};
  DDN_TRY(compact_rows(SmoSets{s.mmask_2, P}, P, R, cm, st));
  for (int set = 0; set < 2; ++set) {
    const bool masked = set == 0;
    SampleRows sn = {};
    if (masked || c.use_image_b_mask_inv) {
      sn.nz = s.nz_m + set * P; sn.counts = s.counts_m + set * csP; sn.nz_stride = 2 * P; sn.counts_stride = 2 * csP; sn.nblk = nblkP;
    }
    sn.ru = masked ? rand->masked_u : rand->background_u; sn.rv = masked ? rand->masked_v : rand->background_v;
    sn.r_stride = masked ? cap_m : cap_b;
    sn.n_dev = out->counts; sn.n_stride = 4; sn.k = masked ? c.k_masked : c.k_background;
    sn.matches_a = out->matches_a; sn.ma_stride = 2 * n;
    sn.out_a = masked ? out->masked_a : out->background_a; sn.out_b = masked ? out->masked_b : out->background_b;
    sn.out_stride = sn.r_stride; sn.pad_to = sn.r_stride;
    sn.count_out = out->counts + 1 + set; sn.count_stride = 4; sn.H = H; sn.W = W;
    DDN_LAUNCH(sample_non_matches_kernel, dim3(blocks(sn.r_stride), B), SAMP_THREADS, 0, st, sn);
  }
  return 0;
}
