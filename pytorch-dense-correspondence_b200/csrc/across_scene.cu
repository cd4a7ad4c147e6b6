// Across-scene training batches on the device: SpartanDataset.get_across_scene_data
// (dense_correspondence/dataset/spartan_dataset_masked.py:1056-1141), which both get_different_object_data (:874-888) and
// get_single_object_across_scene_data (:860-872) return, for B image pairs in one call, given its random numbers.
// Contract and layouts: include/ddn_b200.h (ddn_across_scene_batch).
//
// Launches (5, whatever B):  compact mask_a and mask_b (3)  ->  augment + flip + normalise (1)  ->  blind pixels (1).
#include "sampling.cuh"

namespace ddn {

// row 2*pair: mask_a != 0, row 2*pair + 1: mask_b != 0
struct NonzeroU8Pair {
  const uint8_t* a; const uint8_t* b; int64_t P;
  __device__ __forceinline__ bool operator()(int64_t r, int64_t p) const { return ((r & 1) ? b : a)[(r >> 1) * P + p] != 0; }
};

struct AcrossBlindArgs {
  const int* nz; const int* counts; int64_t counts_stride; int nblk;   // rows 2*pair (mask_a), 2*pair + 1 (mask_b)
  const float* ra; const float* rb; const uint8_t* params;
  int64_t* out_a; int64_t* out_b; int64_t* counts_out; uint8_t* empty; int64_t n, P;
};

// blind_uv_a / blind_uv_b (spartan_dataset_masked.py:1087-1092), flipped with their images (:1102-1104) and flattened
// (:1119-1120); a pair with an empty mask is return_empty_data (:1094-1096): count 0, rows -1
__global__ void __launch_bounds__(SAMP_THREADS)
across_blind_kernel(const AcrossBlindArgs a) {
  pdl_prologue();
  const int64_t b = blockIdx.y, P = a.P, n = a.n;
  const int LA = a.counts[(2 * b + 0) * a.counts_stride + a.nblk];
  const int LB = a.counts[(2 * b + 1) * a.counts_stride + a.nblk];
  const bool empty = LA == 0 || LB == 0;
  if (blockIdx.x == 0 && threadIdx.x < 4) {
    a.counts_out[b * 4 + threadIdx.x] = (threadIdx.x == 3 && !empty) ? n : 0;
    if (threadIdx.x == 0) a.empty[b] = empty ? 1 : 0;
  }
  const bool fa = a.params[(2 * b + 0) * DDN_WS_PARAM_BYTES + DDN_WS_FLIP] != 0;
  const bool fb = a.params[(2 * b + 1) * DDN_WS_PARAM_BYTES + DDN_WS_FLIP] != 0;
  const int* nz_a = a.nz + (2 * b + 0) * P; const int* nz_b = a.nz + (2 * b + 1) * P;
  const float* ra = a.ra + b * n; const float* rb = a.rb + b * n;
  int64_t* out_a = a.out_a + b * n; int64_t* out_b = a.out_b + b * n;
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) {
    if (empty) { out_a[j] = -1; out_b[j] = -1; continue; }
    const int64_t pa = masked_pick(ra[j], LA, nz_a), pb = masked_pick(rb[j], LB, nz_b);
    out_a[j] = fa ? P - 1 - pa : pa;                    // ((W-1) - u, (H-1) - v) on LongTensors, flattened
    out_b[j] = fb ? P - 1 - pb : pb;
  }
}

struct AsScratch { int *counts, *nz; size_t bytes; };

static AsScratch as_layout(const ddn_as_batch_cfg& c, char* base) {
  const int64_t B = c.B, P = (int64_t)c.H * c.W;
  AsScratch s;
  size_t off = 0;
  auto take = [&](size_t bytes) { char* p = base ? base + off : nullptr; off += align_up(bytes, 256); return p; };
  s.counts = (int*)take(sizeof(int) * 2 * B * compact_counts_stride(P)); s.nz = (int*)take(sizeof(int) * 2 * B * P);
  s.bytes = off + 256;
  return s;
}

static bool as_cfg_ok(const ddn_as_batch_cfg* c) {
  if (!c) return false;
  const int64_t P = (int64_t)c->H * c->W;
  bool ok = (c->domain_randomize == 0 || c->domain_randomize == 1) && c->B >= 1 && c->B <= DDN_AS_MAX_PAIRS && c->H >= 1 &&
            c->W >= 1 && P < (1ll << 30) && c->num_samples >= 1 && c->num_samples < (1ll << 30);
  for (int i = 0; i < 3; ++i) ok = ok && c->std[i] != 0.f && c->std[i] == c->std[i] && c->mean[i] == c->mean[i];
  return ok;
}

}  // namespace ddn

using namespace ddn;

extern "C" size_t ddn_across_scene_batch_scratch_bytes(const ddn_as_batch_cfg* cfg) {
  if (!as_cfg_ok(cfg)) return 0;
  return as_layout(*cfg, nullptr).bytes;
}

extern "C" int ddn_across_scene_batch(const ddn_as_batch_cfg* cfg, const uint8_t* rgb_a, const uint8_t* rgb_b,
                                      const uint8_t* mask_a, const uint8_t* mask_b, const ddn_as_batch_rand* rand,
                                      const ddn_as_batch_out* out, void* scratch, size_t scratch_bytes, void* stream) {
  DDN_CHECK_ARG(as_cfg_ok(cfg), "bad across-scene configuration (B in [1, %d], H, W, num_samples >= 1, domain_randomize 0/1, "
                "std != 0)", DDN_AS_MAX_PAIRS);
  const ddn_as_batch_cfg c = *cfg;
  const int B = c.B, H = c.H, W = c.W;
  const int64_t P = (int64_t)H * W, n = c.num_samples;
  DDN_CHECK_ARG(rgb_a && rgb_b && mask_a && mask_b && rand && out, "null argument");
  DDN_CHECK_ARG(rand->params && rand->noise && rand->blind_a && rand->blind_b, "null random-number array");
  DDN_CHECK_ARG(out->image_a && out->image_b && out->blind_a && out->blind_b && out->counts && out->empty, "null output array");
  DDN_CHECK_ARG(scratch && scratch_bytes >= as_layout(c, nullptr).bytes, "scratch too small");

  cudaStream_t st = (cudaStream_t)stream;
  const AsScratch s = as_layout(c, reinterpret_cast<char*>(align_up(reinterpret_cast<uintptr_t>(scratch), 256)));
  const int nblkP = (int)ceil_div(P, SAMP_PER_BLOCK);
  const int64_t csP = compact_counts_stride(P);
  const int wide = num_sms() * 8;
  auto blocks = [&](int64_t items) { return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(items, SAMP_THREADS), wide)); };

  // 1. nonzero pixels of mask_a and mask_b (ascending, as torch.nonzero); their totals mark empty pairs
  const CompactRows cm = {s.counts, s.nz, csP, P, nblkP};
  DDN_TRY(compact_rows(NonzeroU8Pair{mask_a, mask_b, P}, P, 2 * B, cm, st));

  // 2. background randomisation, flip and normalisation of both images
  AugmentArgs aug = {rgb_a, rgb_b, mask_a, mask_b, rand->params, rand->noise, s.counts + nblkP, 2 * csP, s.counts + csP + nblkP,
                     c.domain_randomize, out->image_a, out->image_b, nullptr, nullptr, {c.mean[0], c.mean[1], c.mean[2]},
                     {c.std[0], c.std[1], c.std[2]}, B, H, W};
  DDN_LAUNCH(augment_kernel, blocks(2 * B * P), 256, 0, st, aug);

  // 3. blind pixels, flipped; counts and the empty flag
  const AcrossBlindArgs bl = {s.nz, s.counts, csP, nblkP, rand->blind_a, rand->blind_b, rand->params,
                              out->blind_a, out->blind_b, out->counts, out->empty, n, P};
  DDN_LAUNCH(across_blind_kernel, dim3(blocks(n), B), SAMP_THREADS, 0, st, bl);
  return 0;
}
