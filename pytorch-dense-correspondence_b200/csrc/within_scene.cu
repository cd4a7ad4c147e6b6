// Within-scene training batches on the device: SpartanDataset.get_within_scene_data
// (dense_correspondence/dataset/spartan_dataset_masked.py:646-769) for B image pairs in one call, given its random numbers.
// The DataLoader worker then only decodes the PNGs; the call returns what forward_pair and get_loss(num_valid=...) consume,
// with no host synchronisation.  Contract and layouts: include/ddn_b200.h (ddn_within_scene_batch).
//
// Launches (16, whatever B):  compact mask_a (3)  ->  augment + flip + normalise (1)  ->  candidates (1)  ->  reprojection
// (1)  ->  compact survivors (3)  ->  gather with the flip (1)  ->  compact flipped mask_b != 0, mask_b != 1 and the blind
// predicate (3)  ->  masked, background (2)  ->  blind (1).
#include "sampling.cuh"

namespace ddn {

// Row 3*pair + set over the flipped masks fmask [B, 2 (A, B), P] and the matched-pixel bitmap hit [B, P]:
//   set 0: mask_b != 0 (masked non-matches, blind B side);  set 1: 1 - mask_b != 0 (background non-matches);
//   set 2: mask_a - matched != 0 (blind A side, spartan_dataset_masked.py:736-739; an off-mask match gives -1 and is kept)
struct WsSets {
  const uint8_t* fmask; const uint8_t* hit; int64_t P;
  __device__ __forceinline__ bool operator()(int64_t r, int64_t p) const {
    const int64_t b = r / 3; const int s = (int)(r - 3 * b);
    if (s == 2) return fmask[(2 * b) * P + p] != hit[b * P + p];
    const uint8_t m = fmask[(2 * b + 1) * P + p];
    return s == 0 ? m != 0 : m != 1;
  }
};

struct BlindArgs {
  const int* nz3; const int* counts3; int64_t counts_stride; int nblk;   // rows 3*pair + set of the WsSets compaction
  const float* rand; const uint8_t* empty;
  int64_t* out_a; int64_t* out_b; int64_t* counts; int64_t P;
};

// blind non-matches (spartan_dataset_masked.py:735-769): A side = every set-2 pixel in ascending order, B side =
// random_sample_from_masked_image_torch(mask_b, n) over the set-0 pixels; count 0 when either side is empty
__global__ void __launch_bounds__(SAMP_THREADS)
blind_kernel(const BlindArgs a) {
  pdl_prologue();
  const int64_t b = blockIdx.y, P = a.P;
  const int LB = a.counts3[(3 * b + 0) * a.counts_stride + a.nblk];
  const int LA = a.counts3[(3 * b + 2) * a.counts_stride + a.nblk];
  const int64_t n = (a.empty[b] || LB == 0) ? 0 : LA;
  if (blockIdx.x == 0 && threadIdx.x == 0) a.counts[b * 4 + 3] = n;
  const int* nz_b = a.nz3 + (3 * b + 0) * P; const int* nz_a = a.nz3 + (3 * b + 2) * P;
  int64_t* out_a = a.out_a + b * P; int64_t* out_b = a.out_b + b * P;
  const float* r = a.rand + b * P;
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < P; j += (int64_t)gridDim.x * blockDim.x) {
    if (j >= n) { out_a[j] = -1; out_b[j] = -1; continue; }
    out_a[j] = nz_a[j]; out_b[j] = masked_pick(r[j], LB, nz_b);
  }
}

struct WsScratch {
  int *counts_a, *nz_a, *counts_f, *nz_f, *counts3, *nz3;
  uint8_t *fmask, *hit;
  int64_t *cand, *b_flat;
  float *flag, *u2, *v2;
  size_t bytes;
};

static WsScratch ws_layout(const ddn_ws_batch_cfg& c, char* base) {
  const int64_t B = c.B, P = (int64_t)c.H * c.W, n = c.n_attempts;
  const int64_t csP = compact_counts_stride(P), csN = compact_counts_stride(n);
  WsScratch s;
  size_t off = 0;
  auto take = [&](size_t bytes) { char* p = base ? base + off : nullptr; off += align_up(bytes, 256); return p; };
  s.counts_a = (int*)take(sizeof(int) * B * csP); s.nz_a = (int*)take(sizeof(int) * B * P);
  s.fmask = (uint8_t*)take(2 * B * P); s.hit = (uint8_t*)take(B * P);
  s.cand = (int64_t*)take(8 * B * n); s.flag = (float*)take(4 * B * n); s.b_flat = (int64_t*)take(8 * B * n);
  s.u2 = (float*)take(4 * B * n); s.v2 = (float*)take(4 * B * n);
  s.counts_f = (int*)take(sizeof(int) * B * csN); s.nz_f = (int*)take(sizeof(int) * B * n);
  s.counts3 = (int*)take(sizeof(int) * 3 * B * csP); s.nz3 = (int*)take(sizeof(int) * 3 * B * P);
  s.bytes = off + 256;
  return s;
}

static bool ws_cfg_ok(const ddn_ws_batch_cfg* c) {
  if (!c) return false;
  auto flag = [](int32_t v) { return v == 0 || v == 1; };
  const bool flags = flag(c->sample_matches_only_off_mask) && flag(c->domain_randomize) && flag(c->use_image_b_mask_inv);
  const int64_t P = (int64_t)c->H * c->W;
  const int64_t kmax = c->k_masked > c->k_background ? c->k_masked : c->k_background;
  bool ok = flags && c->B >= 1 && c->B <= DDN_WS_MAX_PAIRS && c->H >= 1 && c->W >= 1 && P < (1ll << 30) &&
            c->n_attempts >= 1 && c->n_attempts < (1ll << 30) && c->k_masked >= 0 && c->k_background >= 0 &&
            kmax <= (1ll << 30) / c->n_attempts;
  for (int i = 0; i < 3; ++i) ok = ok && c->std[i] != 0.f && c->std[i] == c->std[i] && c->mean[i] == c->mean[i];
  return ok;
}

}  // namespace ddn

using namespace ddn;

extern "C" size_t ddn_within_scene_batch_scratch_bytes(const ddn_ws_batch_cfg* cfg) {
  if (!ws_cfg_ok(cfg)) return 0;
  return ws_layout(*cfg, nullptr).bytes;
}

extern "C" int ddn_within_scene_batch(const ddn_ws_batch_cfg* cfg, const uint8_t* rgb_a, const uint8_t* rgb_b,
                                      const uint8_t* mask_a, const uint8_t* mask_b, const float* depth_a, const float* depth_b,
                                      const double* K_host, const double* poses_a_host, const double* poses_b_host,
                                      const ddn_ws_batch_rand* rand, const ddn_ws_batch_out* out,
                                      void* scratch, size_t scratch_bytes, void* stream) {
  DDN_CHECK_ARG(ws_cfg_ok(cfg), "bad within-scene configuration (B in [1, %d], H, W, n_attempts >= 1, k >= 0, flags 0/1, std != 0)",
                DDN_WS_MAX_PAIRS);
  const ddn_ws_batch_cfg c = *cfg;
  const int B = c.B, H = c.H, W = c.W;
  const int64_t P = (int64_t)H * W, n = c.n_attempts, cap_m = n * c.k_masked, cap_b = n * c.k_background;
  DDN_CHECK_ARG(rgb_a && rgb_b && mask_a && mask_b && depth_a && depth_b && K_host && poses_a_host && poses_b_host && rand && out,
                "null argument");
  DDN_CHECK_ARG(rand->params && rand->noise && rand->cand_u && rand->cand_v && rand->blind &&
                (cap_m == 0 || (rand->masked_u && rand->masked_v)) && (cap_b == 0 || (rand->background_u && rand->background_v)),
                "null random-number array");
  DDN_CHECK_ARG(out->image_a && out->image_b && out->matches_a && out->matches_b && out->blind_a && out->blind_b && out->counts &&
                out->empty && (cap_m == 0 || (out->masked_a && out->masked_b)) &&
                (cap_b == 0 || (out->background_a && out->background_b)), "null output array");
  DDN_CHECK_ARG(scratch && scratch_bytes >= ws_layout(c, nullptr).bytes, "scratch too small");
  ReprojBatch<DDN_WS_MAX_PAIRS> mats;
  for (int b = 0; b < B; ++b)
    DDN_CHECK_ARG(reproj_mats(K_host, poses_a_host + 16 * b, poses_b_host + 16 * b, mats.m[b]), "singular intrinsics");

  cudaStream_t st = (cudaStream_t)stream;
  const WsScratch s = ws_layout(c, reinterpret_cast<char*>(align_up(reinterpret_cast<uintptr_t>(scratch), 256)));
  const int nblkP = (int)ceil_div(P, SAMP_PER_BLOCK), nblkN = (int)ceil_div(n, SAMP_PER_BLOCK);
  const int64_t csP = compact_counts_stride(P), csN = compact_counts_stride(n);
  const int wide = num_sms() * 8;
  auto blocks = [&](int64_t items) { return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(items, SAMP_THREADS), wide)); };

  // 1. candidates' mask in A (random_sample_from_masked_image_torch, correspondence_finder.py:92-121); its totals mark empty pairs
  const CompactRows ca = {s.counts_a, s.nz_a, csP, P, nblkP};
  DDN_TRY(compact_rows(NonzeroU8{mask_a, P}, P, B, ca, st));
  const int* total_a = c.sample_matches_only_off_mask ? s.counts_a + nblkP : nullptr;

  // 2. background randomisation, flip and normalisation of both images; flipped masks; zeroed matched-pixel bitmap
  AugmentArgs aug = {rgb_a, rgb_b, mask_a, mask_b, rand->params, rand->noise, total_a, csP, nullptr, c.domain_randomize,
                     out->image_a, out->image_b, s.fmask, s.hit, {c.mean[0], c.mean[1], c.mean[2]},
                     {c.std[0], c.std[1], c.std[2]}, B, H, W};
  DDN_LAUNCH(augment_kernel, blocks(2 * B * P), 256, 0, st, aug);

  // 3. candidates: from mask_a, or pytorch_rand_select_pixel when not sampling on the mask
  SampleRows sc = {};
  if (c.sample_matches_only_off_mask) { sc.nz = s.nz_a; sc.counts = s.counts_a; sc.nz_stride = P; sc.counts_stride = csP; sc.nblk = nblkP; }
  sc.ru = rand->cand_u; sc.rv = rand->cand_v; sc.r_stride = n; sc.n = n; sc.k = 1;
  sc.out_b = s.cand; sc.out_stride = n; sc.H = H; sc.W = W;
  DDN_LAUNCH(sample_non_matches_kernel, dim3(blocks(n), B), SAMP_THREADS, 0, st, sc);

  // 4. reprojection, survivors, and their gather with the flip applied (matches, counts[:, 0], empty, bitmap)
  DDN_LAUNCH(reproject_kernel<DDN_WS_MAX_PAIRS>, dim3(blocks(n), B), SAMP_THREADS, 0, st, depth_a, depth_b, s.cand, n, H, W, mats,
             s.flag, s.b_flat, s.u2, s.v2);
  const CompactRows cf = {s.counts_f, s.nz_f, csN, n, nblkN};
  DDN_TRY(compact_rows(NonzeroF32{s.flag, n}, n, B, cf, st));
  GatherRows g = {};
  g.nz = s.nz_f; g.counts = s.counts_f; g.nz_stride = n; g.counts_stride = csN; g.nblk = nblkN;
  g.cand = s.cand; g.b_flat = s.b_flat; g.u2 = s.u2; g.v2 = s.v2; g.in_stride = n;
  g.out_a = out->matches_a; g.out_b = out->matches_b; g.out_stride = n; g.pad_to = n;
  g.out_count = out->counts; g.count_stride = 4;
  g.flip_a = rand->params + DDN_WS_FLIP; g.flip_b = rand->params + DDN_WS_PARAM_BYTES + DDN_WS_FLIP;
  g.flip_stride = 2 * DDN_WS_PARAM_BYTES;
  g.empty_total = total_a; g.empty_stride = csP; g.empty_out = out->empty;
  g.hit = s.hit; g.H = H; g.W = W;
  DDN_LAUNCH(reproject_gather_kernel, dim3(blocks(n), B), SAMP_THREADS, 0, st, g);

  // 5. the flipped mask_b (!= 0, != 1) and the blind predicate, one compaction
  const CompactRows c3 = {s.counts3, s.nz3, csP, P, nblkP};
  DDN_TRY(compact_rows(WsSets{s.fmask, s.hit, P}, P, 3 * B, c3, st));

  // 6. masked and background non-matches (create_non_correspondences + create_non_matches + flatten_uv_tensor)
  for (int set = 0; set < 2; ++set) {
    const bool masked = set == 0;
    SampleRows sn = {};
    if (masked || c.use_image_b_mask_inv) {
      sn.nz = s.nz3 + set * P; sn.counts = s.counts3 + set * csP; sn.nz_stride = 3 * P; sn.counts_stride = 3 * csP; sn.nblk = nblkP;
    }
    sn.ru = masked ? rand->masked_u : rand->background_u; sn.rv = masked ? rand->masked_v : rand->background_v;
    sn.r_stride = masked ? cap_m : cap_b;
    sn.n_dev = out->counts; sn.n_stride = 4; sn.k = masked ? c.k_masked : c.k_background;
    sn.matches_a = out->matches_a; sn.ma_stride = n;
    sn.out_a = masked ? out->masked_a : out->background_a; sn.out_b = masked ? out->masked_b : out->background_b;
    sn.out_stride = sn.r_stride; sn.pad_to = sn.r_stride;
    sn.count_out = out->counts + 1 + set; sn.count_stride = 4; sn.H = H; sn.W = W;
    DDN_LAUNCH(sample_non_matches_kernel, dim3(blocks(sn.r_stride), B), SAMP_THREADS, 0, st, sn);
  }

  // 7. blind non-matches
  const BlindArgs bl = {s.nz3, s.counts3, csP, nblkP, rand->blind, out->empty, out->blind_a, out->blind_b, out->counts, P};
  DDN_LAUNCH(blind_kernel, dim3(blocks(P), B), SAMP_THREADS, 0, st, bl);
  return 0;
}
