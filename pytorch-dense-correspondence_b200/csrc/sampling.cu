// Non-match sampling on the device (SURVEY.md 8f row 2).
// Replaces the CPU pipeline of dense_correspondence/correspondence_tools/correspondence_finder.py:276-405
// (create_non_correspondences: nonzero(mask) -> rand*len -> floor -> index_select -> (u, v)) followed by
// dense_correspondence/dataset/spartan_dataset_masked.py:841-858 (create_non_matches: every match repeated k times on the
// A side) and :1255-1264 (flatten_uv_tensor: n = u + W*v), i.e. it emits the two int64 index tensors the loss consumes
// directly, so up to 2 x 1.5 M x 8 bytes per pair never cross PCIe.
// The reference's "perturb non-matches that are too close to a match" step is a no-op upstream (`ones = torch.zeros_like`
// at correspondence_finder.py:354 makes need_to_be_perturbed identically zero); it is reproduced as that no-op.
// The uniform random numbers are an INPUT (torch.rand on the device), which makes the op bit-reproducible against the
// restated reference given the same numbers.
// The kernels (sampling.cuh) work on rows of image pairs; the two entry points here are a batch of one.
#include "sampling.cuh"

using namespace ddn;

extern "C" size_t ddn_sample_non_matches_scratch_bytes(int H, int W) {
  int64_t P = (int64_t)H * W;
  return sizeof(int) * (size_t)(P + ceil_div(P, SAMP_PER_BLOCK) + 8) + 256;
}

extern "C" int ddn_sample_non_matches(const float* mask, int H, int W, const float* rand_u, const float* rand_v, int64_t n,
                                      const int64_t* matches_a, int64_t non_matches_per_match, int64_t* out_a, int64_t* out_b,
                                      void* scratch, size_t scratch_bytes, void* stream) {
  DDN_CHECK_ARG(rand_u && rand_v && out_b && H > 0 && W > 0 && n >= 0 && (int64_t)H * W < (1ll << 31), "bad arguments");
  DDN_CHECK_ARG(!out_a || (matches_a && non_matches_per_match >= 1), "A-side output needs matches_a and non_matches_per_match");
  if (n == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t P = (int64_t)H * W;
  SampleRows s = {};
  if (mask) {
    DDN_CHECK_ARG(scratch && scratch_bytes >= ddn_sample_non_matches_scratch_bytes(H, W), "scratch too small");
    const int nblk = (int)ceil_div(P, SAMP_PER_BLOCK);
    DDN_CHECK_ARG(nblk <= 1 << 20, "image too large");
    int* counts = reinterpret_cast<int*>(scratch);      // [nblk + 1]
    const CompactRows c = {counts, counts + nblk + 8, 0, 0, nblk};
    DDN_TRY(compact_rows(NonzeroF32{mask, P}, P, 1, c, st));
    s.nz = c.nz; s.counts = counts; s.nblk = nblk;
  }
  s.ru = rand_u; s.rv = rand_v; s.n = n; s.k = out_a ? non_matches_per_match : 1;
  s.matches_a = matches_a; s.out_a = out_a; s.out_b = out_b; s.H = H; s.W = W;
  int blocks = (int)std::min<int64_t>(ceil_div(n, SAMP_THREADS), (int64_t)num_sms() * 8);
  DDN_LAUNCH(sample_non_matches_kernel, blocks, SAMP_THREADS, 0, st, s);
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Pinhole reprojection match finder: see sampling.cuh.
namespace ddn {

bool reproj_mats(const double* K, const double* pose_a, const double* pose_b, ReprojMats& m) {
  const double det = K[0] * (K[4] * K[8] - K[5] * K[7]) - K[1] * (K[3] * K[8] - K[5] * K[6]) + K[2] * (K[3] * K[7] - K[4] * K[6]);
  if (det == 0.0) return false;
  const double inv[9] = {(K[4] * K[8] - K[5] * K[7]) / det, (K[2] * K[7] - K[1] * K[8]) / det, (K[1] * K[5] - K[2] * K[4]) / det,
                         (K[5] * K[6] - K[3] * K[8]) / det, (K[0] * K[8] - K[2] * K[6]) / det, (K[2] * K[3] - K[0] * K[5]) / det,
                         (K[3] * K[7] - K[4] * K[6]) / det, (K[1] * K[6] - K[0] * K[7]) / det, (K[0] * K[4] - K[1] * K[3]) / det};
  for (int i = 0; i < 9; ++i) { m.Kinv[i] = (float)inv[i]; m.K[i] = (float)K[i]; }
  for (int i = 0; i < 12; ++i) m.Ta[i] = (float)pose_a[i];
  // invert_transform (correspondence_finder.py:52-62): [R^T | -R^T t] in double, then cast to fp32
  const double* P = pose_b;
  const double Rt[9] = {P[0], P[4], P[8], P[1], P[5], P[9], P[2], P[6], P[10]};
  const double t[3] = {P[3], P[7], P[11]};
  for (int r = 0; r < 3; ++r) {
    m.Tb_inv[r * 4 + 0] = (float)Rt[r * 3 + 0]; m.Tb_inv[r * 4 + 1] = (float)Rt[r * 3 + 1]; m.Tb_inv[r * 4 + 2] = (float)Rt[r * 3 + 2];
    m.Tb_inv[r * 4 + 3] = (float)(-1.0 * (Rt[r * 3 + 0] * t[0] + Rt[r * 3 + 1] * t[1] + Rt[r * 3 + 2] * t[2]));
  }
  return true;
}

}  // namespace ddn

extern "C" size_t ddn_find_pixel_correspondences_scratch_bytes(int64_t n) {
  return (size_t)n * (4 + 8 + 4 + 4) + sizeof(int) * (size_t)(n + ceil_div(n, SAMP_PER_BLOCK) + 16) + 1024;
}

// candidates [n] int64 flat pixels of image A; depth images fp32 [H*W] in raw sensor units (millimetres);
// K [9], pose_a [16], pose_b [16] row-major HOST doubles (the reference's numpy matrices).
// out_a / out_b [n] (first *count entries valid, *count is a DEVICE int64), optional out_u2 / out_v2 (sub-pixel positions).
extern "C" int ddn_find_pixel_correspondences(const float* depth_a, const float* depth_b, int H, int W,
                                              const int64_t* candidates, int64_t n,
                                              const double* K_host, const double* pose_a_host, const double* pose_b_host,
                                              int64_t* out_a, int64_t* out_b, float* out_u2, float* out_v2, int64_t* out_count,
                                              void* scratch, size_t scratch_bytes, void* stream) {
  DDN_CHECK_ARG(depth_a && depth_b && candidates && K_host && pose_a_host && pose_b_host && out_a && out_b && out_count && scratch,
                "null argument");
  DDN_CHECK_ARG(H > 0 && W > 0 && n > 0 && n < (1ll << 30) && scratch_bytes >= ddn_find_pixel_correspondences_scratch_bytes(n),
                "bad sizes / scratch too small");
  cudaStream_t st = (cudaStream_t)stream;
  ReprojBatch<1> mats;
  DDN_CHECK_ARG(reproj_mats(K_host, pose_a_host, pose_b_host, mats.m[0]), "singular intrinsics");
  char* p = reinterpret_cast<char*>(align_up(reinterpret_cast<uintptr_t>(scratch), 16));
  float* flag = (float*)p; p += align_up((size_t)n * 4, 16);
  int64_t* b_flat = (int64_t*)p; p += align_up((size_t)n * 8, 16);
  float* u2 = (float*)p; p += align_up((size_t)n * 4, 16);
  float* v2 = (float*)p; p += align_up((size_t)n * 4, 16);
  const int nblk = (int)ceil_div(n, SAMP_PER_BLOCK);
  int* counts = (int*)p;
  const CompactRows c = {counts, counts + nblk + 8, 0, 0, nblk};
  int blocks = (int)std::min<int64_t>(ceil_div(n, SAMP_THREADS), (int64_t)num_sms() * 8);
  DDN_LAUNCH(reproject_kernel<1>, blocks, SAMP_THREADS, 0, st, depth_a, depth_b, candidates, n, H, W, mats, flag, b_flat, u2, v2);
  DDN_TRY(compact_rows(NonzeroF32{flag, n}, n, 1, c, st));
  GatherRows g = {};
  g.nz = c.nz; g.counts = counts; g.nblk = nblk;
  g.cand = candidates; g.b_flat = b_flat; g.u2 = u2; g.v2 = v2;
  g.out_a = out_a; g.out_b = out_b; g.out_u2 = out_u2; g.out_v2 = out_v2; g.out_count = out_count;
  g.H = H; g.W = W;
  DDN_LAUNCH(reproject_gather_kernel, blocks, SAMP_THREADS, 0, st, g);
  return 0;
}
