// Device sampling kernels shared by the single-pair entry points (sampling.cu) and the within-scene and across-scene batch
// producers (within_scene.cu, across_scene.cu).  Every kernel works on ROWS: blockIdx.y (or the row loop) selects one image pair (or one pair x mask),
// and the single-pair entry points are a batch of one row.
#pragma once
#include "common.cuh"

namespace ddn {

constexpr int SAMP_THREADS = 256;
constexpr int SAMP_PER_BLOCK = 1024;     // pixels per block in the compaction passes

// Compaction predicates: pixel p (of P) of row r is selected when pred(r, p) holds.
struct NonzeroF32 {
  const float* x; int64_t P;
  __device__ __forceinline__ bool operator()(int64_t r, int64_t p) const { return x[r * P + p] != 0.f; }
};
struct NonzeroU8 {
  const uint8_t* x; int64_t P;
  __device__ __forceinline__ bool operator()(int64_t r, int64_t p) const { return x[r * P + p] != 0; }
};

// random_sample_from_masked_image_torch (correspondence_finder.py:92-121) for one number: the r-th of the L >= 1 selected
// pixels nz[0..L) at floor(r * L), clamped at L - 1 (fp32 rounding at r ~ 1: the reference's index_select would raise there)
__device__ __forceinline__ int masked_pick(float r, int L, const int* nz) {
  int q = (int)floorf(r * (float)L);
  if (q >= L) q = L - 1;
  return nz[q];
}

// Per-row layout of a compaction: block counts (then the row total at index nblk) at counts + r * counts_stride,
// selected pixels at nz + r * nz_stride.
struct CompactRows { int* counts; int* nz; int64_t counts_stride, nz_stride; int nblk; };

template <class Pred>
__global__ void __launch_bounds__(SAMP_THREADS)
mask_count_kernel(const Pred pred, int64_t P, CompactRows c) {
  pdl_prologue();
  const int64_t r = blockIdx.y;
  const int64_t base = (int64_t)blockIdx.x * SAMP_PER_BLOCK;
  int n = 0;
#pragma unroll
  for (int i = 0; i < SAMP_PER_BLOCK / SAMP_THREADS; ++i) {
    int64_t p = base + i * SAMP_THREADS + threadIdx.x;
    n += (p < P && pred(r, p)) ? 1 : 0;
  }
  n = warp_sum(n);
  __shared__ int s[SAMP_THREADS / 32];
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = n;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int i = 0; i < SAMP_THREADS / 32; ++i) t += s[i];
    c.counts[r * c.counts_stride + blockIdx.x] = t;
  }
}

// exclusive scan of one row's block counts by one block (blockIdx.x = row); the row total -> counts[nblk]
template <int = 0>
__global__ void __launch_bounds__(1024)
mask_scan_kernel(CompactRows c) {
  pdl_prologue();
  int* counts = c.counts + (int64_t)blockIdx.x * c.counts_stride;
  const int nblk = c.nblk;
  __shared__ int s[1024];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < nblk; base += 1024) {
    int i = base + threadIdx.x;
    int v = i < nblk ? counts[i] : 0;
    s[threadIdx.x] = v;
    __syncthreads();
    for (int off = 1; off < 1024; off <<= 1) {
      int t = threadIdx.x >= off ? s[threadIdx.x - off] : 0;
      __syncthreads();
      s[threadIdx.x] += t;
      __syncthreads();
    }
    int incl = s[threadIdx.x];
    if (i < nblk) counts[i] = carry + incl - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry += incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) counts[nblk] = carry;
}

// ascending list of the selected pixels of each row (== torch.nonzero order)
template <class Pred>
__global__ void __launch_bounds__(SAMP_THREADS)
mask_compact_kernel(const Pred pred, int64_t P, CompactRows c) {
  pdl_prologue();
  const int64_t r = blockIdx.y;
  const int64_t base = (int64_t)blockIdx.x * SAMP_PER_BLOCK;
  __shared__ int warp_tot[SAMP_PER_BLOCK / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  bool f[SAMP_PER_BLOCK / SAMP_THREADS];
  int rank[SAMP_PER_BLOCK / SAMP_THREADS];
#pragma unroll
  for (int i = 0; i < SAMP_PER_BLOCK / SAMP_THREADS; ++i) {
    int64_t p = base + i * SAMP_THREADS + threadIdx.x;
    f[i] = p < P && pred(r, p);
    unsigned b = __ballot_sync(0xffffffffu, f[i]);
    rank[i] = __popc(b & ((1u << lane) - 1u));
    if (lane == 0) warp_tot[i * (SAMP_THREADS / 32) + wid] = __popc(b);
  }
  __syncthreads();
  const int off = c.counts[r * c.counts_stride + blockIdx.x];
  int* nz = c.nz + r * c.nz_stride;
  // segment order inside the block: (i, wid) ascending == pixel order
#pragma unroll
  for (int i = 0; i < SAMP_PER_BLOCK / SAMP_THREADS; ++i) {
    if (!f[i]) continue;
    int seg = i * (SAMP_THREADS / 32) + wid, before = 0;
    for (int k = 0; k < seg; ++k) before += warp_tot[k];
    nz[off + before + rank[i]] = (int)(base + i * SAMP_THREADS + threadIdx.x);
  }
}

// count + scan + compact of `rows` rows of P pixels each
template <class Pred>
static inline int compact_rows(const Pred& pred, int64_t P, int rows, const CompactRows& c, cudaStream_t st) {
  DDN_LAUNCH(mask_count_kernel<Pred>, dim3(c.nblk, rows), SAMP_THREADS, 0, st, pred, P, c);
  DDN_LAUNCH(mask_scan_kernel<>, rows, 1024, 0, st, c);
  DDN_LAUNCH(mask_compact_kernel<Pred>, dim3(c.nblk, rows), SAMP_THREADS, 0, st, pred, P, c);
  return 0;
}

static inline int64_t compact_counts_stride(int64_t P) { return ceil_div(P, SAMP_PER_BLOCK) + 8; }

// Sampling rows (blockIdx.y = row).  Row r draws n_r = n_dev ? n_dev[r * n_stride] * k : n samples:
//   out_b[j] = nz[floor(ru[j] * L)] over the row's L selected pixels, or a uniform pixel (floor(ru*W), floor(rv*H)) when the
//   row has no compaction (nz == NULL) or L == 0;  out_a[j] = matches_a[j / k] (out_a may be NULL).
// Entries [n_r, pad_to) are set to -1 and n_r is stored at count_out[r * count_stride] when count_out is given.
struct SampleRows {
  const int* nz; const int* counts; int64_t nz_stride, counts_stride; int nblk;
  const float* ru; const float* rv; int64_t r_stride;
  const int64_t* n_dev; int64_t n_stride; int64_t n; int64_t k;
  const int64_t* matches_a; int64_t ma_stride;
  int64_t* out_a; int64_t* out_b; int64_t out_stride; int64_t pad_to;
  int64_t* count_out; int64_t count_stride;
  int H, W;
};

static __global__ void __launch_bounds__(SAMP_THREADS)
sample_non_matches_kernel(const SampleRows s) {
  pdl_prologue();
  const int64_t r = blockIdx.y;
  const int L = s.nz ? s.counts[r * s.counts_stride + s.nblk] : 0;
  const int* nz = s.nz + r * s.nz_stride;
  const float* rand_u = s.ru + r * s.r_stride;
  const float* rand_v = s.rv + r * s.r_stride;
  const int64_t* matches_a = s.matches_a + r * s.ma_stride;
  int64_t* out_a = s.out_a ? s.out_a + r * s.out_stride : nullptr;
  int64_t* out_b = s.out_b + r * s.out_stride;
  const int64_t n = s.n_dev ? s.n_dev[r * s.n_stride] * s.k : s.n;
  const int H = s.H, W = s.W;
  if (s.count_out && blockIdx.x == 0 && threadIdx.x == 0) s.count_out[r * s.count_stride] = n;
  const int64_t end = n > s.pad_to ? n : s.pad_to;
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < end; j += (int64_t)gridDim.x * blockDim.x) {
    if (j >= n) {
      out_b[j] = -1;
      if (out_a) out_a[j] = -1;
      continue;
    }
    int64_t b;
    if (L > 0) {
      b = masked_pick(rand_u[j], L, nz);              // torch.rand(n) * len(mask_b_indices_flat) -> floor -> long
    } else {                                           // no / empty mask: pytorch_rand_select_pixel (finder.py:64-75)
      int u = (int)floorf(rand_u[j] * (float)W), v = (int)floorf(rand_v[j] * (float)H);
      if (u >= W) u = W - 1;
      if (v >= H) v = H - 1;
      b = (int64_t)u + (int64_t)W * v;
    }
    out_b[j] = b;
    if (out_a) out_a[j] = matches_a[j / s.k];
  }
}

// ------------------------------------------------------------------------------------------------
// Pinhole reprojection match finder (SURVEY.md 8f row 3) == batch_find_pixel_correspondences
// (dense_correspondence/correspondence_tools/correspondence_finder.py:409-619) for candidate pixels already drawn in image A:
// depth lookup (uint16 millimetres / DEPTH_IM_SCALE=1000, constants.py:10) -> K^-1 -> pose_a -> pose_b^-1 -> K -> (u2, v2),
// prune zero depth, out-of-frustum (including the reference's quirk that an exact 0.0 coordinate is pruned by nonzero()),
// and occlusion against depth image B with the 3 mm margin; survivors keep their order (stream compaction).
struct ReprojMats { float Kinv[9]; float Ta[12]; float Tb_inv[12]; float K[9]; };
// one matrix set per row, passed as a kernel parameter (NP * 168 bytes; sm_90 takes up to 32 KB of parameters)
template <int NP> struct ReprojBatch { ReprojMats m[NP]; };

// host-side matrix prep in double, exactly like the reference's numpy (inv(K), invert_transform(pose_b)), then cast to fp32;
// false when K is singular
bool reproj_mats(const double* K, const double* pose_a, const double* pose_b, ReprojMats& m);

__device__ __forceinline__ void mat3_apply(const float* M, float x, float y, float z, float& ox, float& oy, float& oz) {
  ox = M[0] * x + M[1] * y + M[2] * z;
  oy = M[3] * x + M[4] * y + M[5] * z;
  oz = M[6] * x + M[7] * y + M[8] * z;
}
__device__ __forceinline__ void rigid_apply(const float* T, float x, float y, float z, float& ox, float& oy, float& oz) {
  ox = T[0] * x + T[1] * y + T[2] * z + T[3];
  oy = T[4] * x + T[5] * y + T[6] * z + T[7];
  oz = T[8] * x + T[9] * y + T[10] * z + T[11];
}

// row r: candidates cand[r*n + j] of image A (depth_a + r*H*W) against depth_b + r*H*W; outputs [r*n + j]
template <int NP>
__global__ void __launch_bounds__(SAMP_THREADS)
reproject_kernel(const float* __restrict__ depth_a, const float* __restrict__ depth_b, const int64_t* __restrict__ cand, int64_t n,
                 int H, int W, const __grid_constant__ ReprojBatch<NP> mats, float* __restrict__ flag, int64_t* __restrict__ b_flat,
                 float* __restrict__ u2o, float* __restrict__ v2o) {
  pdl_prologue();
  const int64_t r = blockIdx.y, P = (int64_t)H * W;
  const ReprojMats& m = mats.m[r];
  depth_a += r * P; depth_b += r * P; cand += r * n; flag += r * n; b_flat += r * n; u2o += r * n; v2o += r * n;
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) {
    const int64_t ia = cand[j];
    float ok = 0.f; int64_t bf = 0; float u2 = 0.f, v2 = 0.f;
    if (ia >= 0 && ia < P) {
      const float depth = depth_a[ia] * 1.0f / 1000.0f;
      if (depth != 0.f) {
        const float u = (float)(ia % W), v = (float)(ia / W);
        float cx, cy, cz, wx, wy, wz, px, py, pz, qx, qy, qz;
        mat3_apply(m.Kinv, u * depth, v * depth, depth, cx, cy, cz);
        rigid_apply(m.Ta, cx, cy, cz, wx, wy, wz);
        rigid_apply(m.Tb_inv, wx, wy, wz, px, py, pz);
        mat3_apply(m.K, px, py, pz, qx, qy, qz);
        u2 = qx / qz; v2 = qy / qz;
        const float z2 = qz;
        const float ub = (float)W * 1.0f - 1e-3f, vb = (float)H * 1.0f - 1e-3f;
        bool in = !(u2 < 0.f) && !(u2 > ub) && u2 != 0.f && !(v2 < 0.f) && !(v2 > vb) && v2 != 0.f;
        if (in && u2 == u2 && v2 == v2) {
          bf = (int64_t)v2 * W + (int64_t)u2;                 // .type(long): truncation
          float d2 = depth_b[bf] * 1.0f / 1000.0f;
          if (d2 < 0.f) d2 = 0.f;
          if (d2 < z2 - 0.003f) d2 = 0.f;                      // occluded in image b
          ok = d2 != 0.f ? 1.f : 0.f;
        }
      }
    }
    flag[j] = ok; b_flat[j] = bf; u2o[j] = u2; v2o[j] = v2;
  }
}

// Gather of the survivors of each row (blockIdx.y = row), in candidate order.  The within-scene producer also uses:
//   flip_a / flip_b: per-row 180-degree rotation of image A / B (random_image_and_indices_mutation): a -> P-1-a, and
//     u2 -> fp32(W-1 - u2), v2 -> fp32(H-1 - v2) before the truncation to a flat index;
//   empty_total: a row whose value there is 0 keeps no survivor (the reference's empty-mask early return);
//   pad_to: entries [L, pad_to) are set to -1;  hit: 1 at every (flipped) matched pixel of A.
struct GatherRows {
  const int* nz; const int* counts; int64_t nz_stride, counts_stride; int nblk;
  const int64_t* cand; const int64_t* b_flat; const float* u2; const float* v2; int64_t in_stride;
  int64_t* out_a; int64_t* out_b; float* out_u2; float* out_v2; int64_t out_stride; int64_t pad_to;
  int64_t* out_count; int64_t count_stride;
  const uint8_t* flip_a; const uint8_t* flip_b; int64_t flip_stride;
  const int* empty_total; int64_t empty_stride; uint8_t* empty_out;
  uint8_t* hit; int H, W;
};

static __global__ void __launch_bounds__(SAMP_THREADS)
reproject_gather_kernel(const GatherRows g) {
  pdl_prologue();
  const int64_t r = blockIdx.y, P = (int64_t)g.H * g.W;
  const bool empty = g.empty_total && g.empty_total[r * g.empty_stride] == 0;
  const int L = empty ? 0 : g.counts[r * g.counts_stride + g.nblk];
  const bool fa = g.flip_a && g.flip_a[r * g.flip_stride], fb = g.flip_b && g.flip_b[r * g.flip_stride];
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    g.out_count[r * g.count_stride] = L;
    if (g.empty_out) g.empty_out[r] = empty ? 1 : 0;
  }
  const int* nz = g.nz + r * g.nz_stride;
  const int64_t* cand = g.cand + r * g.in_stride; const int64_t* b_flat = g.b_flat + r * g.in_stride;
  const float* u2 = g.u2 + r * g.in_stride; const float* v2 = g.v2 + r * g.in_stride;
  int64_t* out_a = g.out_a + r * g.out_stride; int64_t* out_b = g.out_b + r * g.out_stride;
  const int64_t end = L > g.pad_to ? L : g.pad_to;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < end; i += (int64_t)gridDim.x * blockDim.x) {
    if (i >= L) { out_a[i] = -1; out_b[i] = -1; continue; }
    const int j = nz[i];
    int64_t a = cand[j], b = b_flat[j];
    float u = u2[j], v = v2[j];
    if (fa) a = P - 1 - a;
    if (fb) {
      u = __fsub_rn((float)(g.W - 1), u); v = __fsub_rn((float)(g.H - 1), v);
      b = (int64_t)v * g.W + (int64_t)u;
    }
    out_a[i] = a; out_b[i] = b;
    if (g.out_u2) { g.out_u2[r * g.out_stride + i] = u; g.out_v2[r * g.out_stride + i] = v; }
    if (g.hit) g.hit[r * P + a] = 1;
  }
}

// ------------------------------------------------------------------------------------------------
// Background randomisation, flip and normalisation of both images of each pair (the within-scene and across-scene
// producers).  Per image a DDN_WS_PARAM_BYTES parameter block holds its decisions and colours (ddn_ws_batch_rand.params).
//   total_a / total_b: mask totals at [pair * total_stride]; a pair whose total_a (or, when given, total_b) is 0 is the
//     reference's return_empty_data: both outputs are the normalised, un-augmented image A.  total_a NULL: never empty.
//   fmask (optional): the flipped masks [B, 2, P];  hit (optional): the matched-pixel bitmap [B, P], zeroed.
struct AugmentArgs {
  const uint8_t* rgb_a; const uint8_t* rgb_b; const uint8_t* mask_a; const uint8_t* mask_b;
  const uint8_t* params; const uint8_t* noise;
  const int* total_a; int64_t total_stride;
  const int* total_b;
  int randomize;
  float* image_a; float* image_b; uint8_t* fmask; uint8_t* hit;
  float mean[3], std[3];
  int B, H, W;
};

// numpy.linspace(0, 1, n)[i]: i * (1 / (n - 1)), the last element exactly 1.0, [0.0] for n = 1
__device__ __forceinline__ double linspace01(int i, int n) {
  if (n < 2) return 0.0;
  if (i == n - 1) return 1.0;
  return __dmul_rn((double)i, __ddiv_rn(1.0, (double)(n - 1)));
}

// One thread per output pixel of image A or B of a pair.  The background randomisation (correspondence_augmentation.py:
// 96-214) happens at the source pixel in the unflipped frame; the flip (ImageOps.flip + mirror) then reads that pixel for
// the output pixel P-1-p; ToTensor + Normalize is ((x / 255) - mean) / std in fp32 with IEEE division.
static __global__ void __launch_bounds__(256)
augment_kernel(const AugmentArgs a) {
  pdl_prologue();
  const int64_t P = (int64_t)a.H * a.W, total = 2 * (int64_t)a.B * P;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = t / P, p = t - row * P, b = row >> 1;
    const int img = (int)(row & 1);
    const bool empty = a.total_a && (a.total_a[b * a.total_stride] == 0 || (a.total_b && a.total_b[b * a.total_stride] == 0));
    const uint8_t* prm = a.params + row * DDN_WS_PARAM_BYTES;
    const bool flip = !empty && prm[DDN_WS_FLIP];
    const bool rnd = !empty && a.randomize && prm[DDN_WS_RANDOMIZE];
    const int64_t q = flip ? P - 1 - p : p;
    const bool src_a = img == 0 || empty;         // an empty pair returns image A twice
    const uint8_t* rgb = (src_a ? a.rgb_a : a.rgb_b) + (b * P + q) * 3;
    const int m = (src_a ? a.mask_a : a.mask_b)[b * P + q];
    int v[3] = {rgb[0], rgb[1], rgb[2]};
    if (rnd) {
      const uint8_t* rgb1 = prm + DDN_WS_RGB1; const uint8_t* rgb2 = prm + DDN_WS_RGB2;
      double pp = 0.0;
      if (prm[DDN_WS_GRADIENT])
        pp = prm[DDN_WS_VERTICAL] ? linspace01((int)(q / a.W), a.H) : linspace01((int)(q % a.W), a.W);
      const uint8_t* n1 = a.noise + ((row * 2 + 0) * P + q) * 3;
      const uint8_t* n2 = a.noise + ((row * 2 + 1) * P + q) * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        // get_gradient_image: rgb2 * p + rgb1 * (1.0 - p) in fp64 (no FMA), truncated to uint8
        int R = prm[DDN_WS_GRADIENT] ? (int)__dadd_rn(__dmul_rn((double)rgb2[c], pp), __dmul_rn((double)rgb1[c], __dsub_rn(1.0, pp)))
                                     : (int)rgb1[c];
        if (prm[DDN_WS_NOISE]) R += (int)n1[c] - (int)n2[c];
        v[c] = (v[c] * m + ((1 - m) & 255) * (R & 255)) & 255;      // uint8 arithmetic modulo 256
      }
    }
    float* out = (img == 0 ? a.image_a : a.image_b) + b * 3 * P + p;
#pragma unroll
    for (int c = 0; c < 3; ++c) out[c * P] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)v[c], 255.f), a.mean[c]), a.std[c]);
    if (a.fmask) a.fmask[row * P + p] = (uint8_t)m;
    if (a.hit && img == 0) a.hit[b * P + p] = 0;
  }
}

}  // namespace ddn
