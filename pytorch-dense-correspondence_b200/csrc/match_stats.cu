// Per-match evaluation statistics on the device (SURVEY.md 8f row 4, the evaluation consumer of the backbone).
// Replaces DenseCorrespondenceEvaluation.compute_descriptor_match_statistics
// (dense_correspondence/evaluation/evaluation.py:1006-1178), which the reference runs in host numpy once per ground-truth
// match (up to 100 per image pair, evaluation.py:932-956), scanning the whole descriptor image of B several times per call.
//
// match_stats_scan_kernel: one block = one pixel range x a group of MS_GROUP consecutive queries.  When the group's queries
//   share an image pair (the usual pair-major order) a pixel's descriptor is loaded once and scored against all of them.
//   Per query and block it writes one partial record (best key, masked best, counts, distance sums, mask count).
// match_stats_finish_kernel: one thread per query adds its partial records in block order (so a second call is
//   bit-identical) and writes the reference's columns.
// L2/load bound like best_match_kernel; MS_GROUP queries read the image once instead of MS_GROUP times.
// best_match_batch_kernel: the same scan with the best match only, for the across-object analysis
//   (compute_descriptor_match_statistics_no_ground_truth, evaluation.py:977-1004): per block a 64-bit atomicMax of the
//   complemented key (order-independent, so deterministic), and the last block of each query group (bn_stats.cuh's
//   ticket) writes (u, v) and the distance.  One launch for every pair and query.
//
// Arithmetic, as the reference's numpy does it on a contiguous [H,W,D] float32 array (net.py:488-525):
//   nd(p) = sqrt(sum_c (res_b[p,c] - q_c)^2): each square rounded before it is added (no FMA), the sum in numpy's float32
//   pairwise order (D < 8: sequential from 0; else 8 running partials, ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the rest).
//   masked_nd = nd + (1 - mask_b) * 1e6 is float64 (mask_b is the dataset's uint8 array, evaluation.py:1053-1054), and so
//   are the masked comparison and the masked minimum.
#include <climits>
#include <cmath>
#include <initializer_list>
#include "bn_stats.cuh"
#include "common.cuh"

namespace ddn {

constexpr int MS_THREADS = 256;
constexpr int MS_GROUP = 8;
constexpr int MS_MAXD = 32;

struct MsPartial {
  unsigned long long key;  // (float bits of nd << 32) | pixel: first minimum of nd
  double mval;             // masked minimum and its pixel (first minimum)
  int32_t midx;
  int32_t cnt, cntm, mcnt;  // nd < t, masked_nd < t, nonzero mask pixels
  float thr;                // t = nd(uv_b): every block computes the same value
  double sum, summ;         // sum of pixel distances to uv_b over the two sets
};

struct MsKinv {
  double k[9];
};

struct MsImage {
  const float* base;
  int64_t sn, sh, sw, sc;
};

__device__ __forceinline__ bool ms_query_ok(int64_t n, int64_t ua, int64_t va, int64_t ub, int64_t vb, int N, int H, int W) {
  return n >= 0 && n < N && ua >= 0 && ua < W && va >= 0 && va < H && ub >= 0 && ub < W && vb >= 0 && vb < H;
}

// numpy float32 np.sum(np.square(x - q), axis=-1) over a contiguous last axis, then np.sqrt.
template <int KD>
__device__ __forceinline__ float ms_norm_diff(const float (&x)[KD], const float* q, int D) {
  float a[KD];
#pragma unroll
  for (int c = 0; c < KD; ++c) {
    const float d = __fsub_rn(x[c], q[c]);
    a[c] = c < D ? __fmul_rn(d, d) : 0.f;
  }
  float s;
  if (KD < 8 || D < 8) {
    s = 0.f;
#pragma unroll
    for (int c = 0; c < (KD < 8 ? KD : 8); ++c)
      if (c < D) s = __fadd_rn(s, a[c]);
  } else {
    float r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = a[j];
    const int full = D - D % 8;
#pragma unroll
    for (int i = 8; i < KD; i += 8)
      if (i < full) {
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = __fadd_rn(r[j], a[i + j]);
      }
    s = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])), __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
#pragma unroll
    for (int c = 8; c < KD; ++c)
      if (c >= full && c < D) s = __fadd_rn(s, a[c]);
  }
  return __fsqrt_rn(s);
}

template <int KD>
__device__ __forceinline__ void ms_load(const MsImage& im, int64_t n, int64_t v, int64_t u, int D, float (&x)[KD]) {
  const float* p = im.base + n * im.sn + v * im.sh + u * im.sw;
#pragma unroll
  for (int c = 0; c < KD; ++c) x[c] = c < D ? __ldg(p + c * im.sc) : 0.f;
}

// The full-image best-match scan (find_best_match, net.py:488-525) shared by every kernel here: each of this thread's
// pixels p in [p0, p1) is scored against the group's valid queries, and visit(j, p, v, u, nd, m) receives query j's
// distance nd(p) and, with MASK, mask_b at p (0 otherwise).  When the group's queries share an image pair (`uni`) a
// pixel's descriptor (and mask value) is loaded once for all of them.
template <int KD, bool MASK, typename Visit>
__device__ __forceinline__ void ms_scan_pixels(const MsImage& rb, const float* __restrict__ mask_b, int64_t P, int W, int D,
                                               int64_t p0, int64_t p1, const float (*qd)[KD], const int64_t* qn,
                                               const int* qok, bool uni, Visit&& visit) {
  for (int64_t p = p0 + threadIdx.x; p < p1; p += MS_THREADS) {
    const int64_t v = p / W, u = p - v * W;
    float x[KD];
    float m = 0.f;
    if (uni) {
      ms_load<KD>(rb, qn[0], v, u, D, x);
      if (MASK) m = __ldg(mask_b + qn[0] * P + p);
    }
#pragma unroll
    for (int j = 0; j < MS_GROUP; ++j) {
      if (!qok[j]) continue;
      if (!uni) {
        ms_load<KD>(rb, qn[j], v, u, D, x);
        if (MASK) m = __ldg(mask_b + qn[j] * P + p);
      }
      visit(j, p, v, u, ms_norm_diff<KD>(x, qd[j], D), m);
    }
  }
}

template <int KD>
__global__ void __launch_bounds__(MS_THREADS)
match_stats_scan_kernel(MsImage ra, MsImage rb, int N, int H, int W, int D,
                        const int64_t* __restrict__ pair, const int64_t* __restrict__ uv_a, const int64_t* __restrict__ uv_b,
                        int64_t Q, const float* __restrict__ mask_b, int pixels_per_block, MsPartial* __restrict__ part) {
  pdl_prologue();
  __shared__ float qd[MS_GROUP][KD];
  __shared__ float thr[MS_GROUP];
  __shared__ int64_t qn[MS_GROUP], qub[MS_GROUP], qvb[MS_GROUP];
  __shared__ int qok[MS_GROUP];
  __shared__ int uniform;
  const int64_t q0 = (int64_t)blockIdx.y * MS_GROUP;
  if (threadIdx.x < MS_GROUP) {
    const int j = threadIdx.x;
    const int64_t q = q0 + j;
    int ok = 0;
    if (q < Q) {
      const int64_t n = pair[q], ua = uv_a[2 * q], va = uv_a[2 * q + 1], ub = uv_b[2 * q], vb = uv_b[2 * q + 1];
      ok = ms_query_ok(n, ua, va, ub, vb, N, H, W);
      if (ok) {
        float x[KD];
        ms_load<KD>(ra, n, va, ua, D, x);
#pragma unroll
        for (int c = 0; c < KD; ++c) qd[j][c] = x[c];
        ms_load<KD>(rb, n, vb, ub, D, x);
        thr[j] = ms_norm_diff<KD>(x, qd[j], D);   // t = nd(uv_b), the same arithmetic as every other pixel
        qn[j] = n; qub[j] = ub; qvb[j] = vb;
      }
    }
    qok[j] = ok;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int u = qok[0];
    for (int j = 1; j < MS_GROUP; ++j) u &= (!qok[j] || qn[j] == qn[0]);
    uniform = u;
  }
  __syncthreads();
  const bool uni = uniform;
  const int64_t P = (int64_t)H * W;
  const int64_t p0 = (int64_t)blockIdx.x * pixels_per_block;
  const int64_t p1 = min(P, p0 + pixels_per_block);

  unsigned long long key[MS_GROUP];
  double mval[MS_GROUP], sum[MS_GROUP], summ[MS_GROUP];
  int midx[MS_GROUP], cnt[MS_GROUP], cntm[MS_GROUP], mcnt[MS_GROUP];
#pragma unroll
  for (int j = 0; j < MS_GROUP; ++j) {
    key[j] = ~0ull; mval[j] = INFINITY; midx[j] = INT_MAX; cnt[j] = cntm[j] = mcnt[j] = 0; sum[j] = summ[j] = 0.0;
  }
  ms_scan_pixels<KD, true>(rb, mask_b, P, W, D, p0, p1, qd, qn, qok, uni,
                           [&](int j, int64_t p, int64_t v, int64_t u, float nd, float m) {
    const unsigned long long k = ((unsigned long long)__float_as_uint(nd) << 32) | (unsigned long long)(uint32_t)p;
    key[j] = k < key[j] ? k : key[j];
    const double md = __dadd_rn((double)nd, __dmul_rn(__dsub_rn(1.0, (double)m), 1e6));
    if (md < mval[j]) { mval[j] = md; midx[j] = (int)p; }      // pixels rise along a thread: strict < keeps the first
    const float t = thr[j];
    const bool c1 = nd < t, c2 = md < (double)t;
    if (c1 || c2) {
      const int64_t du = u - qub[j], dv = v - qvb[j];
      const double dist = __dsqrt_rn((double)(du * du + dv * dv));
      if (c1) { cnt[j] += 1; sum[j] = __dadd_rn(sum[j], dist); }
      if (c2) { cntm[j] += 1; summ[j] = __dadd_rn(summ[j], dist); }
    }
    mcnt[j] += m != 0.f;
  });

  // block reduction in a fixed order: xor-shuffle tree inside each warp, then the warps in index order
  __shared__ MsPartial red[MS_THREADS / 32][MS_GROUP];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int j = 0; j < MS_GROUP; ++j) {
    if (!qok[j]) continue;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long ok = __shfl_xor_sync(0xffffffffu, key[j], o);
      key[j] = ok < key[j] ? ok : key[j];
      const double om = __shfl_xor_sync(0xffffffffu, mval[j], o);
      const int oi = __shfl_xor_sync(0xffffffffu, midx[j], o);
      if (om < mval[j] || (om == mval[j] && oi < midx[j])) { mval[j] = om; midx[j] = oi; }
      cnt[j] += __shfl_xor_sync(0xffffffffu, cnt[j], o);
      cntm[j] += __shfl_xor_sync(0xffffffffu, cntm[j], o);
      mcnt[j] += __shfl_xor_sync(0xffffffffu, mcnt[j], o);
      sum[j] = __dadd_rn(sum[j], __shfl_xor_sync(0xffffffffu, sum[j], o));
      summ[j] = __dadd_rn(summ[j], __shfl_xor_sync(0xffffffffu, summ[j], o));
    }
    if (lane == 0) {
      MsPartial r;
      r.key = key[j]; r.mval = mval[j]; r.midx = midx[j]; r.cnt = cnt[j]; r.cntm = cntm[j]; r.mcnt = mcnt[j];
      r.sum = sum[j]; r.summ = summ[j]; r.thr = thr[j];
      red[warp][j] = r;
    }
  }
  __syncthreads();
  if (threadIdx.x < MS_GROUP && qok[threadIdx.x]) {
    const int j = threadIdx.x;
    MsPartial r = red[0][j];
    for (int w = 1; w < MS_THREADS / 32; ++w) {
      const MsPartial& o = red[w][j];
      r.key = o.key < r.key ? o.key : r.key;
      if (o.mval < r.mval || (o.mval == r.mval && o.midx < r.midx)) { r.mval = o.mval; r.midx = o.midx; }
      r.cnt += o.cnt; r.cntm += o.cntm; r.mcnt += o.mcnt;
      r.sum = __dadd_rn(r.sum, o.sum); r.summ = __dadd_rn(r.summ, o.summ);
    }
    part[(q0 + j) * gridDim.x + blockIdx.x] = r;
  }
}

__device__ __forceinline__ bool ms_depth_valid(double d) { return d > 0.0 && d < 10.0; }   // evaluation.py:960-972

// compute_3d_position (evaluation.py:1180-1200) with pinhole_projection_image_to_world (correspondence_finder.py:123-144):
// camera_to_world . (z * K^-1 . (u, v, 1), 1), called with (u, v) as the reference does (its docstring says (row, column)).
__device__ __forceinline__ void ms_position(const MsKinv& ki, const double* T, int64_t u, int64_t v, double z, double* out) {
  double c[3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
    c[i] = __dmul_rn(z, __dadd_rn(__dadd_rn(__dmul_rn(ki.k[3 * i], (double)u), __dmul_rn(ki.k[3 * i + 1], (double)v)), ki.k[3 * i + 2]));
#pragma unroll
  for (int i = 0; i < 3; ++i)
    out[i] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[4 * i], c[0]), __dmul_rn(T[4 * i + 1], c[1])), __dmul_rn(T[4 * i + 2], c[2])),
                       T[4 * i + 3]);
}

__device__ __forceinline__ double ms_dist3(const double* a, const double* b) {
  const double x = __dsub_rn(a[0], b[0]), y = __dsub_rn(a[1], b[1]), z = __dsub_rn(a[2], b[2]);
  return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)));
}

__device__ __forceinline__ void ms_bad_row(float* f32, double* f64, int64_t* i64, unsigned long long* bad) {
  for (int i = 0; i < DDN_MS_NF32; ++i) f32[i] = NAN;
  for (int i = 0; i < DDN_MS_NF64; ++i) f64[i] = NAN;
  for (int i = 0; i < DDN_MS_NI64; ++i) i64[i] = -1;
  atomicAdd(bad, 1ull);
}

__global__ void match_stats_finish_kernel(const MsPartial* __restrict__ part, int nblk, int N, int H, int W,
                                          const int64_t* __restrict__ pair, const int64_t* __restrict__ uv_a,
                                          const int64_t* __restrict__ uv_b, int64_t Q,
                                          const float* __restrict__ depth_a, const float* __restrict__ depth_b, MsKinv ki,
                                          const double* __restrict__ poses_a, const double* __restrict__ poses_b,
                                          float* __restrict__ of32, double* __restrict__ of64, int64_t* __restrict__ oi64,
                                          unsigned long long* __restrict__ bad) {
  pdl_prologue();
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= Q) return;
  float* f32 = of32 + q * DDN_MS_NF32;
  double* f64 = of64 + q * DDN_MS_NF64;
  int64_t* i64 = oi64 + q * DDN_MS_NI64;
  const int64_t n = pair[q], ua = uv_a[2 * q], va = uv_a[2 * q + 1], ub = uv_b[2 * q], vb = uv_b[2 * q + 1];
  if (!ms_query_ok(n, ua, va, ub, vb, N, H, W)) {
    ms_bad_row(f32, f64, i64, bad);
    return;
  }
  MsPartial r = part[q * nblk];
  for (int b = 1; b < nblk; ++b) {
    const MsPartial& o = part[q * nblk + b];
    r.key = o.key < r.key ? o.key : r.key;
    if (o.mval < r.mval || (o.mval == r.mval && o.midx < r.midx)) { r.mval = o.mval; r.midx = o.midx; }
    r.cnt += o.cnt; r.cntm += o.cntm; r.mcnt += o.mcnt;
    r.sum = __dadd_rn(r.sum, o.sum); r.summ = __dadd_rn(r.summ, o.summ);
  }
  const uint32_t pb = (uint32_t)(r.key & 0xffffffffull);
  const int64_t P = (int64_t)H * W;
  if (r.midx >= P) {      // every masked distance was NaN (NaN descriptors): no masked minimum, and no pixel to read
    ms_bad_row(f32, f64, i64, bad);
    return;
  }
  const int64_t up = pb % W, vp = pb / W, upm = r.midx % W, vpm = r.midx / W;

  // pixel errors (evaluation.py:1062-1064): exact integers, one rounding in the sqrt
  const int64_t du = ub - up, dv = vb - vp, dum = ub - upm, dvm = vb - vpm;
  f64[DDN_MS_PIXEL_MATCH_ERROR_L2] = __dsqrt_rn((double)(du * du + dv * dv));
  f64[DDN_MS_PIXEL_MATCH_ERROR_L2_MASKED] = __dsqrt_rn((double)(dum * dum + dvm * dvm));
  f64[DDN_MS_PIXEL_MATCH_ERROR_L1] = (double)((du < 0 ? -du : du) + (dv < 0 ? -dv : dv));
  f32[DDN_MS_NORM_DIFF_DESCRIPTOR_GROUND_TRUTH] = r.thr;
  f32[DDN_MS_NORM_DIFF_DESCRIPTOR] = __uint_as_float((uint32_t)(r.key >> 32));
  f64[DDN_MS_NORM_DIFF_DESCRIPTOR_MASKED] = r.mval;
  // fractions and averages (evaluation.py:1078-1100); an empty mask divides by zero: NaN here, ZeroDivisionError upstream
  f64[DDN_MS_FRACTION_CLOSER] = __ddiv_rn((double)r.cnt, (double)P);
  f64[DDN_MS_FRACTION_CLOSER_MASKED] = r.mcnt ? __ddiv_rn((double)r.cntm, (double)r.mcnt) : (double)NAN;
  f64[DDN_MS_AVERAGE_L2_FALSE_POSITIVES] = r.cnt ? __ddiv_rn(r.sum, (double)r.cnt) : 0.0;
  f64[DDN_MS_AVERAGE_L2_FALSE_POSITIVES_MASKED] = r.cntm ? __ddiv_rn(r.summ, (double)r.cntm) : 0.0;
  // depths in metres (DEPTH_IM_SCALE = 1000.0) and 3-D errors (evaluation.py:1103-1135); the depth at uv_a is never checked
  const double za = __ddiv_rn((double)depth_a[n * P + va * W + ua], 1000.0);
  const double zb = __ddiv_rn((double)depth_b[n * P + vb * W + ub], 1000.0);
  const double zp = __ddiv_rn((double)depth_b[n * P + vp * W + up], 1000.0);
  const double zpm = __ddiv_rn((double)depth_b[n * P + vpm * W + upm], 1000.0);
  const double* Ta = poses_a + n * 16;
  const double* Tb = poses_b + n * 16;
  double pa[3], pbp[3], pp[3], ppm[3];
  ms_position(ki, Ta, ua, va, za, pa);
  ms_position(ki, Tb, ub, vb, zb, pbp);
  ms_position(ki, Tb, up, vp, zp, pp);
  ms_position(ki, Tb, upm, vpm, zpm, ppm);
  const bool vb_ok = ms_depth_valid(zb), vp_ok = ms_depth_valid(zp), vpm_ok = ms_depth_valid(zpm);
  f64[DDN_MS_NORM_DIFF_GROUND_TRUTH_3D] = vb_ok ? ms_dist3(pbp, pa) : (double)NAN;
  f64[DDN_MS_NORM_DIFF_PRED_3D] = vb_ok && vp_ok ? ms_dist3(pbp, pp) : (double)NAN;
  f64[DDN_MS_NORM_DIFF_PRED_3D_MASKED] = vb_ok && vpm_ok ? ms_dist3(pbp, ppm) : (double)NAN;
  i64[DDN_MS_IS_VALID] = vp_ok;
  i64[DDN_MS_IS_VALID_MASKED] = vpm_ok;
  i64[DDN_MS_U_PRED] = up; i64[DDN_MS_V_PRED] = vp;
  i64[DDN_MS_U_PRED_MASKED] = upm; i64[DDN_MS_V_PRED_MASKED] = vpm;
  i64[DDN_MS_NUM_CLOSER] = r.cnt; i64[DDN_MS_NUM_CLOSER_MASKED] = r.cntm; i64[DDN_MS_NUM_MASK_PIXELS] = r.mcnt;
}

// best[q] holds ~key (zero on entry: no candidate yet), ticket[group] zero on entry; both are left as the caller zeroed them
// except that the tickets return to zero.  A query whose pair or pixel is out of range gets (-1, -1), NaN and is counted.
template <int KD>
__global__ void __launch_bounds__(MS_THREADS)
best_match_batch_kernel(MsImage ra, MsImage rb, int N, int H, int W, int D, const int64_t* __restrict__ pair,
                        const int64_t* __restrict__ uv_a, int64_t Q, int pixels_per_block, unsigned long long* __restrict__ best,
                        unsigned int* __restrict__ ticket, int64_t* __restrict__ out_uv, float* __restrict__ out_diff,
                        unsigned long long* __restrict__ bad) {
  pdl_prologue();
  __shared__ float qd[MS_GROUP][KD];
  __shared__ int64_t qn[MS_GROUP];
  __shared__ int qok[MS_GROUP];
  __shared__ int uniform, last;
  const int64_t q0 = (int64_t)blockIdx.y * MS_GROUP;
  if (threadIdx.x < MS_GROUP) {
    const int j = threadIdx.x;
    const int64_t q = q0 + j;
    int ok = 0;
    if (q < Q) {
      const int64_t n = pair[q], ua = uv_a[2 * q], va = uv_a[2 * q + 1];
      ok = ms_query_ok(n, ua, va, 0, 0, N, H, W);
      if (ok) {
        float x[KD];
        ms_load<KD>(ra, n, va, ua, D, x);
#pragma unroll
        for (int c = 0; c < KD; ++c) qd[j][c] = x[c];
        qn[j] = n;
      }
    }
    qok[j] = ok;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int u = qok[0];
    for (int j = 1; j < MS_GROUP; ++j) u &= (!qok[j] || qn[j] == qn[0]);
    uniform = u;
  }
  __syncthreads();
  const int64_t P = (int64_t)H * W;
  const int64_t p0 = (int64_t)blockIdx.x * pixels_per_block;
  const int64_t p1 = min(P, p0 + pixels_per_block);
  unsigned long long key[MS_GROUP];
#pragma unroll
  for (int j = 0; j < MS_GROUP; ++j) key[j] = ~0ull;
  ms_scan_pixels<KD, false>(rb, nullptr, P, W, D, p0, p1, qd, qn, qok, uniform != 0,
                            [&](int j, int64_t p, int64_t, int64_t, float nd, float) {
    const unsigned long long k = ((unsigned long long)__float_as_uint(nd) << 32) | (unsigned long long)(uint32_t)p;
    key[j] = k < key[j] ? k : key[j];
  });
  __shared__ unsigned long long red[MS_THREADS / 32][MS_GROUP];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int j = 0; j < MS_GROUP; ++j) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long other = __shfl_xor_sync(0xffffffffu, key[j], o);
      key[j] = other < key[j] ? other : key[j];
    }
    if (lane == 0) red[warp][j] = key[j];
  }
  __syncthreads();
  if (threadIdx.x < MS_GROUP && qok[threadIdx.x]) {
    unsigned long long k = red[0][threadIdx.x];
    for (int w = 1; w < MS_THREADS / 32; ++w) k = red[w][threadIdx.x] < k ? red[w][threadIdx.x] : k;
    if (k != ~0ull) atomicMax(best + q0 + threadIdx.x, ~k);
  }
  if (!bn_last_cta(ticket + blockIdx.y, gridDim.x, threadIdx.x == 0, &last, [] { __syncthreads(); })) return;
  if (threadIdx.x < MS_GROUP) {
    const int64_t q = q0 + threadIdx.x;
    if (q >= Q) return;
    if (!qok[threadIdx.x]) {
      out_uv[2 * q] = -1; out_uv[2 * q + 1] = -1; out_diff[q] = NAN;
      atomicAdd(bad, 1ull);
      return;
    }
    const unsigned long long k = ~__ldcg(best + q);
    const uint32_t p = (uint32_t)(k & 0xffffffffull);
    out_uv[2 * q] = p % W;          // u = column
    out_uv[2 * q + 1] = p / W;      // v = row
    out_diff[q] = __uint_as_float((uint32_t)(k >> 32));
  }
}

// The pixel split depends on H*W alone, so the scratch size needs no device query.
static int ms_blocks_x(int64_t P, int* ppb) {
  int nb = (int)std::min<int64_t>(64, std::max<int64_t>(1, ceil_div(P, 4096)));
  *ppb = (int)(ceil_div(ceil_div(P, nb), MS_THREADS) * MS_THREADS);
  return (int)ceil_div(P, *ppb);
}

static size_t ms_scratch_bytes(int N, int64_t P, int64_t Q) {
  int ppb;
  const int nb = ms_blocks_x(P, &ppb);
  return align_up(sizeof(double) * 32 * (size_t)N, 256) + sizeof(MsPartial) * (size_t)nb * (size_t)ceil_div(Q, MS_GROUP) * MS_GROUP;
}

}  // namespace ddn

using namespace ddn;

static bool ms_sizes_ok(int N, int H, int W, int64_t Q) {
  return N >= 1 && N <= DDN_MS_MAX_PAIRS && H >= 1 && W >= 1 && (int64_t)H * W < (1ll << 31) && Q >= 1 &&
         Q <= DDN_MS_MAX_QUERIES;
}

extern "C" size_t ddn_match_statistics_scratch_bytes(int N, int H, int W, int64_t Q) {
  if (!ms_sizes_ok(N, H, W, Q)) {
    set_error("ddn_match_statistics_scratch_bytes: bad sizes (N %d, H %d, W %d, Q %lld)", N, H, W, (long long)Q);
    return 0;
  }
  return ms_scratch_bytes(N, (int64_t)H * W, Q);
}

extern "C" int ddn_match_statistics(const float* res_a, const int64_t* strides_a_host, const float* res_b,
                                    const int64_t* strides_b_host, int N, int H, int W, int D,
                                    const int64_t* pair, const int64_t* uv_a, const int64_t* uv_b, int64_t Q,
                                    const float* mask_b, const float* depth_a, const float* depth_b,
                                    const double* K_inv_host, const double* poses_a_host, const double* poses_b_host,
                                    float* out_f32, double* out_f64, int64_t* out_i64, int64_t* bad_queries,
                                    void* scratch, size_t scratch_bytes, void* stream) {
  DDN_CHECK_ARG(res_a && res_b && strides_a_host && strides_b_host && pair && uv_a && uv_b && mask_b && depth_a && depth_b &&
                K_inv_host && poses_a_host && poses_b_host && out_f32 && out_f64 && out_i64 && bad_queries && scratch,
                "ddn_match_statistics: null argument");
  DDN_CHECK_ARG(D >= 1 && D <= MS_MAXD, "ddn_match_statistics: descriptor dimension %d outside 1..%d", D, MS_MAXD);
  DDN_CHECK_ARG(ms_sizes_ok(N, H, W, Q), "ddn_match_statistics: bad sizes (N %d in 1..%d, H*W < 2^31, Q %lld in 1..%d)", N,
                DDN_MS_MAX_PAIRS, (long long)Q, DDN_MS_MAX_QUERIES);
  const int64_t ext[4] = {N, H, W, D};
  for (const int64_t* s : {strides_a_host, strides_b_host}) {
    int64_t last = 0;
    for (int i = 0; i < 4; ++i) {
      DDN_CHECK_ARG(s[i] >= 0 && s[i] < (1ll << 40), "ddn_match_statistics: stride %lld out of range", (long long)s[i]);
      last += (ext[i] - 1) * s[i];
    }
    DDN_CHECK_ARG(last < (1ll << 40), "ddn_match_statistics: strides address more than 2^40 elements");
  }
  const int64_t P = (int64_t)H * W;
  DDN_CHECK_ARG(scratch_bytes >= ms_scratch_bytes(N, P, Q), "ddn_match_statistics: scratch %zu < %zu bytes", scratch_bytes,
                ms_scratch_bytes(N, P, Q));
  cudaStream_t st = (cudaStream_t)stream;
  double* poses = reinterpret_cast<double*>(scratch);
  MsPartial* part = reinterpret_cast<MsPartial*>(reinterpret_cast<char*>(scratch) + align_up(sizeof(double) * 32 * (size_t)N, 256));
  // pageable host -> device: staged at once, so the caller may free its arrays when this returns
  DDN_CUDA(cudaMemcpyAsync(poses, poses_a_host, sizeof(double) * 16 * N, cudaMemcpyHostToDevice, st));
  DDN_CUDA(cudaMemcpyAsync(poses + 16 * N, poses_b_host, sizeof(double) * 16 * N, cudaMemcpyHostToDevice, st));
  DDN_CUDA(cudaMemsetAsync(bad_queries, 0, sizeof(int64_t), st));
  MsKinv ki;
  for (int i = 0; i < 9; ++i) ki.k[i] = K_inv_host[i];
  const MsImage ia{res_a, strides_a_host[0], strides_a_host[1], strides_a_host[2], strides_a_host[3]};
  const MsImage ib{res_b, strides_b_host[0], strides_b_host[1], strides_b_host[2], strides_b_host[3]};
  int ppb;
  const int nb = ms_blocks_x(P, &ppb);
  dim3 grid(nb, (unsigned)ceil_div(Q, MS_GROUP));
  if (D <= 8)
    DDN_LAUNCH(match_stats_scan_kernel<8>, grid, MS_THREADS, 0, st, ia, ib, N, H, W, D, pair, uv_a, uv_b, Q, mask_b, ppb, part);
  else if (D <= 16)
    DDN_LAUNCH(match_stats_scan_kernel<16>, grid, MS_THREADS, 0, st, ia, ib, N, H, W, D, pair, uv_a, uv_b, Q, mask_b, ppb, part);
  else
    DDN_LAUNCH(match_stats_scan_kernel<32>, grid, MS_THREADS, 0, st, ia, ib, N, H, W, D, pair, uv_a, uv_b, Q, mask_b, ppb, part);
  DDN_LAUNCH(match_stats_finish_kernel, (unsigned)ceil_div(Q, 128), 128, 0, st, part, nb, N, H, W, pair, uv_a, uv_b, Q, depth_a,
             depth_b, ki, poses, poses + 16 * N, out_f32, out_f64, out_i64, reinterpret_cast<unsigned long long*>(bad_queries));
  return 0;
}

static bool bm_sizes_ok(int N, int H, int W, int64_t Q) {
  return N >= 1 && N <= DDN_MS_MAX_PAIRS && H >= 1 && W >= 1 && (int64_t)H * W < (1ll << 31) && Q >= 1 &&
         Q <= DDN_BM_MAX_QUERIES;
}

// [groups * MS_GROUP] complemented keys, then [groups] tickets
static size_t bm_scratch_bytes(int64_t Q) {
  const int64_t groups = ceil_div(Q, MS_GROUP);
  return sizeof(unsigned long long) * (size_t)(groups * MS_GROUP) + align_up(sizeof(unsigned int) * (size_t)groups, 256);
}

extern "C" size_t ddn_best_match_batch_scratch_bytes(int64_t Q) {
  if (Q < 1 || Q > DDN_BM_MAX_QUERIES) {
    set_error("ddn_best_match_batch_scratch_bytes: Q %lld outside 1..%d", (long long)Q, DDN_BM_MAX_QUERIES);
    return 0;
  }
  return bm_scratch_bytes(Q);
}

extern "C" int ddn_best_match_batch(const float* res_a, const int64_t* strides_a_host, const float* res_b,
                                    const int64_t* strides_b_host, int N, int H, int W, int D, const int64_t* pair,
                                    const int64_t* uv_a, int64_t Q, int64_t* best_uv, float* best_diff, int64_t* bad_queries,
                                    void* scratch, size_t scratch_bytes, void* stream) {
  DDN_CHECK_ARG(res_a && res_b && strides_a_host && strides_b_host && pair && uv_a && best_uv && best_diff && bad_queries &&
                scratch, "ddn_best_match_batch: null argument");
  DDN_CHECK_ARG(D >= 1 && D <= MS_MAXD, "ddn_best_match_batch: descriptor dimension %d outside 1..%d", D, MS_MAXD);
  DDN_CHECK_ARG(bm_sizes_ok(N, H, W, Q), "ddn_best_match_batch: bad sizes (N %d in 1..%d, H*W < 2^31, Q %lld in 1..%d)", N,
                DDN_MS_MAX_PAIRS, (long long)Q, DDN_BM_MAX_QUERIES);
  const int64_t ext[4] = {N, H, W, D};
  for (const int64_t* s : {strides_a_host, strides_b_host}) {
    int64_t last = 0;
    for (int i = 0; i < 4; ++i) {
      DDN_CHECK_ARG(s[i] >= 0 && s[i] < (1ll << 40), "ddn_best_match_batch: stride %lld out of range", (long long)s[i]);
      last += (ext[i] - 1) * s[i];
    }
    DDN_CHECK_ARG(last < (1ll << 40), "ddn_best_match_batch: strides address more than 2^40 elements");
  }
  DDN_CHECK_ARG(scratch_bytes >= bm_scratch_bytes(Q), "ddn_best_match_batch: scratch %zu < %zu bytes", scratch_bytes,
                bm_scratch_bytes(Q));
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t groups = ceil_div(Q, MS_GROUP);
  unsigned long long* best = reinterpret_cast<unsigned long long*>(scratch);
  unsigned int* ticket = reinterpret_cast<unsigned int*>(best + groups * MS_GROUP);
  DDN_CUDA(cudaMemsetAsync(scratch, 0, bm_scratch_bytes(Q), st));
  DDN_CUDA(cudaMemsetAsync(bad_queries, 0, sizeof(int64_t), st));
  const MsImage ia{res_a, strides_a_host[0], strides_a_host[1], strides_a_host[2], strides_a_host[3]};
  const MsImage ib{res_b, strides_b_host[0], strides_b_host[1], strides_b_host[2], strides_b_host[3]};
  int ppb;
  const int nb = ms_blocks_x((int64_t)H * W, &ppb);
  dim3 grid(nb, (unsigned)groups);
  unsigned long long* bad = reinterpret_cast<unsigned long long*>(bad_queries);
  if (D <= 8)
    DDN_LAUNCH(best_match_batch_kernel<8>, grid, MS_THREADS, 0, st, ia, ib, N, H, W, D, pair, uv_a, Q, ppb, best, ticket, best_uv,
               best_diff, bad);
  else if (D <= 16)
    DDN_LAUNCH(best_match_batch_kernel<16>, grid, MS_THREADS, 0, st, ia, ib, N, H, W, D, pair, uv_a, Q, ppb, best, ticket, best_uv,
               best_diff, bad);
  else
    DDN_LAUNCH(best_match_batch_kernel<32>, grid, MS_THREADS, 0, st, ia, ib, N, H, W, D, pair, uv_a, Q, ppb, best, ticket, best_uv,
               best_diff, bad);
  return 0;
}
