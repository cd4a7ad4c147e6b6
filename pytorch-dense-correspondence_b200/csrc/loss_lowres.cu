// Pixelwise contrastive loss fused with the 8x bilinear upsample that precedes it.
//
// The reference evaluates the loss on the full-resolution descriptor image y = upsample_bilinear(low) (resnet_dilated.py:320,
// pixelwise_contrastive_loss.py:131-213): a few thousand descriptors are gathered out of 1.23*D MB per image, and autograd
// scatters their gradients into a zero-filled tensor of that size which the upsample backward then reads in full.  A descriptor
// at pixel (u, v) is a fixed bilinear blend of 4 cells of the LOW-resolution map (60 x 80 x D per image, NHWC here: a cell's D
// channels are one contiguous 4*D-byte row), and that map -- 0.3*D MB for a batch of 16 -- lives in L2.  So these kernels
//   forward : read the two indices of a pair from HBM, 2 x 4 low-resolution cells from L2, blend (the same fp32 arithmetic as
//             upsample_fwd_kernel), squared distance / hinge / count / reduce -- the full-resolution image is never touched;
//   backward: scatter coef * d(l_j)/d(descriptor) * blend weights straight into d(low) (fp64 reds into an L2-resident
//             array, so that the order in which pairs arrive cannot change the fp32 result: a step's gradient is the same
//             on every run), runs of equal A indices folded by a segmented warp reduction first -- no zero-filled
//             full-resolution gradient, no pass of the upsample backward over it.
// HBM traffic per index pair drops from 16 + 8*D algorithmic bytes (and 8 + 64*D bytes of 32-byte sectors actually moved by
// the channel-strided NCHW gather) to the 16 bytes of the two indices.
//
// Descriptor images: low_a / low_b [B, h*w, D] fp32 (what ddn_resnet34_8s_forward writes to `low_nhwc_out`).
//
// UNIT = true (DDN_LOWRES_UNIT): the descriptor is the blend x normalised to unit length, y = x / ||x||, which is what the
// reference's `normalize` option computes per output pixel after its upsample (dense_correspondence_network.py:256-259).  The
// forward scores y; the backward applies the normalisation's Jacobian dx = (g - y (y.g)) / ||x|| to each side's gradient g
// before the scatter (||x|| recomputed from the 4 cells, nothing stored).  A zero blend gives NaN, as x / ||x|| does in fp32.
#include "bn_stats.cuh"
#include "loss.cuh"

namespace ddn {

constexpr int LR_THREADS = 128;      // small CTAs: the kernels are a single L2 round trip per pair; balance beats reuse

// bilinear source cell + weights of output pixel (u, v): identical arithmetic to head.cu::src_index / upsample_fwd_kernel
struct Blend { int c00, c01, c10, c11; float lh, lw; };
__device__ __forceinline__ Blend blend_of(int64_t n, int W, int h, int w, float sh, float sw) {
  // 0 <= n < H * W < 2^31 (checked by the callers): a 32-bit division -- the 64-bit one is ~80 instructions, and these kernels are
  // instruction-bound (ncu: issue slots 45 % / 65 % busy at C3, DRAM 7 % / 10 %)
  const unsigned ni = (unsigned)n;
  const int v = (int)(ni / (unsigned)W), u = (int)(ni - (unsigned)v * (unsigned)W);
  float r = sh * (float)v;
  int h0 = (int)r; if (h0 > h - 1) h0 = h - 1;
  const int h1 = h0 + ((h0 < h - 1) ? 1 : 0);
  Blend b;
  b.lh = r - (float)h0;
  r = sw * (float)u;
  int w0 = (int)r; if (w0 > w - 1) w0 = w - 1;
  const int w1 = w0 + ((w0 < w - 1) ? 1 : 0);
  b.lw = r - (float)w0;
  b.c00 = h0 * w + w0; b.c01 = h0 * w + w1; b.c10 = h1 * w + w0; b.c11 = h1 * w + w1;
  return b;
}
__device__ __forceinline__ float blend1(float x00, float x01, float x10, float x11, float lh, float lw) {
  const float top = (1.f - lw) * x00 + lw * x01;
  const float bot = (1.f - lw) * x10 + lw * x11;
  return (1.f - lh) * top + lh * bot;
}

// descriptor difference a - b of one pair into d[0..D): D_T > 0 = compile-time D (all 8 * D/4 vector loads are independent and
// issued back to back: one L2 round trip per pair instead of D/4), D_T = 0 = run-time D (scalar loads, any D <= 32)
template <int D_T>
__device__ __forceinline__ void descriptor_diff(const float* __restrict__ A, const float* __restrict__ Bq, const Blend& ba, const Blend& bb,
                                                int D_rt, float (&d)[D_T > 0 ? D_T : LOSS_MAXD]) {
  constexpr int DM = D_T > 0 ? D_T : LOSS_MAXD;
  const int D = D_T > 0 ? D_T : D_rt;
  const float* a00 = A + (size_t)ba.c00 * D; const float* a01 = A + (size_t)ba.c01 * D;
  const float* a10 = A + (size_t)ba.c10 * D; const float* a11 = A + (size_t)ba.c11 * D;
  const float* b00 = Bq + (size_t)bb.c00 * D; const float* b01 = Bq + (size_t)bb.c01 * D;
  const float* b10 = Bq + (size_t)bb.c10 * D; const float* b11 = Bq + (size_t)bb.c11 * D;
  if (D_T > 0 && D_T % 4 == 0) {
    float4 va[D_T / 4 > 0 ? D_T / 4 : 1][4], vb[D_T / 4 > 0 ? D_T / 4 : 1][4];
#pragma unroll
    for (int q = 0; q < D_T / 4; ++q) {
      va[q][0] = __ldg(reinterpret_cast<const float4*>(a00) + q); va[q][1] = __ldg(reinterpret_cast<const float4*>(a01) + q);
      va[q][2] = __ldg(reinterpret_cast<const float4*>(a10) + q); va[q][3] = __ldg(reinterpret_cast<const float4*>(a11) + q);
      vb[q][0] = __ldg(reinterpret_cast<const float4*>(b00) + q); vb[q][1] = __ldg(reinterpret_cast<const float4*>(b01) + q);
      vb[q][2] = __ldg(reinterpret_cast<const float4*>(b10) + q); vb[q][3] = __ldg(reinterpret_cast<const float4*>(b11) + q);
    }
#pragma unroll
    for (int q = 0; q < D_T / 4; ++q) {
      d[4 * q + 0] = blend1(va[q][0].x, va[q][1].x, va[q][2].x, va[q][3].x, ba.lh, ba.lw) - blend1(vb[q][0].x, vb[q][1].x, vb[q][2].x, vb[q][3].x, bb.lh, bb.lw);
      d[4 * q + 1] = blend1(va[q][0].y, va[q][1].y, va[q][2].y, va[q][3].y, ba.lh, ba.lw) - blend1(vb[q][0].y, vb[q][1].y, vb[q][2].y, vb[q][3].y, bb.lh, bb.lw);
      d[4 * q + 2] = blend1(va[q][0].z, va[q][1].z, va[q][2].z, va[q][3].z, ba.lh, ba.lw) - blend1(vb[q][0].z, vb[q][1].z, vb[q][2].z, vb[q][3].z, bb.lh, bb.lw);
      d[4 * q + 3] = blend1(va[q][0].w, va[q][1].w, va[q][2].w, va[q][3].w, ba.lh, ba.lw) - blend1(vb[q][0].w, vb[q][1].w, vb[q][2].w, vb[q][3].w, bb.lh, bb.lw);
    }
  } else {
#pragma unroll
    for (int c = 0; c < DM; ++c) {
      d[c] = 0.f;
      if (c < D)
        d[c] = blend1(__ldg(a00 + c), __ldg(a01 + c), __ldg(a10 + c), __ldg(a11 + c), ba.lh, ba.lw) -
               blend1(__ldg(b00 + c), __ldg(b01 + c), __ldg(b10 + c), __ldg(b11 + c), bb.lh, bb.lw);
    }
  }
}

// one side's blended descriptor x[0..D) of pixel `bl` (the arithmetic of descriptor_diff), channels >= D zero
template <int D_T>
__device__ __forceinline__ void descriptor_blend(const float* __restrict__ A, const Blend& bl, int D_rt, float (&x)[D_T > 0 ? D_T : LOSS_MAXD]) {
  constexpr int DM = D_T > 0 ? D_T : LOSS_MAXD;
  const int D = D_T > 0 ? D_T : D_rt;
  const float* a00 = A + (size_t)bl.c00 * D; const float* a01 = A + (size_t)bl.c01 * D;
  const float* a10 = A + (size_t)bl.c10 * D; const float* a11 = A + (size_t)bl.c11 * D;
#pragma unroll
  for (int c = 0; c < DM; ++c) {
    x[c] = 0.f;
    if (c < D) x[c] = blend1(__ldg(a00 + c), __ldg(a01 + c), __ldg(a10 + c), __ldg(a11 + c), bl.lh, bl.lw);
  }
}

// x <- x / ||x|| over channels [0, D); returns ||x|| (0 gives NaN descriptors, as the division does)
template <int DM>
__device__ __forceinline__ float unit_normalize(float (&x)[DM], int D) {
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < DM; ++c) s = fmaf(x[c], x[c], s);
  const float n = sqrtf(s);
#pragma unroll
  for (int c = 0; c < DM; ++c)
    if (c < D) x[c] = x[c] / n;
  return n;
}

// g <- (g - y (y.g)) / n: the vector-Jacobian product of y = x / ||x|| with n = ||x||
template <int DM>
__device__ __forceinline__ void unit_vjp(float (&g)[DM], const float (&y)[DM], float n, int D) {
  float t = 0.f;
#pragma unroll
  for (int c = 0; c < DM; ++c)
    if (c < D) t = fmaf(y[c], g[c], t);
#pragma unroll
  for (int c = 0; c < DM; ++c)
    if (c < D) g[c] = (g[c] - y[c] * t) / n;
}

// unit descriptors of both sides and their difference d = ya - yb
template <int D_T>
__device__ __forceinline__ void descriptor_diff_unit(const float* __restrict__ A, const float* __restrict__ Bq, const Blend& ba, const Blend& bb,
                                                     int D_rt, float (&d)[D_T > 0 ? D_T : LOSS_MAXD], float (&ya)[D_T > 0 ? D_T : LOSS_MAXD],
                                                     float (&yb)[D_T > 0 ? D_T : LOSS_MAXD], float& na, float& nb) {
  constexpr int DM = D_T > 0 ? D_T : LOSS_MAXD;
  const int D = D_T > 0 ? D_T : D_rt;
  descriptor_blend<D_T>(A, ba, D, ya);
  descriptor_blend<D_T>(Bq, bb, D, yb);
  na = unit_normalize<DM>(ya, D);
  nb = unit_normalize<DM>(yb, D);
#pragma unroll
  for (int c = 0; c < DM; ++c) d[c] = ya[c] - yb[c];
}

template <int D_T, bool UNIT>
__global__ void __launch_bounds__(LR_THREADS)
loss_lowres_fwd_kernel(const float* __restrict__ la, const float* __restrict__ lb, int h, int w, int H, int W, int D_rt, float sh, float sw,
                       const __grid_constant__ DevTerms T, double* __restrict__ sums, unsigned long long* __restrict__ counts) {
  pdl_prologue();
  constexpr int DM = D_T > 0 ? D_T : LOSS_MAXD;
  const int D = D_T > 0 ? D_T : D_rt;
  const int b = blockIdx.y;
  const int t = find_term(T, blockIdx.x);
  const DevTerm& tm = T.t[t];
  const int64_t P = (int64_t)H * W;
  const int64_t cells = (int64_t)h * w;
  const float* A = la + (size_t)b * cells * D;
  const float* Bq = lb + (size_t)b * cells * D;
  const int64_t nvalid = tm.len ? min(tm.len[b], tm.n) : tm.n;
  const int64_t j = (int64_t)(blockIdx.x - tm.block_begin) * LR_THREADS + threadIdx.x;
  float acc = 0.f;
  int cnt = 0;
  if (j < nvalid) {
    const int64_t na = __ldg(tm.ia + b * tm.n + j), nb = __ldg(tm.ib + b * tm.n + j);
    if (na >= 0 && nb >= 0 && na < P && nb < P) {
      const Blend ba = blend_of(na, W, h, w, sh, sw), bb = blend_of(nb, W, h, w, sh, sw);
      float d[DM];
      if constexpr (UNIT) {
        float ya[DM], yb[DM], na, nb;
        descriptor_diff_unit<D_T>(A, Bq, ba, bb, D, d, ya, yb, na, nb);
      } else {
        descriptor_diff<D_T>(A, Bq, ba, bb, D, d);
      }
      float s2 = 0.f;
#pragma unroll
      for (int c = 0; c < DM; ++c) s2 = fmaf(d[c], d[c], s2);
      if (tm.kind == DDN_TERM_MATCH) {
        acc = s2;
      } else {
        const float dist = sqrtf(s2);
        const float hg = (tm.kind == DDN_TERM_HINGE) ? fmaxf(tm.margin - dist, 0.f) : fmaxf(dist - tm.margin, 0.f);
        float l = hg * hg;
        cnt = (l != 0.f);
        if (tm.flags & DDN_TERM_PIXEL_WEIGHT) l *= pixel_weight(tm, b, j, nb, W);
        acc = l;
      }
    }
  }
  double wsum = warp_sum((double)acc);
  int wcnt = warp_sum(cnt);
  __shared__ double s_sum[LR_THREADS / 32];
  __shared__ int s_cnt[LR_THREADS / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) { s_sum[wid] = wsum; s_cnt[wid] = wcnt; }
  __syncthreads();
  if (wid == 0) {
    double v = lane < LR_THREADS / 32 ? s_sum[lane] : 0.0;
    int c = lane < LR_THREADS / 32 ? s_cnt[lane] : 0;
    v = warp_sum(v);
    c = warp_sum(c);
    if (lane == 0) {
      if (v != 0.0) atomicAdd(&sums[b * T.n_terms + t], v);
      if (c) atomicAdd(&counts[b * T.n_terms + t], (unsigned long long)c);
    }
  }
}

// scatter g[0..D) * blend weights into the 4 cells of pixel `bl` of the fp64 accumulator
template <int D_T>
__device__ __forceinline__ void scatter_desc(double* __restrict__ dL, const Blend& bl, int D_rt, const float (&g)[D_T > 0 ? D_T : LOSS_MAXD]) {
  constexpr int DM = D_T > 0 ? D_T : LOSS_MAXD;
  const int D = D_T > 0 ? D_T : D_rt;
  const float wts[4] = {(1.f - bl.lh) * (1.f - bl.lw), (1.f - bl.lh) * bl.lw, bl.lh * (1.f - bl.lw), bl.lh * bl.lw};
  const int cell[4] = {bl.c00, bl.c01, bl.c10, bl.c11};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float wk = wts[k];
    if (k > 0 && wk == 0.f) continue;           // clamped edge cells coincide with cell 0 and carry weight 0
    double* dst = dL + (size_t)cell[k] * D;
#pragma unroll
    for (int c = 0; c < DM; ++c)
      if (c < D) red_add_f64(dst + c, (double)(wk * g[c]));
  }
}

template <int D_T, bool UNIT>
__global__ void __launch_bounds__(LR_THREADS)
loss_lowres_bwd_kernel(const float* __restrict__ la, const float* __restrict__ lb, int h, int w, int H, int W, int D_rt, float sh, float sw,
                       const __grid_constant__ DevTerms T, const float* __restrict__ coef, const float* __restrict__ upstream,
                       double* __restrict__ dla, double* __restrict__ dlb) {
  pdl_prologue();
  constexpr int DM = D_T > 0 ? D_T : LOSS_MAXD;
  const int D = D_T > 0 ? D_T : D_rt;
  const int b = blockIdx.y;
  const int t = find_term(T, blockIdx.x);
  const DevTerm& tm = T.t[t];
  float cf = coef[b * T.n_terms + t];
  if (upstream) cf *= upstream[0];
  const int64_t P = (int64_t)H * W;
  const int64_t cells = (int64_t)h * w;
  const float* A = la + (size_t)b * cells * D;
  const float* Bq = lb + (size_t)b * cells * D;
  double* dA = dla + (size_t)b * cells * D;
  double* dB = dlb + (size_t)b * cells * D;
  const int64_t nvalid = tm.len ? min(tm.len[b], tm.n) : tm.n;
  const int64_t j = (int64_t)(blockIdx.x - tm.block_begin) * LR_THREADS + threadIdx.x;
  const int lane = threadIdx.x & 31;
  const bool hinge = tm.kind != DDN_TERM_MATCH;
  int64_t na = -1, nb = -1;
  if (j < nvalid) { na = __ldg(tm.ia + b * tm.n + j); nb = __ldg(tm.ib + b * tm.n + j); }
  const bool ok = na >= 0 && nb >= 0 && na < P && nb < P;
  Blend ba = {}, bb = {};
  float g[DM];
#pragma unroll
  for (int c = 0; c < DM; ++c) g[c] = 0.f;
  float scale = 0.f;
  float ya[UNIT ? DM : 1], yb[UNIT ? DM : 1], nrm_a = 0.f, nrm_b = 0.f;    // UNIT: both sides' unit descriptors and norms
  if (ok) {
    ba = blend_of(na, W, h, w, sh, sw); bb = blend_of(nb, W, h, w, sh, sw);
    if constexpr (UNIT) descriptor_diff_unit<D_T>(A, Bq, ba, bb, D, g, ya, yb, nrm_a, nrm_b);
    else descriptor_diff<D_T>(A, Bq, ba, bb, D, g);
    float s2 = 0.f;
#pragma unroll
    for (int c = 0; c < DM; ++c) s2 = fmaf(g[c], g[c], s2);
    if (!hinge) {
      scale = 2.f * cf;                                  // d/dA ||A-B||^2
    } else {
      const float dist = sqrtf(s2);
      const float hg = (tm.kind == DDN_TERM_HINGE) ? fmaxf(tm.margin - dist, 0.f) : fmaxf(dist - tm.margin, 0.f);
      if (hg * hg != 0.f && dist > 0.f) {                // norm's subgradient at 0 is 0 (torch)
        const float wgt = (tm.flags & DDN_TERM_PIXEL_WEIGHT) ? pixel_weight(tm, b, j, nb, W) : 1.f;
        const float sgn = (tm.kind == DDN_TERM_HINGE) ? -1.f : 1.f;
        scale = cf * wgt * sgn * 2.f * hg / dist;
      }
    }
  }
#pragma unroll
  for (int c = 0; c < DM; ++c) g[c] *= scale;
  if (ok && scale != 0.f) {                              // B side: random indices
    float gb[DM];
#pragma unroll
    for (int c = 0; c < DM; ++c) gb[c] = -g[c];
    if constexpr (UNIT) unit_vjp<DM>(gb, yb, nrm_b, D);
    scatter_desc<D_T>(dB, bb, D, gb);
  }
  if (!hinge) {
    if (ok && scale != 0.f) {
      if constexpr (UNIT) unit_vjp<DM>(g, ya, nrm_a, D);
      scatter_desc<D_T>(dA, ba, D, g);
    }
    return;
  }
  // runs of equal A indices (every match repeated k times consecutively, spartan_dataset_masked.py:853-854): one scatter per run
  const int64_t key = ok ? na : (int64_t)(-1 - lane);
  const int64_t prev = __shfl_up_sync(0xffffffffu, key, 1);
  const bool head = (lane == 0) || (prev != key);
  const unsigned heads = __ballot_sync(0xffffffffu, head);
  const unsigned above = heads & ~((2u << lane) - 1u);
  const int run_end = above ? (__ffs(above) - 2) : 31;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const bool take = (lane + off) <= run_end;
#pragma unroll
    for (int c = 0; c < DM; ++c) {
      if (c < D) {
        const float o = __shfl_down_sync(0xffffffffu, g[c], off);
        if (take) g[c] += o;
      }
    }
  }
  if (head && ok) {
    if constexpr (UNIT) unit_vjp<DM>(g, ya, nrm_a, D);     // linear: the run's summed gradient takes the head's Jacobian once
    bool any = false;
#pragma unroll
    for (int c = 0; c < DM; ++c) any = any || (g[c] != 0.f);
    if (any) scatter_desc<D_T>(dA, ba, D, g);
  }
}

// ---- D = 8 / 16 / 32: LPP = D / 4 lanes per index pair, one channel QUAD per lane.  A warp instruction then touches one 16 * LPP-byte
// piece of a cell per pair instead of one line per LANE (the one-pair-per-lane kernels above spend their time in L1 tag lookups:
// 32 scattered 16-byte loads per instruction), every lane keeps 8 loads in flight instead of 2 * D, and the backward's segmented
// run reduction moves 4 floats per lane per step instead of D.
template <int LPP>
__device__ __forceinline__ float4 quad_diff(const float* __restrict__ A, const float* __restrict__ Bq, const Blend& ba, const Blend& bb, int sub) {
  constexpr int D = 4 * LPP;
  const float4 a00 = __ldg(reinterpret_cast<const float4*>(A + (size_t)ba.c00 * D) + sub), a01 = __ldg(reinterpret_cast<const float4*>(A + (size_t)ba.c01 * D) + sub);
  const float4 a10 = __ldg(reinterpret_cast<const float4*>(A + (size_t)ba.c10 * D) + sub), a11 = __ldg(reinterpret_cast<const float4*>(A + (size_t)ba.c11 * D) + sub);
  const float4 b00 = __ldg(reinterpret_cast<const float4*>(Bq + (size_t)bb.c00 * D) + sub), b01 = __ldg(reinterpret_cast<const float4*>(Bq + (size_t)bb.c01 * D) + sub);
  const float4 b10 = __ldg(reinterpret_cast<const float4*>(Bq + (size_t)bb.c10 * D) + sub), b11 = __ldg(reinterpret_cast<const float4*>(Bq + (size_t)bb.c11 * D) + sub);
  return make_float4(blend1(a00.x, a01.x, a10.x, a11.x, ba.lh, ba.lw) - blend1(b00.x, b01.x, b10.x, b11.x, bb.lh, bb.lw),
                     blend1(a00.y, a01.y, a10.y, a11.y, ba.lh, ba.lw) - blend1(b00.y, b01.y, b10.y, b11.y, bb.lh, bb.lw),
                     blend1(a00.z, a01.z, a10.z, a11.z, ba.lh, ba.lw) - blend1(b00.z, b01.z, b10.z, b11.z, bb.lh, bb.lw),
                     blend1(a00.w, a01.w, a10.w, a11.w, ba.lh, ba.lw) - blend1(b00.w, b01.w, b10.w, b11.w, bb.lh, bb.lw));
}

// one side's blended channel quad `sub` of pixel `bl` (the arithmetic of quad_diff)
template <int LPP>
__device__ __forceinline__ float4 quad_blend(const float* __restrict__ A, const Blend& bl, int sub) {
  constexpr int D = 4 * LPP;
  const float4 a00 = __ldg(reinterpret_cast<const float4*>(A + (size_t)bl.c00 * D) + sub), a01 = __ldg(reinterpret_cast<const float4*>(A + (size_t)bl.c01 * D) + sub);
  const float4 a10 = __ldg(reinterpret_cast<const float4*>(A + (size_t)bl.c10 * D) + sub), a11 = __ldg(reinterpret_cast<const float4*>(A + (size_t)bl.c11 * D) + sub);
  return make_float4(blend1(a00.x, a01.x, a10.x, a11.x, bl.lh, bl.lw), blend1(a00.y, a01.y, a10.y, a11.y, bl.lh, bl.lw),
                     blend1(a00.z, a01.z, a10.z, a11.z, bl.lh, bl.lw), blend1(a00.w, a01.w, a10.w, a11.w, bl.lh, bl.lw));
}
__device__ __forceinline__ float dot4(float4 a, float4 b) { return fmaf(a.x, b.x, fmaf(a.y, b.y, fmaf(a.z, b.z, a.w * b.w))); }
__device__ __forceinline__ float4 div4(float4 a, float n) { return make_float4(a.x / n, a.y / n, a.z / n, a.w / n); }
// the sum of v over the LPP lanes of one index pair (every lane of the warp must call it)
template <int LPP>
__device__ __forceinline__ float pair_sum(float v) {
#pragma unroll
  for (int off = 1; off < LPP; off <<= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}
// the quad layout of unit_vjp: g <- (g - y (y.g)) / n, y.g summed over the pair's lanes (every lane of the warp must call it)
template <int LPP>
__device__ __forceinline__ float4 quad_unit_vjp(float4 g, float4 y, float n) {
  const float t = pair_sum<LPP>(dot4(y, g));
  return make_float4((g.x - y.x * t) / n, (g.y - y.y * t) / n, (g.z - y.z * t) / n, (g.w - y.w * t) / n);
}

// LR_FWD_ITEMS index pairs per lane group in the forward: that many times fewer blocks = fewer contended atomics on the
// B * n_terms accumulators (they bound the one-pair version), and 8 * LR_FWD_ITEMS loads in flight per lane
constexpr int LR_FWD_ITEMS = 4;
template <int LPP, bool UNIT>
__global__ void __launch_bounds__(LR_THREADS)
loss_lowres_fwd_quad_kernel(const float* __restrict__ la, const float* __restrict__ lb, int h, int w, int H, int W, float sh, float sw,
                            const __grid_constant__ DevTerms T, double* __restrict__ sums, unsigned long long* __restrict__ counts) {
  pdl_prologue();
  constexpr int D = 4 * LPP, PPB = LR_THREADS / LPP;
  const int b = blockIdx.y;
  const int t = find_term(T, blockIdx.x);
  const DevTerm& tm = T.t[t];
  const int64_t P = (int64_t)H * W;
  const int64_t cells = (int64_t)h * w;
  const float* A = la + (size_t)b * cells * D;
  const float* Bq = lb + (size_t)b * cells * D;
  const int64_t nvalid = tm.len ? min(tm.len[b], tm.n) : tm.n;
  const int sub = threadIdx.x % LPP;
  const int64_t j0 = (int64_t)(blockIdx.x - tm.block_begin) * (PPB * LR_FWD_ITEMS) + threadIdx.x / LPP;
  int64_t na[LR_FWD_ITEMS], nb[LR_FWD_ITEMS];
#pragma unroll
  for (int k = 0; k < LR_FWD_ITEMS; ++k) {
    const int64_t j = j0 + k * PPB;
    na[k] = -1; nb[k] = -1;
    if (j < nvalid) { na[k] = __ldg(tm.ia + b * tm.n + j); nb[k] = __ldg(tm.ib + b * tm.n + j); }
  }
  float s2[LR_FWD_ITEMS];
  bool ok[LR_FWD_ITEMS];
  if constexpr (UNIT) {
    float4 xa[LR_FWD_ITEMS], xb[LR_FWD_ITEMS];
#pragma unroll
    for (int k = 0; k < LR_FWD_ITEMS; ++k) {
      ok[k] = na[k] >= 0 && nb[k] >= 0 && na[k] < P && nb[k] < P;
      xa[k] = xb[k] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (ok[k]) {
        xa[k] = quad_blend<LPP>(A, blend_of(na[k], W, h, w, sh, sw), sub);
        xb[k] = quad_blend<LPP>(Bq, blend_of(nb[k], W, h, w, sh, sw), sub);
      }
    }
#pragma unroll
    for (int k = 0; k < LR_FWD_ITEMS; ++k) {
      const float nrm_a = sqrtf(pair_sum<LPP>(dot4(xa[k], xa[k]))), nrm_b = sqrtf(pair_sum<LPP>(dot4(xb[k], xb[k])));
      s2[k] = 0.f;
      if (ok[k]) {
        const float4 ya = div4(xa[k], nrm_a), yb = div4(xb[k], nrm_b);
        const float4 d = make_float4(ya.x - yb.x, ya.y - yb.y, ya.z - yb.z, ya.w - yb.w);
        s2[k] = dot4(d, d);
      }
    }
  } else {
#pragma unroll
    for (int k = 0; k < LR_FWD_ITEMS; ++k) {
      ok[k] = na[k] >= 0 && nb[k] >= 0 && na[k] < P && nb[k] < P;
      s2[k] = 0.f;
      if (ok[k]) {
        const Blend ba = blend_of(na[k], W, h, w, sh, sw), bb = blend_of(nb[k], W, h, w, sh, sw);
        const float4 d = quad_diff<LPP>(A, Bq, ba, bb, sub);
        s2[k] = fmaf(d.x, d.x, fmaf(d.y, d.y, fmaf(d.z, d.z, d.w * d.w)));
      }
    }
  }
  float acc = 0.f;
  int cnt = 0;
#pragma unroll
  for (int k = 0; k < LR_FWD_ITEMS; ++k) {
    float v = s2[k];
#pragma unroll
    for (int off = 1; off < LPP; off <<= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    if (ok[k] && sub == 0) {
      if (tm.kind == DDN_TERM_MATCH) {
        acc += v;
      } else {
        const float dist = sqrtf(v);
        const float hg = (tm.kind == DDN_TERM_HINGE) ? fmaxf(tm.margin - dist, 0.f) : fmaxf(dist - tm.margin, 0.f);
        float l = hg * hg;
        cnt += (l != 0.f);
        if (tm.flags & DDN_TERM_PIXEL_WEIGHT) l *= pixel_weight(tm, b, j0 + k * PPB, nb[k], W);
        acc += l;
      }
    }
  }
  double wsum = warp_sum((double)acc);
  int wcnt = warp_sum(cnt);
  __shared__ double s_sum[LR_THREADS / 32];
  __shared__ int s_cnt[LR_THREADS / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) { s_sum[wid] = wsum; s_cnt[wid] = wcnt; }
  __syncthreads();
  if (wid == 0) {
    double v = lane < LR_THREADS / 32 ? s_sum[lane] : 0.0;
    int c = lane < LR_THREADS / 32 ? s_cnt[lane] : 0;
    v = warp_sum(v);
    c = warp_sum(c);
    if (lane == 0) {
      if (v != 0.0) atomicAdd(&sums[b * T.n_terms + t], v);
      if (c) atomicAdd(&counts[b * T.n_terms + t], (unsigned long long)c);
    }
  }
}

template <int LPP>
__device__ __forceinline__ void scatter_quad(double* __restrict__ dL, const Blend& bl, int sub, float4 g) {
  constexpr int D = 4 * LPP;
  const float wts[4] = {(1.f - bl.lh) * (1.f - bl.lw), (1.f - bl.lh) * bl.lw, bl.lh * (1.f - bl.lw), bl.lh * bl.lw};
  const int cell[4] = {bl.c00, bl.c01, bl.c10, bl.c11};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float wk = wts[k];
    if (k > 0 && wk == 0.f) continue;           // clamped edge cells coincide with cell 0 and carry weight 0
    double* dst = dL + (size_t)cell[k] * D + 4 * sub;
    red_add_f64(dst, (double)(wk * g.x)); red_add_f64(dst + 1, (double)(wk * g.y));
    red_add_f64(dst + 2, (double)(wk * g.z)); red_add_f64(dst + 3, (double)(wk * g.w));
  }
}

template <int LPP, bool UNIT>
__global__ void __launch_bounds__(LR_THREADS)
loss_lowres_bwd_quad_kernel(const float* __restrict__ la, const float* __restrict__ lb, int h, int w, int H, int W, float sh, float sw,
                            const __grid_constant__ DevTerms T, const float* __restrict__ coef, const float* __restrict__ upstream,
                            double* __restrict__ dla, double* __restrict__ dlb) {
  pdl_prologue();
  constexpr int D = 4 * LPP, PPB = LR_THREADS / LPP, PPW = 32 / LPP;      // pairs per block / per warp
  const int b = blockIdx.y;
  const int t = find_term(T, blockIdx.x);
  const DevTerm& tm = T.t[t];
  float cf = coef[b * T.n_terms + t];
  if (upstream) cf *= upstream[0];
  const int64_t P = (int64_t)H * W;
  const int64_t cells = (int64_t)h * w;
  const float* A = la + (size_t)b * cells * D;
  const float* Bq = lb + (size_t)b * cells * D;
  double* dA = dla + (size_t)b * cells * D;
  double* dB = dlb + (size_t)b * cells * D;
  const int64_t nvalid = tm.len ? min(tm.len[b], tm.n) : tm.n;
  const int lane = threadIdx.x & 31;
  const int sub = lane % LPP, pidx = lane / LPP;
  const int64_t j = (int64_t)(blockIdx.x - tm.block_begin) * PPB + threadIdx.x / LPP;
  const bool hinge = tm.kind != DDN_TERM_MATCH;
  int64_t na = -1, nb = -1;
  if (j < nvalid) { na = __ldg(tm.ia + b * tm.n + j); nb = __ldg(tm.ib + b * tm.n + j); }
  const bool ok = na >= 0 && nb >= 0 && na < P && nb < P;
  Blend ba = {}, bb = {};
  float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
  float s2 = 0.f;
  float4 ya = g, yb = g;                                 // UNIT: both sides' unit descriptors and norms
  float nrm_a = 1.f, nrm_b = 1.f;
  if constexpr (UNIT) {
    if (ok) {
      ba = blend_of(na, W, h, w, sh, sw); bb = blend_of(nb, W, h, w, sh, sw);
      ya = quad_blend<LPP>(A, ba, sub); yb = quad_blend<LPP>(Bq, bb, sub);
    }
    nrm_a = sqrtf(pair_sum<LPP>(dot4(ya, ya))); nrm_b = sqrtf(pair_sum<LPP>(dot4(yb, yb)));
    if (ok) {
      ya = div4(ya, nrm_a); yb = div4(yb, nrm_b);
      g = make_float4(ya.x - yb.x, ya.y - yb.y, ya.z - yb.z, ya.w - yb.w);
      s2 = dot4(g, g);
    }
  } else if (ok) {
    ba = blend_of(na, W, h, w, sh, sw); bb = blend_of(nb, W, h, w, sh, sw);
    g = quad_diff<LPP>(A, Bq, ba, bb, sub);
    s2 = fmaf(g.x, g.x, fmaf(g.y, g.y, fmaf(g.z, g.z, g.w * g.w)));
  }
#pragma unroll
  for (int off = 1; off < LPP; off <<= 1) s2 += __shfl_xor_sync(0xffffffffu, s2, off);
  float scale = 0.f;
  if (ok) {
    if (!hinge) {
      scale = 2.f * cf;                                  // d/dA ||A-B||^2
    } else {
      const float dist = sqrtf(s2);
      const float hg = (tm.kind == DDN_TERM_HINGE) ? fmaxf(tm.margin - dist, 0.f) : fmaxf(dist - tm.margin, 0.f);
      if (hg * hg != 0.f && dist > 0.f) {                // norm's subgradient at 0 is 0 (torch)
        const float wgt = (tm.flags & DDN_TERM_PIXEL_WEIGHT) ? pixel_weight(tm, b, j, nb, W) : 1.f;
        const float sgn = (tm.kind == DDN_TERM_HINGE) ? -1.f : 1.f;
        scale = cf * wgt * sgn * 2.f * hg / dist;
      }
    }
  }
  g.x *= scale; g.y *= scale; g.z *= scale; g.w *= scale;
  float4 gb = make_float4(-g.x, -g.y, -g.z, -g.w);
  if constexpr (UNIT) gb = quad_unit_vjp<LPP>(gb, yb, nrm_b);
  if (ok && scale != 0.f) scatter_quad<LPP>(dB, bb, sub, gb);       // B side: random indices
  if (!hinge) {
    if constexpr (UNIT) g = quad_unit_vjp<LPP>(g, ya, nrm_a);
    if (ok && scale != 0.f) scatter_quad<LPP>(dA, ba, sub, g);
    return;
  }
  // runs of equal A indices (every match repeated k times consecutively, spartan_dataset_masked.py:853-854): one scatter per run
  const int64_t key = ok ? na : (int64_t)(-1 - pidx);
  const int64_t prev = __shfl_up_sync(0xffffffffu, key, LPP);
  const bool head = (pidx == 0) || (prev != key);
  const unsigned heads = __ballot_sync(0xffffffffu, head);
  const unsigned below_next = (pidx + 1 == PPW) ? 0xffffffffu : ((1u << ((pidx + 1) * LPP)) - 1u);    // lanes of pairs <= mine
  const unsigned above = heads & ~below_next;
  const int run_end = above ? ((__ffs(above) - 1) / LPP - 1) : (PPW - 1);                               // last pair of my run
#pragma unroll
  for (int off = 1; off < PPW; off <<= 1) {
    const bool take = (pidx + off) <= run_end;
    const float ox = __shfl_down_sync(0xffffffffu, g.x, off * LPP), oy = __shfl_down_sync(0xffffffffu, g.y, off * LPP);
    const float oz = __shfl_down_sync(0xffffffffu, g.z, off * LPP), ow = __shfl_down_sync(0xffffffffu, g.w, off * LPP);
    if (take) { g.x += ox; g.y += oy; g.z += oz; g.w += ow; }
  }
  if constexpr (UNIT) g = quad_unit_vjp<LPP>(g, ya, nrm_a);   // linear: the run's summed gradient takes the head's Jacobian once
  if (head && ok && (g.x != 0.f || g.y != 0.f || g.z != 0.f || g.w != 0.f)) scatter_quad<LPP>(dA, ba, sub, g);
}

static int build_terms_lr(const ddn_loss_term* th, int n_terms, DevTerms* T, int pairs_per_block = LR_THREADS) {
  DDN_TRY(build_terms(th, n_terms, T));
  int blk = 0;                                   // one index pair per thread (or per D / 4 threads: the quad kernels)
  for (int i = 0; i < n_terms; ++i) { T->t[i].block_begin = blk; blk += (int)ceil_div(th[i].n, pairs_per_block); }
  T->total_blocks = blk;
  return 0;
}
static float ac_scale(int in, int out) { return out > 1 ? (float)(in - 1) / (float)(out - 1) : 0.f; }

// dl[i] += (float)acc[i]: the fp64 scatter accumulator into the caller's fp32 gradient
__global__ void add_f64_to_f32_kernel(const double* __restrict__ acc, float* __restrict__ dl, int64_t n) {
  pdl_prologue();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) dl[i] += (float)acc[i];
}

}  // namespace ddn

using namespace ddn;

static int check_lowres_flags(int flags) {
  DDN_CHECK_ARG((flags & ~DDN_LOWRES_UNIT) == 0, "unknown low-resolution loss flags 0x%x", flags);
  return 0;
}

extern "C" int ddn_contrastive_terms_forward_lowres(const float* low_a, const float* low_b, int B, int h, int w, int H, int W, int D,
                                                    const ddn_loss_term* terms_host, int n_terms,
                                                    double* sums, int64_t* counts, void* stream) {
  return ddn_contrastive_terms_forward_lowres_v2(low_a, low_b, B, h, w, H, W, D, terms_host, n_terms, sums, counts, 0, stream);
}

extern "C" int ddn_contrastive_terms_forward_lowres_v2(const float* low_a, const float* low_b, int B, int h, int w, int H, int W, int D,
                                                       const ddn_loss_term* terms_host, int n_terms,
                                                       double* sums, int64_t* counts, int flags, void* stream) {
  DDN_TRY(check_lowres_flags(flags));
  DDN_TRY(check_common(low_a, low_b, B, (int64_t)H * W, D, W));
  DDN_CHECK_ARG(sums && counts && h >= 1 && w >= 1 && H >= h && W >= w && (int64_t)H * W < (1LL << 31), "bad low-resolution geometry / null outputs");
  const int lpp = (D == 8 || D == 16 || D == 32) ? D / 4 : 1;
  DevTerms T;
  DDN_TRY(build_terms_lr(terms_host, n_terms, &T, lpp > 1 ? LR_THREADS / lpp * LR_FWD_ITEMS : LR_THREADS));
  cudaStream_t st = (cudaStream_t)stream;
  DDN_CUDA(cudaMemsetAsync(sums, 0, sizeof(double) * B * n_terms, st));
  DDN_CUDA(cudaMemsetAsync(counts, 0, sizeof(int64_t) * B * n_terms, st));
  if (T.total_blocks == 0) return 0;
  dim3 grid(T.total_blocks, B);
  auto cnt = reinterpret_cast<unsigned long long*>(counts);
  double pairs = 0;
  for (int i = 0; i < n_terms; ++i) pairs += (double)terms_host[i].n * B;
  ProfScope ps(PROF_LOSS_FWD, pairs * (16.0 + 8.0 * D), st);
  const float sh = ac_scale(h, H), sw = ac_scale(w, W);
  const bool unit = flags & DDN_LOWRES_UNIT;
#define FWD(DT)                                                                                                                  \
  if (unit) DDN_LAUNCH((loss_lowres_fwd_kernel<DT, true>), grid, LR_THREADS, 0, st, low_a, low_b, h, w, H, W, D, sh, sw, T, sums, cnt); \
  else DDN_LAUNCH((loss_lowres_fwd_kernel<DT, false>), grid, LR_THREADS, 0, st, low_a, low_b, h, w, H, W, D, sh, sw, T, sums, cnt)
#define FWDQ(L)                                                                                                                    \
  if (unit) DDN_LAUNCH((loss_lowres_fwd_quad_kernel<L, true>), grid, LR_THREADS, 0, st, low_a, low_b, h, w, H, W, sh, sw, T, sums, cnt); \
  else DDN_LAUNCH((loss_lowres_fwd_quad_kernel<L, false>), grid, LR_THREADS, 0, st, low_a, low_b, h, w, H, W, sh, sw, T, sums, cnt)
  switch (D) {
    case 3: FWD(3); break;
    case 4: FWD(4); break;
    case 8: FWDQ(2); break;
    case 16: FWDQ(4); break;
    case 32: FWDQ(8); break;
    default: FWD(0); break;
  }
#undef FWD
#undef FWDQ
  return 0;
}

extern "C" int ddn_contrastive_terms_backward_lowres(const float* low_a, const float* low_b, int B, int h, int w, int H, int W, int D,
                                                     const ddn_loss_term* terms_host, int n_terms,
                                                     const float* coef, const float* upstream,
                                                     float* dlow_a, float* dlow_b, double* scratch, void* stream) {
  return ddn_contrastive_terms_backward_lowres_v2(low_a, low_b, B, h, w, H, W, D, terms_host, n_terms, coef, upstream, dlow_a, dlow_b,
                                                  scratch, 0, stream);
}

extern "C" int ddn_contrastive_terms_backward_lowres_v2(const float* low_a, const float* low_b, int B, int h, int w, int H, int W, int D,
                                                        const ddn_loss_term* terms_host, int n_terms,
                                                        const float* coef, const float* upstream,
                                                        float* dlow_a, float* dlow_b, double* scratch, int flags, void* stream) {
  DDN_TRY(check_lowres_flags(flags));
  DDN_TRY(check_common(low_a, low_b, B, (int64_t)H * W, D, W));
  DDN_CHECK_ARG(coef && dlow_a && dlow_b && scratch && h >= 1 && w >= 1 && H >= h && W >= w && (int64_t)H * W < (1LL << 31), "bad low-resolution geometry / null buffers");
  DDN_CHECK_ARG(((reinterpret_cast<uintptr_t>(dlow_a) | reinterpret_cast<uintptr_t>(dlow_b) | reinterpret_cast<uintptr_t>(scratch) | reinterpret_cast<uintptr_t>(low_a) | reinterpret_cast<uintptr_t>(low_b)) & 15) == 0,
                "low-resolution maps and their gradients must be 16-byte aligned");
  const int lpp = (D == 8 || D == 16 || D == 32) ? D / 4 : 1;
  DevTerms T;
  DDN_TRY(build_terms_lr(terms_host, n_terms, &T, LR_THREADS / lpp));
  if (T.total_blocks == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  dim3 grid(T.total_blocks, B);
  double pairs = 0;
  for (int i = 0; i < n_terms; ++i) pairs += (double)terms_host[i].n * B;
  const int64_t n_low = (int64_t)B * h * w * D;
  double* dacc_a = scratch;                     // [2][B, h*w, D] fp64: the scatter target, added to dlow_a / dlow_b at the end
  double* dacc_b = scratch + n_low;
  DDN_CUDA(cudaMemsetAsync(scratch, 0, sizeof(double) * 2 * (size_t)n_low, st));
  const float sh = ac_scale(h, H), sw = ac_scale(w, W);
  {
  ProfScope ps(PROF_LOSS_BWD, pairs * (16.0 + 24.0 * D), st);
  const bool unit = flags & DDN_LOWRES_UNIT;
#define BWD(DT)                                                                                                                   \
  if (unit) DDN_LAUNCH((loss_lowres_bwd_kernel<DT, true>), grid, LR_THREADS, 0, st, low_a, low_b, h, w, H, W, D, sh, sw, T, coef, upstream, dacc_a, dacc_b); \
  else DDN_LAUNCH((loss_lowres_bwd_kernel<DT, false>), grid, LR_THREADS, 0, st, low_a, low_b, h, w, H, W, D, sh, sw, T, coef, upstream, dacc_a, dacc_b)
#define BWDQ(L)                                                                                                                   \
  if (unit) DDN_LAUNCH((loss_lowres_bwd_quad_kernel<L, true>), grid, LR_THREADS, 0, st, low_a, low_b, h, w, H, W, sh, sw, T, coef, upstream, dacc_a, dacc_b); \
  else DDN_LAUNCH((loss_lowres_bwd_quad_kernel<L, false>), grid, LR_THREADS, 0, st, low_a, low_b, h, w, H, W, sh, sw, T, coef, upstream, dacc_a, dacc_b)
  switch (D) {
    case 3: BWD(3); break;
    case 4: BWD(4); break;
    case 8: BWDQ(2); break;
    case 16: BWDQ(4); break;
    case 32: BWDQ(8); break;
    default: BWD(0); break;
  }
#undef BWD
#undef BWDQ
  }
  const int blocks = (int)std::min<int64_t>(ceil_div(n_low, 256), (int64_t)num_sms() * 8);
  DDN_LAUNCH(add_f64_to_f32_kernel, blocks, 256, 0, st, dacc_a, dlow_a, n_low);
  DDN_LAUNCH(add_f64_to_f32_kernel, blocks, 256, 0, st, dacc_b, dlow_b, n_low);
  return 0;
}
