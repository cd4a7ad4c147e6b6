// BatchNorm2d (+residual, +ReLU) forward/backward on NHWC tensors viewed as [M][C], and the stem's fused
// BN + ReLU + MaxPool(3,2,1).  All HBM-bound elementwise / column-reduction kernels.
//
// Reference semantics: nn.BatchNorm2d / nn.ReLU(inplace) / nn.MaxPool2d(3,2,1) as wired by
// PSD/vision/torchvision/models/resnet.py:53-69 (BasicBlock.forward) and :231-236 (stem):
// training = batch mean and BIASED variance over (N,H,W), eps inside the sqrt, running statistics updated
// with momentum and the UNBIASED variance; eval = running statistics.
//
// Byte diet (tensor-core modes): activations exist ONLY as bf16 hi/lo operand planes (x ~= hi + lo, 16
// mantissa bits -- what every conv reads anyway); the residual add reads the planes, the ReLU mask of a BatchNorm without
// residual is recomputed from its own input, and column statistics are finalized by the last CTA of the kernel that
// produced them (bn_stats.cuh) instead of by a second launch.  G > 1: per-group batch statistics (pair-batched step).
#include "conv.cuh"

namespace ddn {

constexpr int BN_THREADS = 256;

// x -> (hi, lo) bf16 with x ~= hi + lo; 4 values -> two 8-byte stores
__device__ __forceinline__ void store_split4(__nv_bfloat16* hi, __nv_bfloat16* lo, int64_t i4, float4 v) {
  __nv_bfloat16 h0 = __float2bfloat16_rn(v.x), h1 = __float2bfloat16_rn(v.y), h2 = __float2bfloat16_rn(v.z), h3 = __float2bfloat16_rn(v.w);
  __nv_bfloat162 a = __halves2bfloat162(h0, h1), b = __halves2bfloat162(h2, h3);
  uint2 ho; ho.x = *reinterpret_cast<uint32_t*>(&a); ho.y = *reinterpret_cast<uint32_t*>(&b);
  reinterpret_cast<uint2*>(hi)[i4] = ho;
  if (lo) {
    __nv_bfloat162 c = __halves2bfloat162(__float2bfloat16_rn(v.x - __bfloat162float(h0)), __float2bfloat16_rn(v.y - __bfloat162float(h1)));
    __nv_bfloat162 d = __halves2bfloat162(__float2bfloat16_rn(v.z - __bfloat162float(h2)), __float2bfloat16_rn(v.w - __bfloat162float(h3)));
    uint2 l2; l2.x = *reinterpret_cast<uint32_t*>(&c); l2.y = *reinterpret_cast<uint32_t*>(&d);
    reinterpret_cast<uint2*>(lo)[i4] = l2;
  }
}
__device__ __forceinline__ float4 bf16x4_to_float4(uint2 h) {
  return make_float4(__uint_as_float(h.x << 16), __uint_as_float(h.x & 0xffff0000u), __uint_as_float(h.y << 16),
                     __uint_as_float(h.y & 0xffff0000u));
}
// 4 packed bf16 values > 0 ?  (sign bit clear and not +/-0)
__device__ __forceinline__ void mask_from_bf16x4(uint2 h, float4& g) {
  if ((h.x & 0x8000u) || !(h.x & 0x7fffu)) g.x = 0.f;
  if ((h.x & 0x80000000u) || !(h.x & 0x7fff0000u)) g.y = 0.f;
  if ((h.y & 0x8000u) || !(h.y & 0x7fffu)) g.z = 0.f;
  if ((h.y & 0x80000000u) || !(h.y & 0x7fff0000u)) g.w = 0.f;
}

size_t bn_accum_bytes(int C) { return align_up(sizeof(double) * BN_MAX_GROUPS * 2 * (size_t)C, 256) + 256; }
BnAccum bn_accum_at(void* base, int C) {
  BnAccum a;
  a.acc = reinterpret_cast<double*>(base);
  a.ticket = reinterpret_cast<unsigned int*>(reinterpret_cast<char*>(base) + align_up(sizeof(double) * BN_MAX_GROUPS * 2 * (size_t)C, 256));
  return a;
}

// A column-sum block covers at most BN_COLSUM_MAX_C channels (one float4 column per thread); wider tensors are cut into slices
// of that width along gridDim.z.
constexpr int BN_COLSUM_MAX_C = 4 * BN_THREADS;
static inline int bn_slice_c(int C) { return C > BN_COLSUM_MAX_C ? BN_COLSUM_MAX_C : C; }
static inline int bn_rows_per_iter(int C) { return BN_THREADS / (bn_slice_c(C) / 4); }
// blocks per group: exactly one resident wave over all groups (`resident` = SMs x CTAs per SM of the kernel, from the occupancy
// API: a larger grid would run a partial second wave at low occupancy), at least 4 row iterations per block
static int64_t bn_colsum_rows_per_block(int64_t Mg, int C, int G, int resident) {
  const int rpi = bn_rows_per_iter(C);
  const int64_t target = std::max<int64_t>(1, (int64_t)resident / G);
  const int64_t iters = std::max<int64_t>(4, ceil_div(Mg, (int64_t)rpi * target));
  return (int64_t)rpi * iters;
}
static int bn_colsum_blocks(int64_t Mg, int C, int G, int resident) {
  return (int)ceil_div(Mg, bn_colsum_rows_per_block(Mg, C, G, resident));
}

struct BnColsumArgs {
  const float* x; const float* dy; const float* y; const __nv_bfloat16* y_hi;
  const float* mean; const float* invstd; const float* gamma; const float* beta;   // [G][C] statistics (MODE 1)
  int64_t Mg; int C; int64_t rows_per_block; int relu;
  int Cs;               // channels of one slice (blockIdx.z): C, or BN_COLSUM_MAX_C when C is wider
};

// column sums of v0, v1 over this block's rows of group blockIdx.y, added into the fp64 accumulator; the last CTA finalizes
// MODE 0: (x, x^2) -> BatchNorm statistics      MODE 1: (g, g*xhat) with g = dy * (y > 0 if relu) -> dgamma / dbeta / sums
template <int MODE>
__global__ void __launch_bounds__(BN_THREADS)
bn_colsum_kernel(BnColsumArgs a, BnFwdFinal ff, BnBwdFinal fb) {
  pdl_prologue();
  const int C = a.C, q = a.Cs >> 2;
  const int rr = threadIdx.x / q, rpi = BN_THREADS / q;
  const int cq = threadIdx.x % q + (int)blockIdx.z * q;     // float4 column within the full row
  const int g = blockIdx.y;
  const int64_t r0 = (int64_t)g * a.Mg + (int64_t)blockIdx.x * a.rows_per_block;
  const int64_t r1 = min((int64_t)(g + 1) * a.Mg, r0 + a.rows_per_block);
  float4 s0 = make_float4(0, 0, 0, 0), s1 = make_float4(0, 0, 0, 0);
  float4 mu = make_float4(0, 0, 0, 0), is = make_float4(1, 1, 1, 1), sc = is, be = mu;
  const bool recompute_mask = MODE == 1 && a.relu && !a.y && !a.y_hi;
  if (MODE == 1) {
    mu = reinterpret_cast<const float4*>(a.mean + (size_t)g * C)[cq];
    is = reinterpret_cast<const float4*>(a.invstd + (size_t)g * C)[cq];
    if (recompute_mask) {
      const float4 ga = reinterpret_cast<const float4*>(a.gamma)[cq];
      be = reinterpret_cast<const float4*>(a.beta)[cq];
      sc = make_float4(ga.x * is.x, ga.y * is.y, ga.z * is.z, ga.w * is.w);
    }
  }
  // two rows per iteration: twice the loads in flight per thread (the kernel is pure streaming; its speed is the number of
  // outstanding 16-byte loads per SM)
  auto accumulate = [&](const float4 v, float4 gr, const uint2 yh, const float4 yo) {
    if (MODE == 0) {
      s0.x += v.x; s0.y += v.y; s0.z += v.z; s0.w += v.w;
      s1.x = fmaf(v.x, v.x, s1.x); s1.y = fmaf(v.y, v.y, s1.y); s1.z = fmaf(v.z, v.z, s1.z); s1.w = fmaf(v.w, v.w, s1.w);
    } else {
      if (a.relu) {
        if (a.y_hi) {     // the bf16 "hi" plane of y has y's sign and zero-ness
          mask_from_bf16x4(yh, gr);
        } else if (a.y) {
          gr.x = yo.x > 0.f ? gr.x : 0.f; gr.y = yo.y > 0.f ? gr.y : 0.f; gr.z = yo.z > 0.f ? gr.z : 0.f; gr.w = yo.w > 0.f ? gr.w : 0.f;
        } else {          // no residual in the forward: y > 0  <=>  bn(x) > 0, same fmaf as bn_apply_kernel
          if (!(fmaf(v.x - mu.x, sc.x, be.x) > 0.f)) gr.x = 0.f;
          if (!(fmaf(v.y - mu.y, sc.y, be.y) > 0.f)) gr.y = 0.f;
          if (!(fmaf(v.z - mu.z, sc.z, be.z) > 0.f)) gr.z = 0.f;
          if (!(fmaf(v.w - mu.w, sc.w, be.w) > 0.f)) gr.w = 0.f;
        }
      }
      s0.x += gr.x; s0.y += gr.y; s0.z += gr.z; s0.w += gr.w;
      s1.x = fmaf(gr.x, (v.x - mu.x) * is.x, s1.x); s1.y = fmaf(gr.y, (v.y - mu.y) * is.y, s1.y);
      s1.z = fmaf(gr.z, (v.z - mu.z) * is.z, s1.z); s1.w = fmaf(gr.w, (v.w - mu.w) * is.w, s1.w);
    }
  };
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  const uint2 z2 = make_uint2(0u, 0u);
  int64_t r = r0 + rr;
  for (; r + rpi < r1; r += 2 * rpi) {
    const int64_t ra = r, rb = r + rpi;
    const float4 va = __ldg(reinterpret_cast<const float4*>(a.x + ra * C) + cq), vb = __ldg(reinterpret_cast<const float4*>(a.x + rb * C) + cq);
    float4 ga = z4, gb = z4, ya = z4, yb = z4; uint2 ha = z2, hb = z2;
    if (MODE == 1) {
      ga = __ldg(reinterpret_cast<const float4*>(a.dy + ra * C) + cq); gb = __ldg(reinterpret_cast<const float4*>(a.dy + rb * C) + cq);
      if (a.relu && a.y_hi) { ha = __ldg(reinterpret_cast<const uint2*>(a.y_hi + ra * C) + cq); hb = __ldg(reinterpret_cast<const uint2*>(a.y_hi + rb * C) + cq); }
      else if (a.relu && a.y) { ya = __ldg(reinterpret_cast<const float4*>(a.y + ra * C) + cq); yb = __ldg(reinterpret_cast<const float4*>(a.y + rb * C) + cq); }
    }
    accumulate(va, ga, ha, ya);
    accumulate(vb, gb, hb, yb);
  }
  for (; r < r1; r += rpi) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(a.x + r * C) + cq);
    float4 gr = z4, yo = z4; uint2 yh = z2;
    if (MODE == 1) {
      gr = __ldg(reinterpret_cast<const float4*>(a.dy + r * C) + cq);
      if (a.relu && a.y_hi) yh = __ldg(reinterpret_cast<const uint2*>(a.y_hi + r * C) + cq);
      else if (a.relu && a.y) yo = __ldg(reinterpret_cast<const float4*>(a.y + r * C) + cq);
    }
    accumulate(v, gr, yh, yo);
  }
  __shared__ float4 sh0[BN_THREADS], sh1[BN_THREADS];
  __shared__ int s_last;
  sh0[threadIdx.x] = s0; sh1[threadIdx.x] = s1;
  __syncthreads();
  double* acc = MODE == 0 ? ff.a.acc : fb.a.acc;
  if (rr == 0) {
    for (int k = 1; k < rpi; ++k) {
      float4 u = sh0[k * q + threadIdx.x], w = sh1[k * q + threadIdx.x];
      s0.x += u.x; s0.y += u.y; s0.z += u.z; s0.w += u.w;
      s1.x += w.x; s1.y += w.y; s1.z += w.z; s1.w += w.w;
    }
    double* p0 = acc + (size_t)(g * 2) * C + (cq << 2);
    double* p1 = p0 + C;
    red_add_f64(p0, (double)s0.x); red_add_f64(p0 + 1, (double)s0.y); red_add_f64(p0 + 2, (double)s0.z); red_add_f64(p0 + 3, (double)s0.w);
    red_add_f64(p1, (double)s1.x); red_add_f64(p1 + 1, (double)s1.y); red_add_f64(p1 + 2, (double)s1.z); red_add_f64(p1 + 3, (double)s1.w);
  }
  unsigned int* ticket = MODE == 0 ? ff.a.ticket : fb.a.ticket;
  const bool last = bn_last_cta(ticket, gridDim.x * gridDim.y * gridDim.z, threadIdx.x == 0, &s_last, [] { __syncthreads(); });
  if (last) {
    for (int c = threadIdx.x; c < C; c += BN_THREADS) {
      if (MODE == 0) bn_fwd_finalize_channel(ff, c);
      else bn_bwd_finalize_channel(fb, c);
    }
  }
}

// eval-mode BN folded to one multiply-add per element: y = x * scale + shift
__global__ void bn_fold_kernel(const float* __restrict__ rm, const float* __restrict__ rv, const float* __restrict__ gamma,
                               const float* __restrict__ beta, int C, float eps, float* __restrict__ scale, float* __restrict__ shift) {
  pdl_prologue();
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float sc = gamma[c] * (1.0f / sqrtf(rv[c] + eps));
  scale[c] = sc;
  shift[c] = fmaf(-rm[c], sc, beta[c]);
}

__global__ void bn_eval_stats_kernel(const float* __restrict__ rm, const float* __restrict__ rv, int C, int G, float eps,
                                     float* __restrict__ mean, float* __restrict__ invstd) {
  pdl_prologue();
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float m = rm[c], is = 1.0f / sqrtf(rv[c] + eps);
  for (int g = 0; g < G; ++g) { mean[g * C + c] = m; invstd[g * C + c] = is; }
}

constexpr int BN_EVAL_MAX_SEGS = 40;
struct BnEvalSegs { BnEvalSeg s[BN_EVAL_MAX_SEGS]; int n; };
// every BatchNorm of the network in one launch: blockIdx.y = BatchNorm, stats = [G][C] mean then [G][C] invstd
__global__ void bn_eval_stats_all_kernel(const float* __restrict__ buffers, float* __restrict__ stats, BnEvalSegs segs, int G, float eps) {
  pdl_prologue();
  const BnEvalSeg sg = segs.s[blockIdx.y];
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < sg.C; c += gridDim.x * blockDim.x) {
    const float m = buffers[sg.rm_off + c], is = 1.0f / sqrtf(buffers[sg.rv_off + c] + eps);
    for (int g = 0; g < G; ++g) {
      stats[sg.stat_off + (size_t)g * sg.C + c] = m;
      stats[sg.stat_off + (size_t)(G + g) * sg.C + c] = is;
    }
  }
}

__global__ void __launch_bounds__(BN_THREADS)
bn_apply_kernel(BnApplyArgs a) {
  pdl_prologue();
  extern __shared__ float sm[];   // per group: scale[C], mean[C], beta[C] (+ the same three of the residual's BatchNorm)
  const int C = a.C, G = a.G;
  const bool res_bn = a.r && a.rmean;
  const int per_g = (res_bn ? 6 : 3) * C;
  for (int i = threadIdx.x; i < G * C; i += blockDim.x) {
    const int g = i / C, c = i - g * C;
    float* b = sm + g * per_g;
    b[c] = a.gamma[c] * a.invstd[i]; b[C + c] = a.mean[i]; b[2 * C + c] = a.beta[c];
    if (res_bn) { b[3 * C + c] = a.rgamma[c] * a.rinvstd[i]; b[4 * C + c] = a.rmean[i]; b[5 * C + c] = a.rbeta[c]; }
  }
  __syncthreads();
  const int q = C >> 2;
  const bool q_pow2 = (q & (q - 1)) == 0;
  const int64_t total = a.M * q;
  const int64_t per_group = (a.M / G) * q;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (q_pow2 ? (int)(i & (q - 1)) : (int)(i % q)) << 2;           // no 64-bit division on the hot path
    const float* b = sm + ((G > 1 && i >= per_group) ? 1 : 0) * per_g;              // G <= 2
    const float4 sc = *reinterpret_cast<const float4*>(b + c), mu = *reinterpret_cast<const float4*>(b + C + c),
                 be = *reinterpret_cast<const float4*>(b + 2 * C + c);
    float4 v = __ldg(reinterpret_cast<const float4*>(a.x) + i);
    v.x = fmaf(v.x - mu.x, sc.x, be.x); v.y = fmaf(v.y - mu.y, sc.y, be.y);
    v.z = fmaf(v.z - mu.z, sc.z, be.z); v.w = fmaf(v.w - mu.w, sc.w, be.w);
    if (a.r) {
      float4 r = __ldg(reinterpret_cast<const float4*>(a.r) + i);
      if (res_bn) {
        const float4 rsc = *reinterpret_cast<const float4*>(b + 3 * C + c), rmu = *reinterpret_cast<const float4*>(b + 4 * C + c),
                     rbe = *reinterpret_cast<const float4*>(b + 5 * C + c);
        r.x = fmaf(r.x - rmu.x, rsc.x, rbe.x); r.y = fmaf(r.y - rmu.y, rsc.y, rbe.y);
        r.z = fmaf(r.z - rmu.z, rsc.z, rbe.z); r.w = fmaf(r.w - rmu.w, rsc.w, rbe.w);
      }
      v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
    } else if (a.r_hi) {       // identity residual from the operand planes: r = hi + lo
      float4 r = bf16x4_to_float4(__ldg(reinterpret_cast<const uint2*>(a.r_hi) + i));
      if (a.r_lo) {
        const float4 l = bf16x4_to_float4(__ldg(reinterpret_cast<const uint2*>(a.r_lo) + i));
        r.x += l.x; r.y += l.y; r.z += l.z; r.w += l.w;
      }
      v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
    }
    if (a.relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
    if (a.y) reinterpret_cast<float4*>(a.y)[i] = v;
    if (a.hi) store_split4(a.hi, a.lo, i, v);
  }
}

// dx = gamma*invstd*(g - dbeta_g/Mg - xhat*dgamma_g/Mg)  (training)   |   gamma*invstd*g  (eval: frozen statistics)
__global__ void __launch_bounds__(BN_THREADS)
bn_bwd_apply_kernel(BnBwdArgs a) {
  pdl_prologue();
  extern __shared__ float sm[];   // per group: k1[C], mean[C], invstd[C], dbeta/M[C], dgamma/M[C], scale[C], beta[C]
  const int C = a.C, G = a.G;
  const int64_t Mg = a.M / G;
  const float invM = (float)(1.0 / (double)Mg);
  const bool recompute_mask = a.relu && !a.y && !a.y_hi;
  for (int i = threadIdx.x; i < G * C; i += blockDim.x) {
    const int g = i / C, c = i - g * C;
    float* b = sm + g * 7 * C;
    b[c] = a.gamma[c] * a.invstd[i]; b[C + c] = a.mean[i]; b[2 * C + c] = a.invstd[i];
    b[3 * C + c] = a.training ? a.sums[(g * 2) * C + c] * invM : 0.f;
    b[4 * C + c] = a.training ? a.sums[(g * 2 + 1) * C + c] * invM : 0.f;
    b[5 * C + c] = a.gamma[c] * a.invstd[i]; b[6 * C + c] = a.beta ? a.beta[c] : 0.f;
  }
  __syncthreads();
  const int q = C >> 2;
  const bool q_pow2 = (q & (q - 1)) == 0;
  const int64_t total = a.M * q;
  const int64_t per_group = Mg * q;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (q_pow2 ? (int)(i & (q - 1)) : (int)(i % q)) << 2;
    const float* b = sm + ((G > 1 && i >= per_group) ? 1 : 0) * 7 * C;
    const float4 k1 = *reinterpret_cast<const float4*>(b + c), mu = *reinterpret_cast<const float4*>(b + C + c),
                 is = *reinterpret_cast<const float4*>(b + 2 * C + c), mb = *reinterpret_cast<const float4*>(b + 3 * C + c),
                 mg = *reinterpret_cast<const float4*>(b + 4 * C + c);
    float4 g = __ldg(reinterpret_cast<const float4*>(a.dy) + i);
    float4 v = __ldg(reinterpret_cast<const float4*>(a.x) + i);
    if (a.relu) {
      if (a.y_hi) {
        mask_from_bf16x4(__ldg(reinterpret_cast<const uint2*>(a.y_hi) + i), g);
      } else if (a.y) {
        float4 o = __ldg(reinterpret_cast<const float4*>(a.y) + i);
        g.x = o.x > 0.f ? g.x : 0.f; g.y = o.y > 0.f ? g.y : 0.f; g.z = o.z > 0.f ? g.z : 0.f; g.w = o.w > 0.f ? g.w : 0.f;
      } else if (recompute_mask) {
        const float4 sc = *reinterpret_cast<const float4*>(b + 5 * C + c), be = *reinterpret_cast<const float4*>(b + 6 * C + c);
        if (!(fmaf(v.x - mu.x, sc.x, be.x) > 0.f)) g.x = 0.f;
        if (!(fmaf(v.y - mu.y, sc.y, be.y) > 0.f)) g.y = 0.f;
        if (!(fmaf(v.z - mu.z, sc.z, be.z) > 0.f)) g.z = 0.f;
        if (!(fmaf(v.w - mu.w, sc.w, be.w) > 0.f)) g.w = 0.f;
      }
    }
    if (a.g_out) reinterpret_cast<float4*>(a.g_out)[i] = g;
    float4 d;
    d.x = k1.x * (g.x - mb.x - (v.x - mu.x) * is.x * mg.x);
    d.y = k1.y * (g.y - mb.y - (v.y - mu.y) * is.y * mg.y);
    d.z = k1.z * (g.z - mb.z - (v.z - mu.z) * is.z * mg.z);
    d.w = k1.w * (g.w - mb.w - (v.w - mu.w) * is.w * mg.w);
    if (a.dx) reinterpret_cast<float4*>(a.dx)[i] = d;
    if (a.dx_hi) store_split4(a.dx_hi, a.dx_lo, i, d);
  }
}

// ------------------------------------------------------------------------------------------------ stem
// y[n,hp,wp,c] = max over the 3x3/2 pad-1 window of relu(bn(x));  argmax = first maximum in (r,s) scan order
__global__ void __launch_bounds__(256)
stem_bn_relu_pool_kernel(const float* __restrict__ x, const float* __restrict__ mean, const float* __restrict__ invstd,
                         const float* __restrict__ gamma, const float* __restrict__ beta,
                         float* __restrict__ y, uint8_t* __restrict__ argmax, __nv_bfloat16* __restrict__ y_hi,
                         __nv_bfloat16* __restrict__ y_lo, int N, int Hc, int Wc, int C, int Hp, int Wp, int imgs_per_group) {
  pdl_prologue();
  const int q = C >> 2;
  const int64_t total = (int64_t)N * Hp * Wp * q;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int c = (int)(i % q) << 2; int64_t t = i / q;
    int wp = (int)(t % Wp); t /= Wp;
    int hp = (int)(t % Hp); int n = (int)(t / Hp);
    const int so = (n / imgs_per_group) * C + c;
    float4 mu = *reinterpret_cast<const float4*>(mean + so), is = *reinterpret_cast<const float4*>(invstd + so);
    float4 ga = *reinterpret_cast<const float4*>(gamma + c), be = *reinterpret_cast<const float4*>(beta + c);
    float4 sc = make_float4(ga.x * is.x, ga.y * is.y, ga.z * is.z, ga.w * is.w);
    float4 best = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    uchar4 arg = make_uchar4(0, 0, 0, 0);
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      int h = 2 * hp - 1 + r;
      if (h < 0 || h >= Hc) continue;
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        int w = 2 * wp - 1 + s;
        if (w < 0 || w >= Wc) continue;
        float4 v = __ldg(reinterpret_cast<const float4*>(x + (((int64_t)n * Hc + h) * Wc + w) * C + c));
        v.x = fmaxf(fmaf(v.x - mu.x, sc.x, be.x), 0.f); v.y = fmaxf(fmaf(v.y - mu.y, sc.y, be.y), 0.f);
        v.z = fmaxf(fmaf(v.z - mu.z, sc.z, be.z), 0.f); v.w = fmaxf(fmaf(v.w - mu.w, sc.w, be.w), 0.f);
        unsigned char k = (unsigned char)(r * 3 + s);
        if (v.x > best.x) { best.x = v.x; arg.x = k; }
        if (v.y > best.y) { best.y = v.y; arg.y = k; }
        if (v.z > best.z) { best.z = v.z; arg.z = k; }
        if (v.w > best.w) { best.w = v.w; arg.w = k; }
      }
    }
    if (y) reinterpret_cast<float4*>(y)[i] = best;
    reinterpret_cast<uchar4*>(argmax)[i] = arg;
    if (y_hi) store_split4(y_hi, y_lo, i, best);
  }
}

// g[n,h,w,c] = (bn(x) > 0) * sum over pooling windows whose argmax is (h,w) of dy_pool
__global__ void __launch_bounds__(256)
stem_pool_relu_bwd_kernel(const float* __restrict__ dyp, const uint8_t* __restrict__ argmax, const float* __restrict__ x,
                          const float* __restrict__ mean, const float* __restrict__ invstd,
                          const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ g,
                          int N, int Hc, int Wc, int C, int Hp, int Wp, int imgs_per_group) {
  pdl_prologue();
  const int q = C >> 2;
  const int64_t total = (int64_t)N * Hc * Wc * q;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int c = (int)(i % q) << 2; int64_t t = i / q;
    int w = (int)(t % Wc); t /= Wc;
    int h = (int)(t % Hc); int n = (int)(t / Hc);
    float4 acc = make_float4(0, 0, 0, 0);
    int hp0 = h >> 1, hp1 = (h + 1) >> 1, wp0 = w >> 1, wp1 = (w + 1) >> 1;
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      int hp = a ? hp1 : hp0;
      if ((a && hp1 == hp0) || hp >= Hp) continue;
      int r = h - (2 * hp - 1);
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        int wp = b ? wp1 : wp0;
        if ((b && wp1 == wp0) || wp >= Wp) continue;
        int s = w - (2 * wp - 1);
        unsigned char k = (unsigned char)(r * 3 + s);
        int64_t pi = (((int64_t)n * Hp + hp) * Wp + wp) * q + (c >> 2);
        uchar4 am = reinterpret_cast<const uchar4*>(argmax)[pi];
        float4 d = __ldg(reinterpret_cast<const float4*>(dyp) + pi);
        if (am.x == k) acc.x += d.x;
        if (am.y == k) acc.y += d.y;
        if (am.z == k) acc.z += d.z;
        if (am.w == k) acc.w += d.w;
      }
    }
    const int so = (n / imgs_per_group) * C + c;
    float4 mu = *reinterpret_cast<const float4*>(mean + so), is = *reinterpret_cast<const float4*>(invstd + so);
    float4 ga = *reinterpret_cast<const float4*>(gamma + c), be = *reinterpret_cast<const float4*>(beta + c);
    float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
    if (!(fmaf(v.x - mu.x, ga.x * is.x, be.x) > 0.f)) acc.x = 0.f;
    if (!(fmaf(v.y - mu.y, ga.y * is.y, be.y) > 0.f)) acc.y = 0.f;
    if (!(fmaf(v.z - mu.z, ga.z * is.z, be.z) > 0.f)) acc.z = 0.f;
    if (!(fmaf(v.w - mu.w, ga.w * is.w, be.w) > 0.f)) acc.w = 0.f;
    reinterpret_cast<float4*>(g)[i] = acc;
  }
}

// ------------------------------------------------------------------------------------------------ launchers
bool bn_c_supported(int C) {
  return C >= 4 && C % 4 == 0 && (C <= BN_COLSUM_MAX_C ? BN_THREADS % (C / 4) == 0 : (C % BN_COLSUM_MAX_C == 0 && C <= 4096));
}

static int check_c(int C, int G, int64_t M) {
  DDN_CHECK_ARG(bn_c_supported(C), "BatchNorm kernels need C in {4..1024} with 256 %% (C/4) == 0, or a multiple of 1024 up to 4096 (got %d)", C);
  DDN_CHECK_ARG(G >= 1 && G <= BN_MAX_GROUPS && M % G == 0, "BatchNorm groups: need 1 <= G <= %d dividing the row count", BN_MAX_GROUPS);
  return 0;
}
// Grid of a grid-stride kernel = exactly the CTAs that are resident at once (SMs x occupancy): a larger grid runs a second,
// partial wave at low occupancy AFTER the first one has finished its (already complete-looking) share -- with 40 registers
// per thread only 6 CTAs of 256 threads fit an SM, and an 8-per-SM grid costs these kernels ~1.5x.
template <typename K>
static int resident_blocks(K kernel, size_t smem) {
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, BN_THREADS, smem) != cudaSuccess || per_sm < 1) per_sm = 4;
  return per_sm * num_sms();
}
template <typename K>
static int ew_blocks(K kernel, size_t smem, int64_t total) {
  return (int)std::min<int64_t>(ceil_div(total, BN_THREADS), (int64_t)resident_blocks(kernel, smem));
}

int launch_bn_stats(const float* x, int64_t M, int C, int G, BnAccum acc, float* mean, float* invstd,
                    float* running_mean, float* running_var, float momentum, float eps, cudaStream_t st) {
  DDN_TRY(check_c(C, G, M));
  const int64_t Mg = M / G;
  const int resident = resident_blocks(bn_colsum_kernel<0>, 0);
  const int Cs = bn_slice_c(C), slices = C / Cs;
  BnColsumArgs a = {x, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, Mg, C, bn_colsum_rows_per_block(Mg, C, G * slices, resident), 0, Cs};
  BnFwdFinal ff = {acc, mean, invstd, running_mean, running_var, Mg, G, C, momentum, eps};
  BnBwdFinal fb = {};
  dim3 grid((unsigned)bn_colsum_blocks(Mg, C, G * slices, resident), (unsigned)G, (unsigned)slices);
  DDN_LAUNCH(bn_colsum_kernel<0>, grid, BN_THREADS, 0, st, a, ff, fb);
  return 0;
}

int launch_bn_eval_stats(const float* rm, const float* rv, int C, int G, float eps, float* mean, float* invstd, cudaStream_t st) {
  DDN_LAUNCH(bn_eval_stats_kernel, (int)ceil_div(C, 128), 128, 0, st, rm, rv, C, G, eps, mean, invstd);
  return 0;
}

int launch_bn_eval_stats_all(const float* buffers, float* stats_base, const BnEvalSeg* segs, int n_segs, int G, float eps, cudaStream_t st) {
  DDN_CHECK_ARG(n_segs >= 1, "no BatchNorm segments");
  for (int i0 = 0; i0 < n_segs; i0 += BN_EVAL_MAX_SEGS) {     // one launch per table slice
    BnEvalSegs s; s.n = std::min(BN_EVAL_MAX_SEGS, n_segs - i0);
    for (int i = 0; i < s.n; ++i) s.s[i] = segs[i0 + i];
    dim3 grid(2, (unsigned)s.n);
    DDN_LAUNCH(bn_eval_stats_all_kernel, grid, 256, 0, st, buffers, stats_base, s, G, eps);
  }
  return 0;
}

int launch_bn_fold(const float* rm, const float* rv, const float* gamma, const float* beta, int C, float eps,
                   float* scale, float* shift, cudaStream_t st) {
  DDN_LAUNCH(bn_fold_kernel, (int)ceil_div(C, 128), 128, 0, st, rm, rv, gamma, beta, C, eps, scale, shift);
  return 0;
}

// the per-channel tables of the apply kernels exceed the default 48 KB of dynamic shared memory above C = 512 (G = 2)
template <typename K>
static int allow_smem(K kernel, size_t smem) {
  if (smem > 48 * 1024) DDN_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  return 0;
}

int launch_bn_apply(const BnApplyArgs& a, cudaStream_t st) {
  DDN_TRY(check_c(a.C, a.G, a.M));
  const size_t smem = (size_t)a.G * ((a.r && a.rmean) ? 6 : 3) * a.C * sizeof(float);
  DDN_TRY(allow_smem(bn_apply_kernel, smem));
  DDN_LAUNCH(bn_apply_kernel, ew_blocks(bn_apply_kernel, smem, a.M * (a.C / 4)), BN_THREADS, smem, st, a);
  return 0;
}

int launch_bn_backward(const BnBwdArgs& a, cudaStream_t st) {
  DDN_TRY(check_c(a.C, a.G, a.M));
  const int64_t Mg = a.M / a.G;
  const int resident = resident_blocks(bn_colsum_kernel<1>, 0);
  const int Cs = bn_slice_c(a.C), slices = a.C / Cs;
  BnColsumArgs ca = {a.x, a.dy, a.y, a.y_hi, a.mean, a.invstd, a.gamma, a.beta, Mg, a.C, bn_colsum_rows_per_block(Mg, a.C, a.G * slices, resident),
                     a.relu, Cs};
  DDN_CHECK_ARG(!(a.relu && !a.y && !a.y_hi) || a.beta, "recomputing the ReLU mask needs beta");
  BnFwdFinal ff = {};
  BnBwdFinal fb = {a.acc, a.sums, a.dgamma, a.dbeta, a.G, a.C};
  dim3 grid((unsigned)bn_colsum_blocks(Mg, a.C, a.G * slices, resident), (unsigned)a.G, (unsigned)slices);
  if (!a.sums_ready) DDN_LAUNCH(bn_colsum_kernel<1>, grid, BN_THREADS, 0, st, ca, ff, fb);
  const size_t smem = (size_t)a.G * 7 * a.C * sizeof(float);
  DDN_TRY(allow_smem(bn_bwd_apply_kernel, smem));
  DDN_LAUNCH(bn_bwd_apply_kernel, ew_blocks(bn_bwd_apply_kernel, smem, a.M * (a.C / 4)), BN_THREADS, smem, st, a);
  return 0;
}

int launch_stem_bn_relu_pool(const float* x, const float* mean, const float* invstd, const float* gamma, const float* beta,
                             float* y, uint8_t* argmax, __nv_bfloat16* y_hi, __nv_bfloat16* y_lo,
                             int N, int Hc, int Wc, int C, int G, cudaStream_t st) {
  int Hp = (Hc - 1) / 2 + 1, Wp = (Wc - 1) / 2 + 1;
  int64_t total = (int64_t)N * Hp * Wp * (C / 4);
  DDN_LAUNCH(stem_bn_relu_pool_kernel, ew_blocks(stem_bn_relu_pool_kernel, 0, total), 256, 0, st, x, mean, invstd, gamma, beta, y, argmax, y_hi, y_lo, N, Hc, Wc, C,
             Hp, Wp, N / G);
  return 0;
}

int launch_stem_pool_relu_backward(const float* dy_pool, const uint8_t* argmax, const float* x, const float* mean,
                                   const float* invstd, const float* gamma, const float* beta, float* g,
                                   int N, int Hc, int Wc, int C, int G, cudaStream_t st) {
  int Hp = (Hc - 1) / 2 + 1, Wp = (Wc - 1) / 2 + 1;
  int64_t total = (int64_t)N * Hc * Wc * (C / 4);
  DDN_LAUNCH(stem_pool_relu_bwd_kernel, ew_blocks(stem_pool_relu_bwd_kernel, 0, total), 256, 0, st, dy_pool, argmax, x, mean, invstd, gamma, beta, g,
             N, Hc, Wc, C, Hp, Wp, N / G);
  return 0;
}

}  // namespace ddn
