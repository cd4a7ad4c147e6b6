// Pixelwise contrastive loss: gather + squared-L2 / hinge + reduction in one pass, and its
// hand-written backward (recompute + scatter-add).  HBM-bound: 16 + 8*D algorithmic bytes per
// index pair forward, 16 + 24*D backward (SURVEY.md 8d).
//
// Reference semantics (dense_correspondence/loss_functions/pixelwise_contrastive_loss.py):
//   match term   :131-167   hinge vector + nonzero count :170-213   pixel weight :307-352
// and loss_composer.get_within_scene_loss (loss_composer.py:70-143) for the compose kernel.
#include "loss.cuh"

namespace ddn {

template <int D_T>
__global__ void __launch_bounds__(LOSS_THREADS)
loss_terms_fwd_kernel(const float* __restrict__ pa, const float* __restrict__ pb,
                      int64_t sb, int64_t sp, int64_t sc, int64_t P, int D_rt, int W,
                      const __grid_constant__ DevTerms T, double* __restrict__ sums,
                      unsigned long long* __restrict__ counts) {
  pdl_prologue();
  const int D = D_T > 0 ? D_T : D_rt;
  const int b = blockIdx.y;
  const int t = find_term(T, blockIdx.x);
  const DevTerm& tm = T.t[t];
  const int64_t base = (int64_t)(blockIdx.x - tm.block_begin) * (LOSS_THREADS * LOSS_ITEMS);
  const float* A = pa + b * sb;
  const float* Bp = pb + b * sb;
  const int64_t* ia = tm.ia + b * tm.n;
  const int64_t* ib = tm.ib + b * tm.n;

  const int64_t nvalid = tm.len ? min(tm.len[b], tm.n) : tm.n;
  float acc = 0.f;
  int cnt = 0;
  int64_t ja[LOSS_ITEMS], jb[LOSS_ITEMS];
#pragma unroll
  for (int it = 0; it < LOSS_ITEMS; ++it) {   // all index loads first (MLP)
    int64_t j = base + it * LOSS_THREADS + threadIdx.x;
    bool ok = j < nvalid;
    ja[it] = ok ? __ldg(ia + j) : -1;
    jb[it] = ok ? __ldg(ib + j) : -1;
  }
#pragma unroll
  for (int it = 0; it < LOSS_ITEMS; ++it) {
    int64_t j = base + it * LOSS_THREADS + threadIdx.x;
    int64_t na = ja[it], nb = jb[it];
    if (na < 0 || nb < 0 || na >= P || nb >= P) continue;
    const float* a = A + na * sp;
    const float* bq = Bp + nb * sp;
    float s2 = 0.f;
#pragma unroll
    for (int c = 0; c < (D_T > 0 ? D_T : LOSS_MAXD); ++c) {
      if (c < D) {
        float d = __ldg(a + c * sc) - __ldg(bq + c * sc);
        s2 = fmaf(d, d, s2);
      }
    }
    if (tm.kind == DDN_TERM_MATCH) {
      acc += s2;
    } else {
      float d = sqrtf(s2);
      float h = (tm.kind == DDN_TERM_HINGE) ? fmaxf(tm.margin - d, 0.f) : fmaxf(d - tm.margin, 0.f);
      float l = h * h;
      cnt += (l != 0.f);
      if (tm.flags & DDN_TERM_PIXEL_WEIGHT) l *= pixel_weight(tm, b, j, nb, W);
      acc += l;
    }
  }
  // block reduction: fp64 from the warp level up, one atomic pair per block
  double wsum = warp_sum((double)acc);
  int wcnt = warp_sum(cnt);
  __shared__ double s_sum[LOSS_THREADS / 32];
  __shared__ int s_cnt[LOSS_THREADS / 32];
  int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) { s_sum[wid] = wsum; s_cnt[wid] = wcnt; }
  __syncthreads();
  if (wid == 0) {
    double v = lane < LOSS_THREADS / 32 ? s_sum[lane] : 0.0;
    int c = lane < LOSS_THREADS / 32 ? s_cnt[lane] : 0;
    v = warp_sum(v);
    c = warp_sum(c);
    if (lane == 0) {
      atomicAdd(&sums[b * T.n_terms + t], v);
      if (c) atomicAdd(&counts[b * T.n_terms + t], (unsigned long long)c);
    }
  }
}

// Backward: recompute the per-pair quantities, scatter coef * d(l_j)/d(descriptor).
// A-side indices of the hinge terms come in runs (every match repeated k times consecutively,
// spartan_dataset_masked.py:853-854): a segmented warp reduction folds each run into ONE atomic per channel.
template <int D_T>
__global__ void __launch_bounds__(LOSS_THREADS)
loss_terms_bwd_kernel(const float* __restrict__ pa, const float* __restrict__ pb,
                      int64_t sb, int64_t sp, int64_t sc, int64_t P, int D_rt, int W,
                      const __grid_constant__ DevTerms T, const float* __restrict__ coef,
                      const float* __restrict__ upstream, float* __restrict__ da, float* __restrict__ db) {
  pdl_prologue();
  const int D = D_T > 0 ? D_T : D_rt;
  constexpr int DM = D_T > 0 ? D_T : LOSS_MAXD;
  const int b = blockIdx.y;
  const int t = find_term(T, blockIdx.x);
  const DevTerm& tm = T.t[t];
  float cf = coef[b * T.n_terms + t];
  if (upstream) cf *= upstream[0];
  const int64_t base = (int64_t)(blockIdx.x - tm.block_begin) * (LOSS_THREADS * LOSS_ITEMS);
  const float* A = pa + b * sb;
  const float* Bp = pb + b * sb;
  float* dA = da + b * sb;
  float* dB = db + b * sb;
  const int64_t* ia = tm.ia + b * tm.n;
  const int64_t* ib = tm.ib + b * tm.n;
  const int lane = threadIdx.x & 31;
  const bool hinge = tm.kind != DDN_TERM_MATCH;
  const int64_t nvalid = tm.len ? min(tm.len[b], tm.n) : tm.n;

#pragma unroll 1
  for (int it = 0; it < LOSS_ITEMS; ++it) {
    int64_t j = base + it * LOSS_THREADS + threadIdx.x;
    int64_t na = -1, nb = -1;
    if (j < nvalid) { na = __ldg(ia + j); nb = __ldg(ib + j); }
    bool ok = na >= 0 && nb >= 0 && na < P && nb < P;
    float g[DM];
    float s2 = 0.f;
#pragma unroll
    for (int c = 0; c < DM; ++c) {
      g[c] = 0.f;
      if (ok && c < D) {
        float d = __ldg(A + na * sp + c * sc) - __ldg(Bp + nb * sp + c * sc);
        g[c] = d;
        s2 = fmaf(d, d, s2);
      }
    }
    float scale = 0.f;
    if (ok) {
      if (!hinge) {
        scale = 2.f * cf;                                  // d/dA ||A-B||^2
      } else {
        float d = sqrtf(s2);
        float h = (tm.kind == DDN_TERM_HINGE) ? fmaxf(tm.margin - d, 0.f) : fmaxf(d - tm.margin, 0.f);
        if (h * h != 0.f && d > 0.f) {                     // norm's subgradient at 0 is 0 (torch)
          float w = (tm.flags & DDN_TERM_PIXEL_WEIGHT) ? pixel_weight(tm, b, j, nb, W) : 1.f;
          float sgn = (tm.kind == DDN_TERM_HINGE) ? -1.f : 1.f;
          scale = cf * w * sgn * 2.f * h / d;
        }
      }
    }
#pragma unroll
    for (int c = 0; c < DM; ++c) g[c] *= scale;
    // B side: random indices, plain atomics
    if (scale != 0.f) {
#pragma unroll
      for (int c = 0; c < DM; ++c)
        if (c < D) atomicAdd(dB + nb * sp + c * sc, -g[c]);
    }
    // A side
    if (!hinge) {
      if (scale != 0.f) {
#pragma unroll
        for (int c = 0; c < DM; ++c)
          if (c < D) atomicAdd(dA + na * sp + c * sc, g[c]);
      }
    } else {
      // segmented suffix-sum over runs of equal keys (whole warp participates)
      int64_t key = ok ? na : (int64_t)(-1 - lane);
      int64_t prev = __shfl_up_sync(0xffffffffu, key, 1);
      bool head = (lane == 0) || (prev != key);
      unsigned heads = __ballot_sync(0xffffffffu, head);
      unsigned above = heads & ~((2u << lane) - 1u);          // run heads at higher lanes
      int run_end = above ? (__ffs(above) - 2) : 31;          // last lane of my run
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        bool take = (lane + off) <= run_end;
#pragma unroll
        for (int c = 0; c < DM; ++c) {
          if (c < D) {
            float o = __shfl_down_sync(0xffffffffu, g[c], off);
            if (take) g[c] += o;
          }
        }
      }
      if (head && ok) {
#pragma unroll
        for (int c = 0; c < DM; ++c)
          if (c < D && g[c] != 0.f) atomicAdd(dA + na * sp + c * sc, g[c]);
      }
    }
  }
}

__global__ void within_scene_compose_kernel(const double* __restrict__ sums, const unsigned long long* __restrict__ counts,
                                            int B, int n_terms, ddn_within_scene_cfg cfg,
                                            float* __restrict__ five, float* __restrict__ coef) {
  pdl_prologue();
  // One warp; lane-strided over pairs.  loss_composer.py:107-141.
  double acc[5] = {0, 0, 0, 0, 0};
  for (int b = threadIdx.x; b < B; b += 32) {
    const double* S = sums + b * n_terms;
    const unsigned long long* H = counts + b * n_terms;
    const long long n_match = cfg.len_match ? (long long)cfg.len_match[b] : (long long)cfg.n_match;
    double match = S[0] / (double)(n_match > 1 ? n_match : 1);
    double Sm = S[1], Sb = S[2], Sx = cfg.has_blind ? S[3] : 0.0;
    double scale, tm, tb, tx;
    if (cfg.scale_by_hard_negatives) {
      long long hm = (long long)H[1], hb = (long long)H[2], hx = cfg.has_blind ? (long long)H[3] : 1;
      long long tot = hm + hb; if (tot < 1) tot = 1;
      scale = (double)tot;
      tm = Sm / (double)(hm > 1 ? hm : 1);
      tb = Sb / (double)(hb > 1 ? hb : 1);
      tx = Sx / (double)(hx > 1 ? hx : 1);
    } else {
      long long nm = cfg.len_masked ? (long long)cfg.len_masked[b] : (long long)cfg.n_masked;
      long long nb = cfg.len_background ? (long long)cfg.len_background[b] : (long long)cfg.n_background;
      long long nx = cfg.len_blind ? (long long)cfg.len_blind[b] : (long long)cfg.n_blind;
      nm = nm > 1 ? nm : 1; nb = nb > 1 ? nb : 1; nx = nx > 1 ? nx : 1;
      scale = (double)(nm + nb);
      tm = Sm / (double)nm; tb = Sb / (double)nb; tx = Sx / (double)nx;
    }
    double non_match = (Sm + Sb) / scale;
    double loss = cfg.match_loss_weight * match + cfg.non_match_loss_weight * non_match;
    acc[0] += loss; acc[1] += match; acc[2] += tm; acc[3] += tb; acc[4] += tx;
    float* cf = coef + b * n_terms;
    cf[0] = (float)(cfg.match_loss_weight / ((double)(n_match > 1 ? n_match : 1) * B));
    cf[1] = cf[2] = (float)(cfg.non_match_loss_weight / (scale * B));
    if (n_terms > 3) cf[3] = 0.f;   // blind non-matches are reported, never optimised (loss_composer.py:136-139)
  }
#pragma unroll
  for (int i = 0; i < 5; ++i) {
    double v = warp_sum(acc[i]);
    if (threadIdx.x == 0) five[i] = (float)(v / B);
  }
}

// SpartanDatasetDataType.DIFFERENT_OBJECT (dataset/spartan_dataset_masked.py:31-36); every other type the caller lets
// through is a within-scene type.
constexpr int PAIR_DIFFERENT_OBJECT = 2;

// Terms {match, masked, background, blind@M_masked, blind@M_background}.  Each pair takes its own type's formula:
// within-scene types as within_scene_compose_kernel with the blind term (loss_composer.py:70-143), DIFFERENT_OBJECT
// loss_composer.py:168-191.  One warp, lane-strided over pairs, then a fixed-order warp sum, as the kernel above.
__global__ void pair_type_compose_kernel(const double* __restrict__ sums, const unsigned long long* __restrict__ counts,
                                         int B, ddn_pair_type_cfg cfg, const int32_t* __restrict__ pair_type,
                                         float* __restrict__ five, float* __restrict__ coef) {
  pdl_prologue();
  constexpr int NT = 5;
  double acc[5] = {0, 0, 0, 0, 0};
  for (int b = threadIdx.x; b < B; b += 32) {
    const double* S = sums + b * NT;
    const unsigned long long* H = counts + b * NT;
    float* cf = coef + b * NT;
    if (pair_type[b] == PAIR_DIFFERENT_OBJECT) {
      long long n;
      if (cfg.scale_by_hard_negatives_different_object) n = (long long)H[4];
      else n = cfg.len_blind ? (long long)cfg.len_blind[b] : (long long)cfg.n_blind;
      const double scale = (double)(n > 1 ? n : 1);
      const double blind = S[4] / scale;
      acc[0] += blind; acc[4] += blind;
      cf[0] = cf[1] = cf[2] = cf[3] = 0.f;
      cf[4] = (float)(1.0 / (scale * B));
      continue;
    }
    const long long n_match = cfg.len_match ? (long long)cfg.len_match[b] : (long long)cfg.n_match;
    double match = S[0] / (double)(n_match > 1 ? n_match : 1);
    double Sm = S[1], Sb = S[2], Sx = S[3];
    double scale, tm, tb, tx;
    if (cfg.scale_by_hard_negatives) {
      long long hm = (long long)H[1], hb = (long long)H[2], hx = (long long)H[3];
      long long tot = hm + hb; if (tot < 1) tot = 1;
      scale = (double)tot;
      tm = Sm / (double)(hm > 1 ? hm : 1);
      tb = Sb / (double)(hb > 1 ? hb : 1);
      tx = Sx / (double)(hx > 1 ? hx : 1);
    } else {
      long long nm = cfg.len_masked ? (long long)cfg.len_masked[b] : (long long)cfg.n_masked;
      long long nb = cfg.len_background ? (long long)cfg.len_background[b] : (long long)cfg.n_background;
      long long nx = cfg.len_blind ? (long long)cfg.len_blind[b] : (long long)cfg.n_blind;
      nm = nm > 1 ? nm : 1; nb = nb > 1 ? nb : 1; nx = nx > 1 ? nx : 1;
      scale = (double)(nm + nb);
      tm = Sm / (double)nm; tb = Sb / (double)nb; tx = Sx / (double)nx;
    }
    double non_match = (Sm + Sb) / scale;
    double loss = cfg.match_loss_weight * match + cfg.non_match_loss_weight * non_match;
    acc[0] += loss; acc[1] += match; acc[2] += tm; acc[3] += tb; acc[4] += tx;
    cf[0] = (float)(cfg.match_loss_weight / ((double)(n_match > 1 ? n_match : 1) * B));
    cf[1] = cf[2] = (float)(cfg.non_match_loss_weight / (scale * B));
    cf[3] = cf[4] = 0.f;   // blind non-matches of a within-scene pair are reported, never optimised
  }
#pragma unroll
  for (int i = 0; i < 5; ++i) {
    double v = warp_sum(acc[i]);
    if (threadIdx.x == 0) five[i] = (float)(v / B);
  }
}

__global__ void scale_inplace_kernel(float* __restrict__ g, int64_t n, float s) {
  pdl_prologue();
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t n4 = n >> 2;
  for (int64_t k = i; k < n4; k += (int64_t)gridDim.x * blockDim.x) {
    float4 v = reinterpret_cast<float4*>(g)[k];
    v.x *= s; v.y *= s; v.z *= s; v.w *= s;
    reinterpret_cast<float4*>(g)[k] = v;
  }
  if (i < (n & 3)) g[(n4 << 2) + i] *= s;
}

}  // namespace ddn

using namespace ddn;

extern "C" int ddn_contrastive_terms_forward(const float* pred_a, const float* pred_b,
                                             int64_t stride_b, int64_t stride_p, int64_t stride_c,
                                             int B, int64_t P, int D, int image_width,
                                             const ddn_loss_term* terms_host, int n_terms,
                                             double* sums, int64_t* counts, void* stream) {
  DDN_TRY(check_common(pred_a, pred_b, B, P, D, image_width));
  DDN_CHECK_ARG(sums && counts, "null outputs");
  DevTerms T;
  DDN_TRY(build_terms(terms_host, n_terms, &T));
  cudaStream_t st = (cudaStream_t)stream;
  DDN_CUDA(cudaMemsetAsync(sums, 0, sizeof(double) * B * n_terms, st));
  DDN_CUDA(cudaMemsetAsync(counts, 0, sizeof(int64_t) * B * n_terms, st));
  if (T.total_blocks == 0) return 0;
  dim3 grid(T.total_blocks, B);
  auto cnt = reinterpret_cast<unsigned long long*>(counts);
  double pairs = 0;
  for (int i = 0; i < n_terms; ++i) pairs += (double)terms_host[i].n * B;
  ProfScope ps(PROF_LOSS_FWD, pairs * (16.0 + 8.0 * D), st);
#define FWD(DT) DDN_LAUNCH(loss_terms_fwd_kernel<DT>, grid, LOSS_THREADS, 0, st, pred_a, pred_b, stride_b, stride_p, \
                           stride_c, P, D, image_width, T, sums, cnt)
  switch (D) {
    case 3: FWD(3); break;
    case 8: FWD(8); break;
    case 16: FWD(16); break;
    default: FWD(0); break;
  }
#undef FWD
  return 0;
}

extern "C" int ddn_contrastive_terms_backward(const float* pred_a, const float* pred_b,
                                              int64_t stride_b, int64_t stride_p, int64_t stride_c,
                                              int B, int64_t P, int D, int image_width,
                                              const ddn_loss_term* terms_host, int n_terms,
                                              const float* coef, const float* upstream,
                                              float* dpred_a, float* dpred_b, void* stream) {
  DDN_TRY(check_common(pred_a, pred_b, B, P, D, image_width));
  DDN_CHECK_ARG(coef && dpred_a && dpred_b, "null coef / gradient buffers");
  DevTerms T;
  DDN_TRY(build_terms(terms_host, n_terms, &T));
  if (T.total_blocks == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  dim3 grid(T.total_blocks, B);
  double pairs = 0;
  for (int i = 0; i < n_terms; ++i) pairs += (double)terms_host[i].n * B;
  ProfScope ps(PROF_LOSS_BWD, pairs * (16.0 + 24.0 * D), st);
#define BWD(DT) DDN_LAUNCH(loss_terms_bwd_kernel<DT>, grid, LOSS_THREADS, 0, st, pred_a, pred_b, stride_b, stride_p, \
                           stride_c, P, D, image_width, T, coef, upstream, dpred_a, dpred_b)
  switch (D) {
    case 3: BWD(3); break;
    case 8: BWD(8); break;
    case 16: BWD(16); break;
    default: BWD(0); break;
  }
#undef BWD
  return 0;
}

extern "C" int ddn_within_scene_compose(const double* sums, const int64_t* counts, int B, int n_terms,
                                        const ddn_within_scene_cfg* cfg, float* five, float* coef, void* stream) {
  DDN_CHECK_ARG(sums && counts && cfg && five && coef, "null argument");
  DDN_CHECK_ARG(B >= 1 && (n_terms == 3 || n_terms == 4), "within-scene compose needs 3 or 4 terms");
  DDN_CHECK_ARG((cfg->has_blind != 0) == (n_terms == 4), "has_blind must match n_terms");
  DDN_CHECK_ARG(cfg->n_match > 0, "n_match must be positive");
  DDN_LAUNCH(within_scene_compose_kernel, 1, 32, 0, (cudaStream_t)stream, sums,
             reinterpret_cast<const unsigned long long*>(counts), B, n_terms, *cfg, five, coef);
  return 0;
}

extern "C" int ddn_pair_type_compose(const double* sums, const int64_t* counts, int B, int n_terms,
                                     const ddn_pair_type_cfg* cfg, const int32_t* pair_type, float* five, float* coef,
                                     void* stream) {
  DDN_CHECK_ARG(sums && counts && cfg && pair_type && five && coef, "null argument");
  DDN_CHECK_ARG(B >= 1 && n_terms == 5, "pair-type compose needs B >= 1 and 5 terms");
  DDN_LAUNCH(pair_type_compose_kernel, 1, 32, 0, (cudaStream_t)stream, sums,
             reinterpret_cast<const unsigned long long*>(counts), B, *cfg, pair_type, five, coef);
  return 0;
}

extern "C" int ddn_scale_inplace(float* g, int64_t n, float scale, void* stream) {
  DDN_CHECK_ARG(g && n >= 0, "bad buffer");
  if (n == 0) return 0;
  DDN_CHECK_ARG((reinterpret_cast<uintptr_t>(g) & 15) == 0, "buffer must be 16-byte aligned");
  int blocks = (int)std::min<int64_t>(ceil_div(n / 4 + 1, 256), (int64_t)num_sms() * 8);
  DDN_LAUNCH(scale_inplace_kernel, blocks, 256, 0, (cudaStream_t)stream, g, n, scale);
  return 0;
}

extern "C" int ddn_within_scene_loss_host(const float* pred_a_host, const float* pred_b_host,
                                          int B, int H, int W, int D,
                                          const int64_t* ma, const int64_t* mb, int64_t n_match,
                                          const int64_t* ka, const int64_t* kb, int64_t n_masked,
                                          const int64_t* ga, const int64_t* gb, int64_t n_background,
                                          float m_masked, float m_background,
                                          float match_loss_weight, float non_match_loss_weight,
                                          int scale_by_hard_negatives, float* five_host) {
  DDN_CHECK_ARG(pred_a_host && pred_b_host && five_host && ma && mb && ka && kb && ga && gb, "null host buffer");
  DDN_CHECK_ARG(B >= 1 && H >= 1 && W >= 1 && n_match > 0 && n_masked >= 0 && n_background >= 0, "bad sizes");
  const int64_t P = (int64_t)H * W;
  const size_t img_bytes = sizeof(float) * (size_t)B * D * P;
  const size_t n_idx = (size_t)B * (2 * n_match + 2 * n_masked + 2 * n_background);
  cudaStream_t st;
  DDN_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  char* dev = nullptr;
  size_t tail = sizeof(double) * B * 3 + sizeof(int64_t) * B * 3 + sizeof(float) * (5 + 3 * B) + 256;
  int rc = (int)cudaMalloc(&dev, 2 * img_bytes + n_idx * sizeof(int64_t) + tail);
  if (rc) { set_error("cudaMalloc failed"); cudaStreamDestroy(st); return rc; }
  float* da = (float*)dev; float* db = (float*)(dev + img_bytes);
  int64_t* di = (int64_t*)(dev + 2 * img_bytes);
  auto up = [&](int64_t*& cur, const int64_t* h, int64_t n) {
    int64_t* p = cur; cudaMemcpyAsync(p, h, sizeof(int64_t) * B * n, cudaMemcpyHostToDevice, st); cur += (size_t)B * n; return p; };
  cudaMemcpyAsync(da, pred_a_host, img_bytes, cudaMemcpyHostToDevice, st);
  cudaMemcpyAsync(db, pred_b_host, img_bytes, cudaMemcpyHostToDevice, st);
  int64_t* cur = di;
  ddn_loss_term terms[3] = {};
  terms[0].idx_a = up(cur, ma, n_match); terms[0].idx_b = up(cur, mb, n_match); terms[0].n = n_match; terms[0].kind = DDN_TERM_MATCH;
  terms[1].idx_a = up(cur, ka, n_masked); terms[1].idx_b = up(cur, kb, n_masked); terms[1].n = n_masked; terms[1].kind = DDN_TERM_HINGE; terms[1].margin = m_masked;
  terms[2].idx_a = up(cur, ga, n_background); terms[2].idx_b = up(cur, gb, n_background); terms[2].n = n_background; terms[2].kind = DDN_TERM_HINGE; terms[2].margin = m_background;
  char* t0 = (char*)align_up((size_t)cur, 16);
  double* sums = (double*)t0; int64_t* counts = (int64_t*)(sums + 3 * B);
  float* five = (float*)(counts + 3 * B); float* coef = five + 8;
  ddn_within_scene_cfg cfg = {match_loss_weight, non_match_loss_weight, scale_by_hard_negatives, 0,
                              n_match, n_masked, n_background, 0, nullptr, nullptr, nullptr, nullptr};
  rc = ddn_contrastive_terms_forward(da, db, (int64_t)D * P, 1, P, B, P, D, W, terms, 3, sums, counts, st);
  if (!rc) rc = ddn_within_scene_compose(sums, counts, B, 3, &cfg, five, coef, st);
  if (!rc) rc = (int)cudaMemcpyAsync(five_host, five, 5 * sizeof(float), cudaMemcpyDeviceToHost, st);
  if (!rc) rc = (int)cudaStreamSynchronize(st);
  cudaFree(dev);
  cudaStreamDestroy(st);
  if (rc > 0) set_error("ddn_within_scene_loss_host: %s", cudaGetErrorString((cudaError_t)rc));
  return rc;
}
