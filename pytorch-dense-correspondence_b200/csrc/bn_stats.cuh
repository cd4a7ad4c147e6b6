// Per-channel batch statistics without a second kernel launch.
//
// Every CTA that holds partial column sums (a conv epilogue's tile, a BatchNorm column-sum block) adds them with fp64
// `red.global.add` into ONE small accumulator [G][2][C]; the CTAs then take a ticket, and the last one to arrive turns
// the sums into BatchNorm statistics (forward: mean / 1/sqrt(var+eps) / running statistics; backward: dgamma, dbeta and
// the per-group sums the dx pass needs), zeroes the accumulator and resets the ticket for the next user.  This replaces
// per-tile partial-sum buffers and a separate `bn_*_finalize` launch per BatchNorm.
//
// G = number of BatchNorm groups in the batch: images [g*B/G, (g+1)*B/G) share one set of batch statistics.  G = 1 is
// nn.BatchNorm2d over the whole call; G = 2 is the pair-batched step (image A batch and image B batch of
// dense_correspondence/training/training.py:329-333 in ONE launch, each normalised by its own statistics, running
// statistics updated A-then-B exactly as the two reference forward calls would).
//
// Reference semantics: nn.BatchNorm2d as wired by PSD/vision/torchvision/models/resnet.py:46-69 (biased variance for
// normalisation, unbiased for the running estimate, eps inside the sqrt).
#pragma once
#include "common.cuh"

namespace ddn {

constexpr int BN_MAX_GROUPS = 2;

struct BnAccum {
  double* acc;            // [G][2][C], all zero between users
  unsigned int* ticket;   // zero between users
};

struct BnFwdFinal {
  BnAccum a;
  float* mean; float* invstd;                 // [G][C]
  float* running_mean; float* running_var;    // [C] or null (left untouched)
  int64_t count;                              // elements per channel and group (= B/G * Ho * Wo)
  int G, C;
  float momentum, eps;
};

struct BnBwdFinal {
  BnAccum a;
  float* sums;            // [G][2][C] floats: (sum g, sum g*xhat) per group, read by the dx pass
  float* dgamma; float* dbeta;                // [C], overwritten with the sum over groups
  int G, C;
};

__device__ __forceinline__ void red_add_f64(double* addr, double v) {
  asm volatile("red.global.add.f64 [%0], %1;" ::"l"(addr), "d"(v) : "memory");
}

// One thread of the finalizing CTA per channel.
__device__ __forceinline__ void bn_fwd_finalize_channel(const BnFwdFinal& f, int c) {
  float rm = f.running_mean ? f.running_mean[c] : 0.f, rv = f.running_var ? f.running_var[c] : 0.f;
  for (int g = 0; g < f.G; ++g) {
    double* ps = f.a.acc + (size_t)(g * 2) * f.C + c;
    double* pq = ps + f.C;
    const double s = __ldcg(ps), ss = __ldcg(pq);
    *ps = 0.0; *pq = 0.0;
    const double mu = s / (double)f.count;
    double var = ss / (double)f.count - mu * mu;
    if (var < 0) var = 0;
    f.mean[g * f.C + c] = (float)mu;
    f.invstd[g * f.C + c] = (float)(1.0 / sqrt(var + (double)f.eps));
    if (f.running_mean) {       // sequential updates: group 0 first, then group 1 (= forward(A), then forward(B))
      const double unbiased = f.count > 1 ? var * (double)f.count / (double)(f.count - 1) : var;
      rm = (float)((1.0 - f.momentum) * (double)rm + f.momentum * mu);
      rv = (float)((1.0 - f.momentum) * (double)rv + f.momentum * unbiased);
    }
  }
  if (f.running_mean) { f.running_mean[c] = rm; f.running_var[c] = rv; }
}

__device__ __forceinline__ void bn_bwd_finalize_channel(const BnBwdFinal& f, int c) {
  double db = 0, dg = 0;
  for (int g = 0; g < f.G; ++g) {
    double* ps = f.a.acc + (size_t)(g * 2) * f.C + c;
    double* pq = ps + f.C;
    const double s = __ldcg(ps), ss = __ldcg(pq);
    *ps = 0.0; *pq = 0.0;
    f.sums[(g * 2) * f.C + c] = (float)s;
    f.sums[(g * 2 + 1) * f.C + c] = (float)ss;
    db += s; dg += ss;
  }
  f.dbeta[c] = (float)db;
  f.dgamma[c] = (float)dg;
}

// Ticket: every participating thread group of every CTA calls this once after its last red.  `sync` is the barrier of
// the participating threads (the whole block, or a named barrier of the epilogue warps); `leader` is true in exactly one
// of them.  Returns true (in all participating threads) in the CTA that arrived last.
template <typename Sync>
__device__ __forceinline__ bool bn_last_cta(unsigned int* ticket, unsigned int n_ctas, bool leader, int* s_flag, Sync sync) {
  __threadfence();            // this thread's reds are ordered before the ticket
  sync();
  if (leader) {
    const unsigned int old = atomicAdd(ticket, 1u);
    *s_flag = (old == n_ctas - 1) ? 1 : 0;
    if (old == n_ctas - 1) *ticket = 0u;     // nobody else touches it any more in this launch
  }
  sync();
  const bool last = *s_flag != 0;
  if (last) __threadfence();  // acquire side: the other CTAs' reds are visible to the loads below
  return last;
}

}  // namespace ddn
