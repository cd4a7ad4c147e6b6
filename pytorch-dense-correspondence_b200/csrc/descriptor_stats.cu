// Per-image, per-channel descriptor statistics on the device (SURVEY.md 8f row 4, the evaluation consumer of the backbone).
// Replaces compute_descriptor_statistics (dense_correspondence/evaluation/evaluation.py:2177-2219), which the reference
// runs once per image inside compute_descriptor_statistics_on_dataset (:2157-2305): min / max / mean over the whole
// descriptor image and over its object mask.
//
// descriptor_stats_kernel: grid (pixel blocks, N).  A block sweeps its pixel range once per chunk of DS_CHUNK channels
//   (so a thread holds 8 channels' running values, not 32), reduces them in a fixed order (xor-shuffle tree inside each
//   warp, then the warps in index order) and writes one partial record per channel.  The image's last block to finish
//   (bn_stats.cuh's ticket) adds the partial records in block order and writes the statistics: one launch for all images,
//   deterministic.
// Reads every descriptor once (N*H*W*D*4 bytes) and the mask once per channel chunk (the later reads hit L2).  A thread
// issues the loads of DS_UNROLL pixels before it uses them, so that enough bytes are in flight to approach HBM bandwidth.
#include <cmath>
#include "bn_stats.cuh"
#include "common.cuh"

namespace ddn {

constexpr int DS_THREADS = 256;
constexpr int DS_CHUNK = 8;
constexpr int DS_UNROLL = 4;
constexpr int DS_MAXD = 32;

struct DsImage {
  const float* base;
  int64_t sn, sh, sw, sc;
};

// per (image, pixel block, channel); counts per (image, pixel block)
struct DsScratch {
  double* sum; double* msum;
  float* mn; float* mx; float* mmn; float* mmx;
  unsigned long long* cnt;
  unsigned int* ticket;       // [N], zero on entry and on exit
};

// torch.min / torch.max semantics: a NaN anywhere wins
__device__ __forceinline__ float ds_min(float a, float b) { return (a < b || a != a) ? a : b; }
__device__ __forceinline__ float ds_max(float a, float b) { return (a > b || a != a) ? a : b; }

template <typename MaskT>
__global__ void __launch_bounds__(DS_THREADS)
descriptor_stats_kernel(DsImage im, const MaskT* __restrict__ mask, int H, int W, int D, int pixels_per_block, DsScratch s,
                        float* __restrict__ out, int64_t* __restrict__ out_count) {
  pdl_prologue();
  const int n = blockIdx.y, nbx = gridDim.x;
  const int64_t P = (int64_t)H * W;
  const int64_t p0 = (int64_t)blockIdx.x * pixels_per_block;
  const int64_t p1 = min(P, p0 + pixels_per_block);
  const MaskT* mk = mask + (int64_t)n * P;
  const float* img = im.base + (int64_t)n * im.sn;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool dense = im.sh == (int64_t)W * im.sw;
  __shared__ double r_sum[DS_THREADS / 32][DS_CHUNK], r_msum[DS_THREADS / 32][DS_CHUNK];
  __shared__ float r_mn[DS_THREADS / 32][DS_CHUNK], r_mx[DS_THREADS / 32][DS_CHUNK];
  __shared__ float r_mmn[DS_THREADS / 32][DS_CHUNK], r_mmx[DS_THREADS / 32][DS_CHUNK];
  __shared__ unsigned long long r_cnt[DS_THREADS / 32];
  __shared__ int last;
  unsigned long long cnt = 0;
  for (int c0 = 0; c0 < D; c0 += DS_CHUNK) {
    double sum[DS_CHUNK], msum[DS_CHUNK];
    float mn[DS_CHUNK], mx[DS_CHUNK], mmn[DS_CHUNK], mmx[DS_CHUNK];
#pragma unroll
    for (int k = 0; k < DS_CHUNK; ++k) {
      sum[k] = msum[k] = 0.0;
      mn[k] = mmn[k] = INFINITY; mx[k] = mmx[k] = -INFINITY;
    }
    // DS_UNROLL pixels per trip: all their loads are issued before any is used, so more bytes are in flight
    for (int64_t pb = p0 + threadIdx.x; pb < p1; pb += DS_THREADS * DS_UNROLL) {
      float x[DS_UNROLL][DS_CHUNK];
      bool in[DS_UNROLL];
#pragma unroll
      for (int r = 0; r < DS_UNROLL; ++r) {
        const int64_t p = pb + r * DS_THREADS;
        in[r] = false;
        if (p < p1) {
          const int pi = (int)p;                  // H*W < 2^31
          in[r] = mk[pi] != MaskT(0);
          // pixel-dense layouts (NCHW, NHWC) skip the division by W
          const int64_t off = dense ? (int64_t)pi * im.sw : (int64_t)(pi / W) * im.sh + (int64_t)(pi % W) * im.sw;
          const float* px = img + off + (int64_t)c0 * im.sc;
#pragma unroll
          for (int k = 0; k < DS_CHUNK; ++k) x[r][k] = c0 + k < D ? __ldg(px + k * im.sc) : 0.f;
        }
      }
#pragma unroll
      for (int r = 0; r < DS_UNROLL; ++r) {
        if (pb + r * DS_THREADS >= p1) break;
        if (c0 == 0) cnt += in[r];
#pragma unroll
        for (int k = 0; k < DS_CHUNK; ++k) {
          if (c0 + k >= D) break;
          const float v = x[r][k];
          sum[k] = __dadd_rn(sum[k], (double)v);
          mn[k] = ds_min(mn[k], v); mx[k] = ds_max(mx[k], v);
          if (in[r]) {
            msum[k] = __dadd_rn(msum[k], (double)v);
            mmn[k] = ds_min(mmn[k], v); mmx[k] = ds_max(mmx[k], v);
          }
        }
      }
    }
#pragma unroll
    for (int k = 0; k < DS_CHUNK; ++k) {
      if (c0 + k >= D) break;       // uniform across the block
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        sum[k] = __dadd_rn(sum[k], __shfl_xor_sync(0xffffffffu, sum[k], o));
        msum[k] = __dadd_rn(msum[k], __shfl_xor_sync(0xffffffffu, msum[k], o));
        mn[k] = ds_min(mn[k], __shfl_xor_sync(0xffffffffu, mn[k], o));
        mx[k] = ds_max(mx[k], __shfl_xor_sync(0xffffffffu, mx[k], o));
        mmn[k] = ds_min(mmn[k], __shfl_xor_sync(0xffffffffu, mmn[k], o));
        mmx[k] = ds_max(mmx[k], __shfl_xor_sync(0xffffffffu, mmx[k], o));
      }
      if (lane == 0) {
        r_sum[warp][k] = sum[k]; r_msum[warp][k] = msum[k];
        r_mn[warp][k] = mn[k]; r_mx[warp][k] = mx[k]; r_mmn[warp][k] = mmn[k]; r_mmx[warp][k] = mmx[k];
      }
    }
    if (c0 == 0) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
      if (lane == 0) r_cnt[warp] = cnt;
    }
    __syncthreads();
    if (threadIdx.x < DS_CHUNK && c0 + (int)threadIdx.x < D) {
      const int k = threadIdx.x;
      double a = r_sum[0][k], b = r_msum[0][k];
      float lo = r_mn[0][k], hi = r_mx[0][k], mlo = r_mmn[0][k], mhi = r_mmx[0][k];
      for (int w = 1; w < DS_THREADS / 32; ++w) {
        a = __dadd_rn(a, r_sum[w][k]); b = __dadd_rn(b, r_msum[w][k]);
        lo = ds_min(lo, r_mn[w][k]); hi = ds_max(hi, r_mx[w][k]); mlo = ds_min(mlo, r_mmn[w][k]); mhi = ds_max(mhi, r_mmx[w][k]);
      }
      const int64_t i = ((int64_t)n * nbx + blockIdx.x) * D + c0 + k;
      s.sum[i] = a; s.msum[i] = b; s.mn[i] = lo; s.mx[i] = hi; s.mmn[i] = mlo; s.mmx[i] = mhi;
    }
    if (c0 == 0 && threadIdx.x == 0) {
      unsigned long long c = 0;
      for (int w = 0; w < DS_THREADS / 32; ++w) c += r_cnt[w];
      s.cnt[(int64_t)n * nbx + blockIdx.x] = c;
    }
    __syncthreads();              // the shared records are reused by the next chunk
  }

  if (!bn_last_cta(s.ticket + n, nbx, threadIdx.x == 0, &last, [] { __syncthreads(); })) return;
  unsigned long long count = 0;
  for (int b = 0; b < nbx; ++b) count += __ldcg(s.cnt + (int64_t)n * nbx + b);
  if (threadIdx.x == 0) out_count[n] = (int64_t)count;
  for (int c = threadIdx.x; c < D; c += DS_THREADS) {
    int64_t i = (int64_t)n * nbx * D + c;
    double a = __ldcg(s.sum + i), b = __ldcg(s.msum + i);
    float lo = __ldcg(s.mn + i), hi = __ldcg(s.mx + i), mlo = __ldcg(s.mmn + i), mhi = __ldcg(s.mmx + i);
    for (int bx = 1; bx < nbx; ++bx) {
      i += D;
      a = __dadd_rn(a, __ldcg(s.sum + i)); b = __dadd_rn(b, __ldcg(s.msum + i));
      lo = ds_min(lo, __ldcg(s.mn + i)); hi = ds_max(hi, __ldcg(s.mx + i));
      mlo = ds_min(mlo, __ldcg(s.mmn + i)); mhi = ds_max(mhi, __ldcg(s.mmx + i));
    }
    float* o = out + (int64_t)n * DDN_DS_NSTATS * D + c;
    o[DDN_DS_MIN * D] = lo;
    o[DDN_DS_MAX * D] = hi;
    o[DDN_DS_MEAN * D] = (float)__ddiv_rn(a, (double)P);
    o[DDN_DS_MASK_MIN * D] = count ? mlo : NAN;
    o[DDN_DS_MASK_MAX * D] = count ? mhi : NAN;
    o[DDN_DS_MASK_MEAN * D] = count ? (float)__ddiv_rn(b, (double)count) : NAN;
  }
}

// The pixel split depends on H*W alone, so the scratch size needs no device query.
static int ds_blocks_x(int64_t P, int* ppb) {
  const int nb = (int)std::min<int64_t>(64, std::max<int64_t>(1, ceil_div(P, 8192)));
  *ppb = (int)(ceil_div(ceil_div(P, nb), DS_THREADS) * DS_THREADS);
  return (int)ceil_div(P, *ppb);
}

static size_t ds_layout(int N, int64_t P, int D, DsScratch* s, char* base) {
  int ppb;
  const size_t rec = (size_t)N * ds_blocks_x(P, &ppb) * D;
  size_t off = 0;
  auto take = [&](size_t bytes) { char* p = base ? base + off : nullptr; off += align_up(bytes, 256); return p; };
  s->ticket = reinterpret_cast<unsigned int*>(take(sizeof(unsigned int) * (size_t)N));
  s->sum = reinterpret_cast<double*>(take(sizeof(double) * rec));
  s->msum = reinterpret_cast<double*>(take(sizeof(double) * rec));
  s->cnt = reinterpret_cast<unsigned long long*>(take(sizeof(unsigned long long) * rec / D));
  s->mn = reinterpret_cast<float*>(take(sizeof(float) * rec));
  s->mx = reinterpret_cast<float*>(take(sizeof(float) * rec));
  s->mmn = reinterpret_cast<float*>(take(sizeof(float) * rec));
  s->mmx = reinterpret_cast<float*>(take(sizeof(float) * rec));
  return off;
}

}  // namespace ddn

using namespace ddn;

static bool ds_sizes_ok(int N, int H, int W, int D) {
  return N >= 1 && N <= DDN_DS_MAX_IMAGES && H >= 1 && W >= 1 && (int64_t)H * W < (1ll << 31) && D >= 1 && D <= DS_MAXD;
}

extern "C" size_t ddn_descriptor_statistics_scratch_bytes(int N, int H, int W, int D) {
  if (!ds_sizes_ok(N, H, W, D)) {
    set_error("ddn_descriptor_statistics_scratch_bytes: bad sizes (N %d, H %d, W %d, D %d)", N, H, W, D);
    return 0;
  }
  DsScratch s;
  return ds_layout(N, (int64_t)H * W, D, &s, nullptr);
}

extern "C" int ddn_descriptor_statistics(const float* res, const int64_t* strides_host, int N, int H, int W, int D,
                                         const void* mask, int mask_dtype, float* out_stats, int64_t* out_count, void* scratch,
                                         size_t scratch_bytes, void* stream) {
  DDN_CHECK_ARG(res && strides_host && mask && out_stats && out_count && scratch, "ddn_descriptor_statistics: null argument");
  DDN_CHECK_ARG(D >= 1 && D <= DS_MAXD, "ddn_descriptor_statistics: descriptor dimension %d outside 1..%d", D, DS_MAXD);
  DDN_CHECK_ARG(ds_sizes_ok(N, H, W, D), "ddn_descriptor_statistics: bad sizes (N %d in 1..%d, H %d, W %d, H*W < 2^31)", N,
                DDN_DS_MAX_IMAGES, H, W);
  DDN_CHECK_ARG(mask_dtype == DDN_DS_MASK_F32 || mask_dtype == DDN_DS_MASK_U8, "ddn_descriptor_statistics: mask dtype %d",
                mask_dtype);
  const int64_t ext[4] = {N, H, W, D};
  int64_t last = 0;
  for (int i = 0; i < 4; ++i) {
    DDN_CHECK_ARG(strides_host[i] >= 0 && strides_host[i] < (1ll << 40), "ddn_descriptor_statistics: stride %lld out of range",
                  (long long)strides_host[i]);
    last += (ext[i] - 1) * strides_host[i];
  }
  DDN_CHECK_ARG(last < (1ll << 40), "ddn_descriptor_statistics: strides address more than 2^40 elements");
  const int64_t P = (int64_t)H * W;
  DsScratch s;
  const size_t need = ds_layout(N, P, D, &s, reinterpret_cast<char*>(scratch));
  DDN_CHECK_ARG(scratch_bytes >= need, "ddn_descriptor_statistics: scratch %zu < %zu bytes", scratch_bytes, need);
  cudaStream_t st = (cudaStream_t)stream;
  DDN_CUDA(cudaMemsetAsync(s.ticket, 0, sizeof(unsigned int) * (size_t)N, st));
  const DsImage im{res, strides_host[0], strides_host[1], strides_host[2], strides_host[3]};
  int ppb;
  const int nb = ds_blocks_x(P, &ppb);
  const dim3 grid(nb, N);
  if (mask_dtype == DDN_DS_MASK_F32)
    DDN_LAUNCH(descriptor_stats_kernel<float>, grid, DS_THREADS, 0, st, im, reinterpret_cast<const float*>(mask), H, W, D, ppb, s,
               out_stats, out_count);
  else
    DDN_LAUNCH(descriptor_stats_kernel<uint8_t>, grid, DS_THREADS, 0, st, im, reinterpret_cast<const uint8_t*>(mask), H, W, D,
               ppb, s, out_stats, out_count);
  return 0;
}
