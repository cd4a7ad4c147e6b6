// Input layout change, the 1x1 scoring layer (fc), and the 8x bilinear upsample, forward and backward.
//   fc       = nn.Conv2d(512, D, 1) with bias   PSD/pytorch_segmentation_detection/models/resnet_dilated.py:298
//   upsample = nn.functional.upsample_bilinear(size=input_spatial_dim) == align_corners=True   resnet_dilated.py:320
// All HBM-bound.
#include "conv.cuh"

namespace ddn {

constexpr int FC_MAXD = 32;

// x [N,3,H,W] -> y [N,H,W,4] (4th channel zero) so the stem conv can use float4 gathers
__global__ void nchw_to_nhwc4_kernel(const float* __restrict__ x, float* __restrict__ y, int N, int64_t HW) {
  pdl_prologue();
  int64_t total = (int64_t)N * HW;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t n = i / HW, p = i - n * HW;
    const float* b = x + n * 3 * HW + p;
    reinterpret_cast<float4*>(y)[i] = make_float4(__ldg(b), __ldg(b + HW), __ldg(b + 2 * HW), 0.f);
  }
}

// 4 consecutive features: fp32, or reconstructed from the bf16 operand planes (feat = hi + lo) when feat == nullptr
__device__ __forceinline__ float4 load_feat4(const float* feat, const __nv_bfloat16* hi, const __nv_bfloat16* lo, int64_t i4) {
  if (feat) return __ldg(reinterpret_cast<const float4*>(feat) + i4);
  const uint2 h = __ldg(reinterpret_cast<const uint2*>(hi) + i4);
  float4 v = make_float4(__uint_as_float(h.x << 16), __uint_as_float(h.x & 0xffff0000u), __uint_as_float(h.y << 16),
                         __uint_as_float(h.y & 0xffff0000u));
  if (lo) {
    const uint2 l = __ldg(reinterpret_cast<const uint2*>(lo) + i4);
    v.x += __uint_as_float(l.x << 16); v.y += __uint_as_float(l.x & 0xffff0000u);
    v.z += __uint_as_float(l.y << 16); v.w += __uint_as_float(l.y & 0xffff0000u);
  }
  return v;
}

// low[n][d][p] = bias[d] + sum_c feat[n][p][c] * w[d][c]; one warp per pixel, lanes split the channels
template <int DM>
__global__ void __launch_bounds__(256)
fc_forward_kernel(const float* __restrict__ feat, const __nv_bfloat16* __restrict__ feat_hi, const __nv_bfloat16* __restrict__ feat_lo,
                  const float* __restrict__ w, const float* __restrict__ bias,
                  float* __restrict__ low, float* __restrict__ low_t, int64_t Mimg, int N, int C, int D) {
  pdl_prologue();
  extern __shared__ float ws[];   // [D][C]
  for (int i = threadIdx.x; i < D * C; i += blockDim.x) ws[i] = w[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  const int64_t total = (int64_t)N * Mimg;
  for (int64_t pix = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); pix < total; pix += warps) {
    float acc[DM];
#pragma unroll
    for (int d = 0; d < DM; ++d) acc[d] = 0.f;
    for (int c4 = lane; c4 < (C >> 2); c4 += 32) {
      const float4 v = load_feat4(feat, feat_hi, feat_lo, pix * (C >> 2) + c4);
#pragma unroll
      for (int d = 0; d < DM; ++d) {
        if (d < D) {
          float4 wv = *reinterpret_cast<const float4*>(ws + d * C + (c4 << 2));
          acc[d] = fmaf(v.x, wv.x, fmaf(v.y, wv.y, fmaf(v.z, wv.z, fmaf(v.w, wv.w, acc[d]))));
        }
      }
    }
    int64_t n = pix / Mimg, p = pix - n * Mimg;
#pragma unroll
    for (int d = 0; d < DM; ++d) {
      if (d < D) {
        float s = warp_sum(acc[d]);
        if (lane == 0) {
          low[(n * D + d) * Mimg + p] = s + bias[d];
          if (low_t) low_t[pix * D + d] = s + bias[d];       // NHWC copy for the loss fused with the upsample (loss_lowres.cu)
        }
      }
    }
  }
}

// dfeat[n][p][c] = sum_d dlow[n][d][p] * w[d][c]
template <int DM>
__global__ void __launch_bounds__(256)
fc_dgrad_kernel(const float* __restrict__ dlow, const float* __restrict__ w, float* __restrict__ dfeat,
                int64_t Mimg, int N, int C, int D) {
  pdl_prologue();
  extern __shared__ float ws[];
  for (int i = threadIdx.x; i < D * C; i += blockDim.x) ws[i] = w[i];
  __syncthreads();
  const int q = C >> 2;
  const int64_t total = (int64_t)N * Mimg * q;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int c = (int)(i % q) << 2; int64_t pix = i / q;
    int64_t n = pix / Mimg, p = pix - n * Mimg;
    float4 a = make_float4(0, 0, 0, 0);
#pragma unroll
    for (int d = 0; d < DM; ++d) {
      if (d < D) {
        float g = __ldg(dlow + (n * D + d) * Mimg + p);
        float4 wv = *reinterpret_cast<const float4*>(ws + d * C + c);
        a.x = fmaf(g, wv.x, a.x); a.y = fmaf(g, wv.y, a.y); a.z = fmaf(g, wv.z, a.z); a.w = fmaf(g, wv.w, a.w);
      }
    }
    reinterpret_cast<float4*>(dfeat)[i] = a;
  }
}

// dw[d][c] = sum_{n,p} dlow[n][d][p]*feat[n][p][c];  dbias[d] = sum dlow.  Block = C threads-quads x pixel chunk; every block
// stores its partial sums in its own slot of `part` ([D*C] weights, then [D] biases) and fc_part_reduce_kernel adds the slots
// in a fixed order, so the gradient is the same on every run (no float atomics).
template <int DM>
__global__ void __launch_bounds__(256)
fc_wgrad_kernel(const float* __restrict__ dlow, const float* __restrict__ feat, const __nv_bfloat16* __restrict__ feat_hi,
                const __nv_bfloat16* __restrict__ feat_lo, float* __restrict__ part, int64_t Mimg, int N, int C, int D, int pix_per_block) {
  pdl_prologue();
  const int64_t total = (int64_t)N * Mimg;
  const int64_t p0 = (int64_t)blockIdx.x * pix_per_block;
  const int64_t p1 = min(total, p0 + pix_per_block);
  // each thread owns channels c = tid, tid+256, ... (C <= 512 -> at most 2)
  float acc[2][DM];
  float bsum[DM];
#pragma unroll
  for (int d = 0; d < DM; ++d) { acc[0][d] = acc[1][d] = 0.f; bsum[d] = 0.f; }
  for (int64_t pix = p0; pix < p1; ++pix) {
    int64_t n = pix / Mimg, p = pix - n * Mimg;
    float g[DM];
#pragma unroll
    for (int d = 0; d < DM; ++d) g[d] = d < D ? __ldg(dlow + (n * D + d) * Mimg + p) : 0.f;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      int c = threadIdx.x + k * 256;
      if (c < C) {
        float f;
        if (feat) f = __ldg(feat + pix * C + c);
        else {
          f = __bfloat162float(feat_hi[pix * C + c]);
          if (feat_lo) f += __bfloat162float(feat_lo[pix * C + c]);
        }
#pragma unroll
        for (int d = 0; d < DM; ++d) acc[k][d] = fmaf(g[d], f, acc[k][d]);
      }
    }
    if (threadIdx.x == 0) {
#pragma unroll
      for (int d = 0; d < DM; ++d) bsum[d] += g[d];
    }
  }
  float* slot = part + (size_t)blockIdx.x * (D * C + D);
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    int c = threadIdx.x + k * 256;
    if (c < C) {
#pragma unroll
      for (int d = 0; d < DM; ++d)
        if (d < D) slot[d * C + c] = acc[k][d];
    }
  }
  if (threadIdx.x == 0) {
#pragma unroll
    for (int d = 0; d < DM; ++d)
      if (d < D) slot[D * C + d] = bsum[d];
  }
}

// dw / dbias = the sum of the per-block slots of fc_wgrad_kernel / fc_wgrad_planes_kernel, in block order (fp64)
__global__ void __launch_bounds__(256)
fc_part_reduce_kernel(const float* __restrict__ part, int n_slots, int slot_len, int DC, float* __restrict__ dw, float* __restrict__ dbias) {
  pdl_prologue();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < slot_len; i += gridDim.x * blockDim.x) {
    double s = 0.0;
    for (int b = 0; b < n_slots; ++b) s += (double)__ldg(part + (size_t)b * slot_len + i);
    if (i < DC) dw[i] = (float)s;
    else dbias[i - DC] = (float)s;
  }
}

// ---- bilinear, align_corners=True.  Source coordinate = dst * (in-1)/(out-1) computed in fp32 like ATen
// (upsample_bilinear2d: area_pixel_compute_scale / source index, then h1lambda = h1r - h1).
__device__ __forceinline__ void src_index(float scale, int dst, int in_size, int& i0, int& i1, float& l1) {
  float r = scale * (float)dst;
  i0 = (int)r;
  if (i0 > in_size - 1) i0 = in_size - 1;
  i1 = i0 + ((i0 < in_size - 1) ? 1 : 0);
  l1 = r - (float)i0;
}

__global__ void __launch_bounds__(256)
upsample_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, int NC, int h, int w, int H, int W,
                    float sh, float sw) {
  pdl_prologue();
  // thread -> 4 consecutive output columns of one row of one map
  const int Wq = W >> 2;
  const int64_t total = (int64_t)NC * H * Wq;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int wq = (int)(i % Wq); int64_t t = i / Wq;
    int oh = (int)(t % H); int64_t m = t / H;
    int h0, h1; float lh;
    src_index(sh, oh, h, h0, h1, lh);
    const float* r0 = x + (m * h + h0) * w;
    const float* r1 = x + (m * h + h1) * w;
    float o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      int w0, w1; float lw;
      src_index(sw, (wq << 2) + k, w, w0, w1, lw);
      float top = (1.f - lw) * __ldg(r0 + w0) + lw * __ldg(r0 + w1);
      float bot = (1.f - lw) * __ldg(r1 + w0) + lw * __ldg(r1 + w1);
      o[k] = (1.f - lh) * top + lh * bot;
    }
    reinterpret_cast<float4*>(y)[i] = make_float4(o[0], o[1], o[2], o[3]);
  }
}

// adjoint in gather form (deterministic): each low-res cell visits the output pixels whose stencil touches it
__global__ void __launch_bounds__(256)
upsample_bwd_kernel(const float* __restrict__ dy, float* __restrict__ dx, int NC, int h, int w, int H, int W,
                    float sh, float sw, float inv_sh, float inv_sw) {
  pdl_prologue();
  const int64_t total = (int64_t)NC * h * w;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int j = (int)(i % w); int64_t t = i / w;
    int ii = (int)(t % h); int64_t m = t / h;
    int oh_lo = max(0, (int)floorf((float)(ii - 1) * inv_sh) - 1), oh_hi = min(H - 1, (int)ceilf((float)(ii + 1) * inv_sh) + 1);
    int ow_lo = max(0, (int)floorf((float)(j - 1) * inv_sw) - 1), ow_hi = min(W - 1, (int)ceilf((float)(j + 1) * inv_sw) + 1);
    float acc = 0.f;
    const float* base = dy + m * H * W;
    for (int oh = oh_lo; oh <= oh_hi; ++oh) {
      int h0, h1; float lh;
      src_index(sh, oh, h, h0, h1, lh);
      float wh = 0.f;
      if (h0 == ii) wh += 1.f - lh;
      if (h1 == ii) wh += lh;
      if (wh == 0.f) continue;
      float row = 0.f;
      for (int ow = ow_lo; ow <= ow_hi; ++ow) {
        int w0, w1; float lw;
        src_index(sw, ow, w, w0, w1, lw);
        float ww = 0.f;
        if (w0 == j) ww += 1.f - lw;
        if (w1 == j) ww += lw;
        if (ww != 0.f) row = fmaf(ww, __ldg(base + (int64_t)oh * W + ow), row);
      }
      acc = fmaf(wh, row, acc);
    }
    dx[i] = acc;
  }
}

// ------------------------------------------------------------------------------------------------
static int ew_blocks(int64_t total, int threads) { return (int)std::min<int64_t>(ceil_div(total, threads), (int64_t)num_sms() * 8); }

int launch_nchw_to_nhwc4(const float* x, float* y, int N, int H, int W, cudaStream_t st) {
  int64_t total = (int64_t)N * H * W;
  DDN_LAUNCH(nchw_to_nhwc4_kernel, ew_blocks(total, 256), 256, 0, st, x, y, N, (int64_t)H * W);
  return 0;
}

#define FC_DISPATCH(D, CALL)              \
  do {                                    \
    if ((D) <= 4) { CALL(4); }            \
    else if ((D) <= 8) { CALL(8); }       \
    else if ((D) <= 16) { CALL(16); }     \
    else { CALL(32); }                    \
  } while (0)

// Plane variant of fc_wgrad_kernel for C = 512 and D <= 8: 64 threads x 8 channels (one 16-byte load per plane and pixel) cover a
// pixel, the 4 thread groups of a block walk 4 pixels at a time and two are in flight per thread -- the scalar version above moves
// 2 bytes per load and runs at 1/7 of the HBM rate on the 157 MB feature map.
template <int DM>
__global__ void __launch_bounds__(256)
fc_wgrad_planes_kernel(const float* __restrict__ dlow, const __nv_bfloat16* __restrict__ feat_hi, const __nv_bfloat16* __restrict__ feat_lo,
                       float* __restrict__ part, int64_t Mimg, int N, int D, int pix_per_block) {
  pdl_prologue();
  constexpr int C = 512;
  const int64_t total = (int64_t)N * Mimg;
  const int64_t p0 = (int64_t)blockIdx.x * pix_per_block;
  const int64_t p1 = min(total, p0 + pix_per_block);
  const int cq = threadIdx.x & 63, rr = threadIdx.x >> 6;
  float acc[8][DM];
  float bsum[DM];
#pragma unroll
  for (int d = 0; d < DM; ++d) {
    bsum[d] = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j][d] = 0.f;
  }
  auto fma_pixel = [&](const uint4 h, const uint4 l, const float (&g)[DM]) {
    const uint32_t hw[4] = {h.x, h.y, h.z, h.w}, lw[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      // bf16 -> fp32 is a 16-bit shift; feature = hi + lo
      const float f0 = __uint_as_float(hw[j] << 16) + __uint_as_float(lw[j] << 16);
      const float f1 = __uint_as_float(hw[j] & 0xffff0000u) + __uint_as_float(lw[j] & 0xffff0000u);
#pragma unroll
      for (int d = 0; d < DM; ++d) { acc[2 * j][d] = fmaf(g[d], f0, acc[2 * j][d]); acc[2 * j + 1][d] = fmaf(g[d], f1, acc[2 * j + 1][d]); }
    }
  };
  const uint4 z = make_uint4(0u, 0u, 0u, 0u);
  for (int64_t pix = p0 + rr; pix < p1; pix += 8) {
    const int64_t pa = pix, pb = pix + 4;
    const bool hb = pb < p1;
    const uint4 ha = __ldg(reinterpret_cast<const uint4*>(feat_hi + pa * C) + cq);
    const uint4 la = feat_lo ? __ldg(reinterpret_cast<const uint4*>(feat_lo + pa * C) + cq) : z;
    const uint4 hbv = hb ? __ldg(reinterpret_cast<const uint4*>(feat_hi + pb * C) + cq) : z;
    const uint4 lbv = (hb && feat_lo) ? __ldg(reinterpret_cast<const uint4*>(feat_lo + pb * C) + cq) : z;
    float ga[DM], gb[DM];
    const int64_t na = pa / Mimg, qa = pa - na * Mimg, nb = hb ? pb / Mimg : 0, qb = hb ? pb - nb * Mimg : 0;
#pragma unroll
    for (int d = 0; d < DM; ++d) {
      ga[d] = d < D ? __ldg(dlow + (na * D + d) * Mimg + qa) : 0.f;
      gb[d] = (hb && d < D) ? __ldg(dlow + (nb * D + d) * Mimg + qb) : 0.f;
    }
    fma_pixel(ha, la, ga);
    fma_pixel(hbv, lbv, gb);
    if (cq == 0) {
#pragma unroll
      for (int d = 0; d < DM; ++d) bsum[d] += ga[d] + gb[d];
    }
  }
  // the 4 pixel groups of the block are folded through shared memory one after the other, then the block's slot is stored
  __shared__ float s_acc[DM][C];
  __shared__ float s_b[4][DM];
  if (cq == 0) {
#pragma unroll
    for (int d = 0; d < DM; ++d) s_b[rr][d] = bsum[d];
  }
  for (int r = 1; r < 4; ++r) {
    if (rr == r) {
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int d = 0; d < DM; ++d) s_acc[d][cq * 8 + j] = acc[j][d];
    }
    __syncthreads();
    if (rr == 0) {
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int d = 0; d < DM; ++d) acc[j][d] += s_acc[d][cq * 8 + j];
    }
    __syncthreads();
  }
  if (rr == 0) {
    float* slot = part + (size_t)blockIdx.x * (D * C + D);
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int d = 0; d < DM; ++d)
        if (d < D) slot[d * C + cq * 8 + j] = acc[j][d];
    if (cq == 0) {
#pragma unroll
      for (int d = 0; d < DM; ++d)
        if (d < D) slot[D * C + d] = s_b[0][d] + s_b[1][d] + s_b[2][d] + s_b[3][d];
    }
  }
}

// ---- the same three for a wide trunk (C > 512: the 2048 channels of the Bottleneck backbone).  [D][C] fp32 weights no longer
// fit in shared memory (256 KB at D = 32, C = 2048) and one partial slot of the weight gradient holds D*C floats, so every kernel
// below walks the channels in chunks of FC_WIDE_CHUNK, and the weight gradient keeps FC_WIDE_SLOTS pixel slots.
constexpr int FC_WIDE_CHUNK = 512;
constexpr int FC_WIDE_TILE = 64;        // pixels per forward tile: 8 warps x 8 pixels
constexpr int FC_WIDE_SLOTS = 64;
constexpr int FC_WIDE_WG_CH = 256;      // channels of one weight-gradient block: 64 threads x 4 channels

// low[n][d][p] = bias[d] + sum_c feat[n][p][c] * w[d][c]: per tile of 64 pixels, the chunk's weights are staged in shared memory
// and every warp adds the chunk's dot products of its pixels to the tile's accumulators (fixed chunk order: deterministic)
template <int DM>
__global__ void __launch_bounds__(256)
fc_forward_wide_kernel(const float* __restrict__ feat, const __nv_bfloat16* __restrict__ feat_hi, const __nv_bfloat16* __restrict__ feat_lo,
                       const float* __restrict__ w, const float* __restrict__ bias,
                       float* __restrict__ low, float* __restrict__ low_t, int64_t Mimg, int N, int C, int D) {
  pdl_prologue();
  extern __shared__ float sm[];           // [D][FC_WIDE_CHUNK] weights, then [FC_WIDE_TILE][D] accumulators
  float* ws = sm;
  float* acc_s = sm + D * FC_WIDE_CHUNK;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t total = (int64_t)N * Mimg;
  const int64_t n_tiles = (total + FC_WIDE_TILE - 1) / FC_WIDE_TILE;
  const int q = C >> 2;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t pix0 = tile * FC_WIDE_TILE;
    for (int c0 = 0; c0 < C; c0 += FC_WIDE_CHUNK) {
      __syncthreads();                    // the previous chunk's weights are no longer read
      for (int i = threadIdx.x; i < D * FC_WIDE_CHUNK; i += blockDim.x) {
        const int d = i / FC_WIDE_CHUNK, j = i - d * FC_WIDE_CHUNK;
        ws[i] = w[(size_t)d * C + c0 + j];
      }
      __syncthreads();
      for (int pl = warp; pl < FC_WIDE_TILE; pl += 8) {
        const int64_t pix = pix0 + pl;
        if (pix >= total) break;
        float acc[DM];
#pragma unroll
        for (int d = 0; d < DM; ++d) acc[d] = 0.f;
        for (int c4 = lane; c4 < FC_WIDE_CHUNK / 4; c4 += 32) {
          const float4 v = load_feat4(feat, feat_hi, feat_lo, pix * q + (c0 >> 2) + c4);
#pragma unroll
          for (int d = 0; d < DM; ++d) {
            if (d < D) {
              const float4 wv = *reinterpret_cast<const float4*>(ws + d * FC_WIDE_CHUNK + (c4 << 2));
              acc[d] = fmaf(v.x, wv.x, fmaf(v.y, wv.y, fmaf(v.z, wv.z, fmaf(v.w, wv.w, acc[d]))));
            }
          }
        }
#pragma unroll
        for (int d = 0; d < DM; ++d) {
          if (d < D) {
            const float t = warp_sum(acc[d]);
            if (lane == 0) acc_s[pl * D + d] = c0 == 0 ? t : acc_s[pl * D + d] + t;
          }
        }
      }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < FC_WIDE_TILE * D; i += blockDim.x) {
      const int pl = i / D, d = i - pl * D;
      const int64_t pix = pix0 + pl;
      if (pix >= total) continue;
      const int64_t n = pix / Mimg, p = pix - n * Mimg;
      const float v = acc_s[i] + bias[d];
      low[(n * D + d) * Mimg + p] = v;
      if (low_t) low_t[pix * D + d] = v;
    }
  }
}

// dfeat[n][p][c] = sum_d dlow[n][d][p] * w[d][c]; blockIdx.y = channel chunk, its [D][FC_WIDE_CHUNK] weights in shared memory
template <int DM>
__global__ void __launch_bounds__(256)
fc_dgrad_wide_kernel(const float* __restrict__ dlow, const float* __restrict__ w, float* __restrict__ dfeat, int64_t Mimg, int N, int C, int D) {
  pdl_prologue();
  extern __shared__ float ws[];
  const int c0 = blockIdx.y * FC_WIDE_CHUNK;
  for (int i = threadIdx.x; i < D * FC_WIDE_CHUNK; i += blockDim.x) {
    const int d = i / FC_WIDE_CHUNK, j = i - d * FC_WIDE_CHUNK;
    ws[i] = w[(size_t)d * C + c0 + j];
  }
  __syncthreads();
  constexpr int QC = FC_WIDE_CHUNK / 4;
  const int64_t total = (int64_t)N * Mimg * QC;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int cl = (int)(i % QC) << 2; const int64_t pix = i / QC;
    const int64_t n = pix / Mimg, p = pix - n * Mimg;
    float4 a = make_float4(0, 0, 0, 0);
#pragma unroll
    for (int d = 0; d < DM; ++d) {
      if (d < D) {
        const float g = __ldg(dlow + (n * D + d) * Mimg + p);
        const float4 wv = *reinterpret_cast<const float4*>(ws + d * FC_WIDE_CHUNK + cl);
        a.x = fmaf(g, wv.x, a.x); a.y = fmaf(g, wv.y, a.y); a.z = fmaf(g, wv.z, a.z); a.w = fmaf(g, wv.w, a.w);
      }
    }
    reinterpret_cast<float4*>(dfeat + pix * C + c0)[cl >> 2] = a;
  }
}

// dw[d][c] / dbias[d] partial sums: blockIdx.x = pixel slot (a contiguous pixel range), blockIdx.y = 256-channel chunk.  Thread =
// 4 consecutive channels (one 8-byte load per plane and pixel) x one of 4 pixel rows; the rows are folded through shared memory
// in a fixed order and the block writes its chunk of slot blockIdx.x.  fc_part_reduce_kernel adds the slots in slot order.
template <int DM>
__global__ void __launch_bounds__(256)
fc_wgrad_wide_kernel(const float* __restrict__ dlow, const float* __restrict__ feat, const __nv_bfloat16* __restrict__ feat_hi,
                     const __nv_bfloat16* __restrict__ feat_lo, float* __restrict__ part, int64_t Mimg, int N, int C, int D, int pix_per_slot) {
  pdl_prologue();
  const int64_t total = (int64_t)N * Mimg;
  const int64_t p0 = (int64_t)blockIdx.x * pix_per_slot;
  const int64_t p1 = min(total, p0 + pix_per_slot);
  const int cq = threadIdx.x & 63, rr = threadIdx.x >> 6;
  const int c = blockIdx.y * FC_WIDE_WG_CH + cq * 4;
  float acc[4][DM];
  float bsum[DM];
#pragma unroll
  for (int d = 0; d < DM; ++d) {
    bsum[d] = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[j][d] = 0.f;
  }
  for (int64_t pix = p0 + rr; pix < p1; pix += 4) {
    const float4 f = load_feat4(feat, feat_hi, feat_lo, (pix * C + c) >> 2);
    const int64_t n = pix / Mimg, p = pix - n * Mimg;
#pragma unroll
    for (int d = 0; d < DM; ++d) {
      const float g = d < D ? __ldg(dlow + (n * D + d) * Mimg + p) : 0.f;
      acc[0][d] = fmaf(g, f.x, acc[0][d]); acc[1][d] = fmaf(g, f.y, acc[1][d]);
      acc[2][d] = fmaf(g, f.z, acc[2][d]); acc[3][d] = fmaf(g, f.w, acc[3][d]);
      bsum[d] += g;
    }
  }
  __shared__ float s_acc[DM][FC_WIDE_WG_CH];
  __shared__ float s_b[4][DM];
  if (cq == 0) {
#pragma unroll
    for (int d = 0; d < DM; ++d) s_b[rr][d] = bsum[d];
  }
  for (int r = 1; r < 4; ++r) {
    if (rr == r) {
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int d = 0; d < DM; ++d) s_acc[d][cq * 4 + j] = acc[j][d];
    }
    __syncthreads();
    if (rr == 0) {
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int d = 0; d < DM; ++d) acc[j][d] += s_acc[d][cq * 4 + j];
    }
    __syncthreads();
  }
  if (rr == 0) {
    float* slot = part + (size_t)blockIdx.x * (D * C + D);
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int d = 0; d < DM; ++d)
        if (d < D) slot[d * C + c + j] = acc[j][d];
    if (cq == 0 && blockIdx.y == 0) {
#pragma unroll
      for (int d = 0; d < DM; ++d)
        if (d < D) slot[D * C + d] = s_b[0][d] + s_b[1][d] + s_b[2][d] + s_b[3][d];
    }
  }
}

size_t fc_part_floats(int C, int D) {
  return C <= 512 ? (size_t)FC_PART_SLOTS * (D * C + D) : (size_t)FC_WIDE_SLOTS * (D * C + D);
}

static int check_fc(const float* feat, const __nv_bfloat16* feat_hi, int C, int D) {
  DDN_CHECK_ARG(feat || feat_hi, "fc: no feature tensor");
  DDN_CHECK_ARG(D >= 1 && D <= FC_MAXD && C % 4 == 0 && (C <= 512 || C % FC_WIDE_CHUNK == 0),
                "fc: need 1<=D<=32 and C%%4==0 with C<=512 or C a multiple of %d (got C=%d D=%d)", FC_WIDE_CHUNK, C, D);
  return 0;
}

int launch_fc_forward(const float* feat, const __nv_bfloat16* feat_hi, const __nv_bfloat16* feat_lo, const float* w, const float* bias,
                      float* low, float* low_nhwc, int64_t Mimg, int N, int C, int D, cudaStream_t st) {
  DDN_TRY(check_fc(feat, feat_hi, C, D));
  if (C > 512) {
    const size_t smem = sizeof(float) * ((size_t)D * FC_WIDE_CHUNK + (size_t)FC_WIDE_TILE * D);
    const int blocks = (int)std::min<int64_t>(ceil_div((int64_t)N * Mimg, FC_WIDE_TILE), (int64_t)num_sms() * 4);
#define CALL(DM)                                                                                                       \
  DDN_CUDA(cudaFuncSetAttribute(fc_forward_wide_kernel<DM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));    \
  DDN_LAUNCH(fc_forward_wide_kernel<DM>, blocks, 256, smem, st, feat, feat_hi, feat_lo, w, bias, low, low_nhwc, Mimg, N, C, D)
    FC_DISPATCH(D, CALL);
#undef CALL
    return 0;
  }
  size_t smem = sizeof(float) * D * C;
  int blocks = (int)std::min<int64_t>(ceil_div((int64_t)N * Mimg, 8), (int64_t)num_sms() * 8);
#define CALL(DM)                                                                                              \
  DDN_CUDA(cudaFuncSetAttribute(fc_forward_kernel<DM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
  DDN_LAUNCH(fc_forward_kernel<DM>, blocks, 256, smem, st, feat, feat_hi, feat_lo, w, bias, low, low_nhwc, Mimg, N, C, D)
  FC_DISPATCH(D, CALL);
#undef CALL
  return 0;
}

int launch_fc_backward(const float* dlow, const float* feat, const __nv_bfloat16* feat_hi, const __nv_bfloat16* feat_lo, const float* w,
                       float* dfeat, float* dw, float* dbias, float* part, int64_t Mimg, int N, int C, int D, cudaStream_t st) {
  DDN_TRY(check_fc(feat, feat_hi, C, D));
  if (C > 512) {
    const int64_t total = (int64_t)N * Mimg;
    const size_t smem = sizeof(float) * (size_t)D * FC_WIDE_CHUNK;
    const int chunks = C / FC_WIDE_CHUNK;
    dim3 dgrid((unsigned)std::max<int64_t>(1, std::min<int64_t>(ceil_div(total * (FC_WIDE_CHUNK / 4), 256), (int64_t)num_sms() * 8 / chunks)),
               (unsigned)chunks);
#define CALL(DM)                                                                                                    \
  DDN_CUDA(cudaFuncSetAttribute(fc_dgrad_wide_kernel<DM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));   \
  DDN_LAUNCH(fc_dgrad_wide_kernel<DM>, dgrid, 256, smem, st, dlow, w, dfeat, Mimg, N, C, D)
    FC_DISPATCH(D, CALL);
#undef CALL
    const int pps = (int)ceil_div(total, FC_WIDE_SLOTS);
    const int slots = (int)ceil_div(total, pps);           // <= FC_WIDE_SLOTS
    dim3 wgrid((unsigned)slots, (unsigned)(C / FC_WIDE_WG_CH));
#define CALL(DM) DDN_LAUNCH(fc_wgrad_wide_kernel<DM>, wgrid, 256, 0, st, dlow, feat, feat_hi, feat_lo, part, Mimg, N, C, D, pps)
    FC_DISPATCH(D, CALL);
#undef CALL
    const int slot_len = D * C + D;
    DDN_LAUNCH(fc_part_reduce_kernel, (int)ceil_div(slot_len, 256), 256, 0, st, part, slots, slot_len, D * C, dw, dbias);
    return 0;
  }
  size_t smem = sizeof(float) * D * C;
  int64_t total = (int64_t)N * Mimg;
#define CALL(DM)                                                                                               \
  DDN_CUDA(cudaFuncSetAttribute(fc_dgrad_kernel<DM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));    \
  DDN_LAUNCH(fc_dgrad_kernel<DM>, ew_blocks(total * (C / 4), 256), 256, smem, st, dlow, w, dfeat, Mimg, N, C, D)
  FC_DISPATCH(D, CALL);
#undef CALL
  const int ppb = (int)std::max<int64_t>(16, ceil_div(total, FC_PART_SLOTS));
  const int blocks = (int)ceil_div(total, ppb);            // <= FC_PART_SLOTS
  if (!feat && C == 512 && D <= 8) {
    if (D <= 4) DDN_LAUNCH(fc_wgrad_planes_kernel<4>, blocks, 256, 0, st, dlow, feat_hi, feat_lo, part, Mimg, N, D, ppb);
    else DDN_LAUNCH(fc_wgrad_planes_kernel<8>, blocks, 256, 0, st, dlow, feat_hi, feat_lo, part, Mimg, N, D, ppb);
  } else {
#define CALL(DM) DDN_LAUNCH(fc_wgrad_kernel<DM>, blocks, 256, 0, st, dlow, feat, feat_hi, feat_lo, part, Mimg, N, C, D, ppb)
    FC_DISPATCH(D, CALL);
#undef CALL
  }
  const int slot_len = D * C + D;
  DDN_LAUNCH(fc_part_reduce_kernel, (int)ceil_div(slot_len, 256), 256, 0, st, part, blocks, slot_len, D * C, dw, dbias);
  return 0;
}

static float ac_scale(int in, int out) { return out > 1 ? (float)(in - 1) / (float)(out - 1) : 0.f; }

int launch_upsample_fwd(const float* x, float* y, int NC, int h, int w, int H, int W, cudaStream_t st) {
  DDN_CHECK_ARG(W % 4 == 0, "upsample: output width must be a multiple of 4");
  int64_t total = (int64_t)NC * H * (W / 4);
  DDN_LAUNCH(upsample_fwd_kernel, ew_blocks(total, 256), 256, 0, st, x, y, NC, h, w, H, W, ac_scale(h, H), ac_scale(w, W));
  return 0;
}

int launch_upsample_bwd(const float* dy, float* dx, int NC, int h, int w, int H, int W, cudaStream_t st) {
  float sh = ac_scale(h, H), sw = ac_scale(w, W);
  float ish = sh > 0 ? 1.f / sh : (float)H, isw = sw > 0 ? 1.f / sw : (float)W;
  int64_t total = (int64_t)NC * h * w;
  DDN_LAUNCH(upsample_bwd_kernel, (int)ceil_div(total, 128), 128, 0, st, dy, dx, NC, h, w, H, W, sh, sw, ish, isw);
  return 0;
}

// dlow [N, D, Mimg] (+)= dlow_t [N, Mimg, D]: the gradient the fused loss scattered into the NHWC low-resolution map
__global__ void add_lowres_nhwc_kernel(const float* __restrict__ dlow_t, float* __restrict__ dlow, int64_t Mimg, int N, int D, int accumulate) {
  pdl_prologue();
  const int64_t total = (int64_t)N * D * Mimg;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = i % Mimg; const int64_t t = i / Mimg;
    const int d = (int)(t % D); const int64_t n = t / D;
    const float v = __ldg(dlow_t + (n * Mimg + p) * D + d);
    dlow[i] = accumulate ? dlow[i] + v : v;
  }
}
int launch_add_lowres_nhwc(const float* dlow_t, float* dlow, int64_t Mimg, int N, int D, int accumulate, cudaStream_t st) {
  const int64_t total = (int64_t)N * D * Mimg;
  DDN_LAUNCH(add_lowres_nhwc_kernel, ew_blocks(total, 256), 256, 0, st, dlow_t, dlow, Mimg, N, D, accumulate);
  return 0;
}

int launch_fill_zero(void* p, size_t bytes, cudaStream_t st) {
  DDN_CUDA(cudaMemsetAsync(p, 0, bytes, st));
  return 0;
}

}  // namespace ddn

using namespace ddn;

extern "C" int ddn_upsample_bilinear_forward(const float* x, float* y, int NC, int h, int w, int H, int W, void* stream) {
  DDN_CHECK_ARG(x && y && NC > 0 && h > 0 && w > 0 && H > 0 && W > 0, "bad upsample arguments");
  return launch_upsample_fwd(x, y, NC, h, w, H, W, (cudaStream_t)stream);
}
extern "C" int ddn_upsample_bilinear_backward(const float* dy, float* dx, int NC, int h, int w, int H, int W, void* stream) {
  DDN_CHECK_ARG(dy && dx && NC > 0 && h > 0 && w > 0 && H > 0 && W > 0, "bad upsample arguments");
  return launch_upsample_bwd(dy, dx, NC, h, w, H, W, (cudaStream_t)stream);
}
