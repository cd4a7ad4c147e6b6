// Input layout change, the 1x1 scoring layer (fc), and the 8x bilinear upsample, forward and backward.
//   fc       = nn.Conv2d(512, D, 1) with bias (Resnet34_8s)   PSD/pytorch_segmentation_detection/models/resnet_dilated.py:298
//              nn.Conv2d(2048, D, 1) with bias (Resnet50_8s)  resnet_dilated.py:414
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

// NQ (1 or 2) consecutive quads of features, the 4*NQ features from 4*NQ*i on: fp32, or reconstructed from the bf16 operand
// planes (feat = hi + lo) when feat == nullptr, with one 8*NQ-byte load per plane
template <int NQ>
__device__ __forceinline__ void load_feat4(const float* feat, const __nv_bfloat16* hi, const __nv_bfloat16* lo, int64_t i, float4 (&v)[NQ]) {
  static_assert(NQ == 1 || NQ == 2, "one or two quads per load");
  if (feat) {
#pragma unroll
    for (int q = 0; q < NQ; ++q) v[q] = __ldg(reinterpret_cast<const float4*>(feat) + i * NQ + q);
    return;
  }
  // both planes are loaded before either is converted (a missing lo plane adds 0); bf16 -> fp32 is a 16-bit shift
  uint32_t hw[2 * NQ], lw[2 * NQ];
  if constexpr (NQ == 1) {
    const uint2 h = __ldg(reinterpret_cast<const uint2*>(hi) + i), l = lo ? __ldg(reinterpret_cast<const uint2*>(lo) + i) : make_uint2(0u, 0u);
    hw[0] = h.x; hw[1] = h.y; lw[0] = l.x; lw[1] = l.y;
  } else {
    const uint4 h = __ldg(reinterpret_cast<const uint4*>(hi) + i), l = lo ? __ldg(reinterpret_cast<const uint4*>(lo) + i) : make_uint4(0u, 0u, 0u, 0u);
    hw[0] = h.x; hw[1] = h.y; hw[2] = h.z; hw[3] = h.w; lw[0] = l.x; lw[1] = l.y; lw[2] = l.z; lw[3] = l.w;
  }
#pragma unroll
  for (int q = 0; q < NQ; ++q)
    v[q] = make_float4(__uint_as_float(hw[2 * q] << 16) + __uint_as_float(lw[2 * q] << 16),
                       __uint_as_float(hw[2 * q] & 0xffff0000u) + __uint_as_float(lw[2 * q] & 0xffff0000u),
                       __uint_as_float(hw[2 * q + 1] << 16) + __uint_as_float(lw[2 * q + 1] << 16),
                       __uint_as_float(hw[2 * q + 1] & 0xffff0000u) + __uint_as_float(lw[2 * q + 1] & 0xffff0000u));
}

// [D][C] fp32 weights do not fit in shared memory for the 2048-channel trunk (256 KB at D = 32), so the forward and the data
// gradient stage the weights of one FC_CHUNK-channel chunk at a time.
constexpr int FC_CHUNK = 512;
constexpr int FC_TILE = 32;             // pixels per forward tile: 8 warps x 4 pixels

// low[n][d][p] = bias[d] + sum_c feat[n][p][c] * w[d][c]: per tile of FC_TILE pixels, the chunk's weights are staged in shared memory
// and every warp adds the chunk's dot products of its pixels to the tile's accumulators (fixed chunk order: deterministic)
template <int DM>
__global__ void __launch_bounds__(256)
fc_forward_kernel(const float* __restrict__ feat, const __nv_bfloat16* __restrict__ feat_hi, const __nv_bfloat16* __restrict__ feat_lo,
                  const float* __restrict__ w, const float* __restrict__ bias,
                  float* __restrict__ low, float* __restrict__ low_t, int64_t Mimg, int N, int C, int D) {
  pdl_prologue();
  extern __shared__ float sm[];           // [D][FC_CHUNK] weights, then [FC_TILE][D] accumulators
  float* ws = sm;
  float* acc_s = sm + D * FC_CHUNK;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t total = (int64_t)N * Mimg;
  const int64_t n_tiles = (total + FC_TILE - 1) / FC_TILE;
  const int q = C >> 2;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t pix0 = tile * FC_TILE;
    for (int c0 = 0; c0 < C; c0 += FC_CHUNK) {
      __syncthreads();                    // the previous chunk's weights and the previous tile's accumulators are no longer read
      if (C > FC_CHUNK || tile == blockIdx.x) {   // a single chunk's weights stay resident for all tiles of the block
        for (int i = threadIdx.x; i < D * FC_CHUNK; i += blockDim.x) {
          const int d = i / FC_CHUNK, j = i - d * FC_CHUNK;
          ws[i] = w[(size_t)d * C + c0 + j];
        }
        __syncthreads();
      }
      for (int pl = warp; pl < FC_TILE; pl += 8) {
        const int64_t pix = pix0 + pl;
        if (pix >= total) break;
        float acc[DM];
#pragma unroll
        for (int d = 0; d < DM; ++d) acc[d] = 0.f;
        for (int c4 = lane; c4 < FC_CHUNK / 4; c4 += 32) {
          float4 v[1];
          load_feat4(feat, feat_hi, feat_lo, pix * q + (c0 >> 2) + c4, v);
#pragma unroll
          for (int d = 0; d < DM; ++d) {
            if (d < D) {
              const float4 wv = *reinterpret_cast<const float4*>(ws + d * FC_CHUNK + (c4 << 2));
              acc[d] = fmaf(v[0].x, wv.x, fmaf(v[0].y, wv.y, fmaf(v[0].z, wv.z, fmaf(v[0].w, wv.w, acc[d]))));
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
    for (int i = threadIdx.x; i < FC_TILE * D; i += blockDim.x) {
      const int pl = i / D, d = i - pl * D;
      const int64_t pix = pix0 + pl;
      if (pix >= total) continue;
      const int64_t n = pix / Mimg, p = pix - n * Mimg;
      const float v = acc_s[i] + bias[d];
      low[(n * D + d) * Mimg + p] = v;
      if (low_t) low_t[pix * D + d] = v;    // NHWC copy for the loss fused with the upsample (loss_lowres.cu)
    }
  }
}

// dfeat[n][p][c] = sum_d dlow[n][d][p] * w[d][c]; blockIdx.y = channel chunk, its [D][FC_CHUNK] weights in shared memory
template <int DM>
__global__ void __launch_bounds__(256)
fc_dgrad_kernel(const float* __restrict__ dlow, const float* __restrict__ w, float* __restrict__ dfeat, int64_t Mimg, int N, int C, int D) {
  pdl_prologue();
  extern __shared__ float ws[];
  const int c0 = blockIdx.y * FC_CHUNK;
  for (int i = threadIdx.x; i < D * FC_CHUNK; i += blockDim.x) {
    const int d = i / FC_CHUNK, j = i - d * FC_CHUNK;
    ws[i] = w[(size_t)d * C + c0 + j];
  }
  __syncthreads();
  constexpr int QC = FC_CHUNK / 4;
  const int64_t total = (int64_t)N * Mimg * QC;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int cl = (int)(i % QC) << 2; const int64_t pix = i / QC;
    const int64_t n = pix / Mimg, p = pix - n * Mimg;
    float4 a = make_float4(0, 0, 0, 0);
#pragma unroll
    for (int d = 0; d < DM; ++d) {
      if (d < D) {
        const float g = __ldg(dlow + (n * D + d) * Mimg + p);
        const float4 wv = *reinterpret_cast<const float4*>(ws + d * FC_CHUNK + cl);
        a.x = fmaf(g, wv.x, a.x); a.y = fmaf(g, wv.y, a.y); a.z = fmaf(g, wv.z, a.z); a.w = fmaf(g, wv.w, a.w);
      }
    }
    reinterpret_cast<float4*>(dfeat + pix * C + c0)[cl >> 2] = a;
  }
}

// dw[d][c] = sum_{n,p} dlow[n][d][p]*feat[n][p][c];  dbias[d] = sum dlow.  blockIdx.x = pixel slot (a contiguous pixel range),
// blockIdx.y = chunk of 64 x 4*NQ channels.  Thread = 4*NQ consecutive channels x one of 4 pixel rows: row rr takes the pixels
// p0 + rr, p0 + rr + 4, ... of the slot in increasing order, two at a time so that both loads are in flight.  NQ = 2 (8 channels,
// one 16-byte load per plane and pixel) while DM <= 8; with more descriptor channels the accumulators need NQ = 1 not to spill.
// The rows are folded through shared memory in a fixed order and the block writes its chunk of slot blockIdx.x (chunk 0 also the
// bias sums); fc_part_reduce_kernel adds the slots in slot order, so the gradient is the same on every run (no float atomics).
// The launch bounds hold DM = 4 at 3 resident blocks per SM and DM = 8 at 2 without spilling.
template <int DM, int NQ>
__global__ void __launch_bounds__(256, DM <= 4 ? 3 : DM <= 8 ? 2 : 1)
fc_wgrad_kernel(const float* __restrict__ dlow, const float* __restrict__ feat, const __nv_bfloat16* __restrict__ feat_hi,
                const __nv_bfloat16* __restrict__ feat_lo, float* __restrict__ part, int64_t Mimg, int N, int C, int D, int pix_per_slot) {
  pdl_prologue();
  constexpr int CH = 4 * NQ;              // channels per thread
  const int64_t total = (int64_t)N * Mimg;
  const int64_t p0 = (int64_t)blockIdx.x * pix_per_slot;
  const int64_t p1 = min(total, p0 + pix_per_slot);
  const int cq = threadIdx.x & 63, rr = threadIdx.x >> 6;
  const int cg = blockIdx.y * 64 + cq;    // the thread's group of CH channels
  const int c = cg * CH;
  const bool sums_bias = cq == 0 && blockIdx.y == 0;
  float acc[CH][DM];
  float bsum[DM];
#pragma unroll
  for (int d = 0; d < DM; ++d) {
    bsum[d] = 0.f;
#pragma unroll
    for (int j = 0; j < CH; ++j) acc[j][d] = 0.f;
  }
  auto fma_pixel = [&](const float4 (&f)[NQ], const float (&g)[DM]) {
#pragma unroll
    for (int q = 0; q < NQ; ++q)
#pragma unroll
      for (int d = 0; d < DM; ++d) {
        acc[4 * q][d] = fmaf(g[d], f[q].x, acc[4 * q][d]); acc[4 * q + 1][d] = fmaf(g[d], f[q].y, acc[4 * q + 1][d]);
        acc[4 * q + 2][d] = fmaf(g[d], f[q].z, acc[4 * q + 2][d]); acc[4 * q + 3][d] = fmaf(g[d], f[q].w, acc[4 * q + 3][d]);
      }
  };
  for (int64_t pa = p0 + rr; pa < p1; pa += 8) {
    const int64_t pb = pa + 4;
    const bool hb = pb < p1;              // a missing second pixel adds 0 * 0
    float4 fa[NQ], fb[NQ];
    load_feat4(feat, feat_hi, feat_lo, pa * (C / CH) + cg, fa);
    load_feat4(feat, feat_hi, feat_lo, (hb ? pb : pa) * (C / CH) + cg, fb);   // no branch between the loads
#pragma unroll
    for (int q = 0; q < NQ; ++q)
      if (!hb) fb[q] = make_float4(0.f, 0.f, 0.f, 0.f);
    float ga[DM], gb[DM];
    const int64_t na = pa / Mimg, qa = pa - na * Mimg, nb = hb ? pb / Mimg : 0, qb = hb ? pb - nb * Mimg : 0;
#pragma unroll
    for (int d = 0; d < DM; ++d) {
      ga[d] = d < D ? __ldg(dlow + (na * D + d) * Mimg + qa) : 0.f;
      gb[d] = (hb && d < D) ? __ldg(dlow + (nb * D + d) * Mimg + qb) : 0.f;
    }
    fma_pixel(fa, ga);
    fma_pixel(fb, gb);
    if (sums_bias) {
#pragma unroll
      for (int d = 0; d < DM; ++d) bsum[d] += ga[d] + gb[d];
    }
  }
  __shared__ float s_acc[DM][64 * CH];
  __shared__ float s_b[4][DM];
  if (sums_bias) {
#pragma unroll
    for (int d = 0; d < DM; ++d) s_b[rr][d] = bsum[d];
  }
  for (int r = 1; r < 4; ++r) {
    if (rr == r) {
#pragma unroll
      for (int j = 0; j < CH; ++j)
#pragma unroll
        for (int d = 0; d < DM; ++d) s_acc[d][cq * CH + j] = acc[j][d];
    }
    __syncthreads();
    if (rr == 0) {
#pragma unroll
      for (int j = 0; j < CH; ++j)
#pragma unroll
        for (int d = 0; d < DM; ++d) acc[j][d] += s_acc[d][cq * CH + j];
    }
    __syncthreads();
  }
  if (rr == 0) {
    float* slot = part + (size_t)blockIdx.x * (D * C + D);
#pragma unroll
    for (int j = 0; j < CH; ++j)
#pragma unroll
      for (int d = 0; d < DM; ++d)
        if (d < D) slot[d * C + c + j] = acc[j][d];
    if (sums_bias) {
#pragma unroll
      for (int d = 0; d < DM; ++d)
        if (d < D) slot[D * C + d] = s_b[0][d] + s_b[1][d] + s_b[2][d] + s_b[3][d];
    }
  }
}

// dw / dbias = the sum of the per-slot partials of fc_wgrad_kernel, in slot order (fp64)
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

// ---- unit-length descriptors (the reference's `normalize` option, dense_correspondence_network.py:256-259, per pixel): the
// bilinear blend x of all D maps of one output pixel, then y = x / ||x||.  One thread per output pixel; consecutive threads are
// consecutive columns, so every channel's loads and stores are coalesced.  The blend is upsample_fwd_kernel's arithmetic.  A
// zero blend gives NaN, as x / ||x|| does in fp32 (no epsilon).
template <int DM>
__device__ __forceinline__ float unit_blend(const float* __restrict__ x, int64_t n, int D, int h, int w, int oh, int ow, float sh, float sw,
                                            float (&v)[DM]) {
  int h0, h1, w0, w1; float lh, lw;
  src_index(sh, oh, h, h0, h1, lh);
  src_index(sw, ow, w, w0, w1, lw);
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < DM; ++c) {
    v[c] = 0.f;
    if (c < D) {
      const float* m = x + (n * D + c) * h * w;
      float top = (1.f - lw) * __ldg(m + h0 * w + w0) + lw * __ldg(m + h0 * w + w1);
      float bot = (1.f - lw) * __ldg(m + h1 * w + w0) + lw * __ldg(m + h1 * w + w1);
      v[c] = (1.f - lh) * top + lh * bot;
      s = fmaf(v[c], v[c], s);
    }
  }
  return sqrtf(s);
}

template <int DM>
__global__ void __launch_bounds__(256)
upsample_unit_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, int N, int D, int h, int w, int H, int W, float sh, float sw) {
  pdl_prologue();
  const int64_t HW = (int64_t)H * W, total = (int64_t)N * HW;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t n = i / HW, p = i - n * HW;
    const int oh = (int)(p / W), ow = (int)(p - (int64_t)oh * W);
    float v[DM];
    const float nrm = unit_blend<DM>(x, n, D, h, w, oh, ow, sh, sw, v);
#pragma unroll
    for (int c = 0; c < DM; ++c)
      if (c < D) y[(n * D + c) * HW + p] = v[c] / nrm;
  }
}

// g = (dy - y (y.dy)) / ||x||: the full-resolution cotangent through the normalisation (x recomputed from the low-resolution
// maps); upsample_bwd_kernel then takes g to the low-resolution maps
template <int DM>
__global__ void __launch_bounds__(256)
unit_vjp_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ g, int N, int D, int h, int w, int H, int W,
                float sh, float sw) {
  pdl_prologue();
  const int64_t HW = (int64_t)H * W, total = (int64_t)N * HW;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t n = i / HW, p = i - n * HW;
    const int oh = (int)(p / W), ow = (int)(p - (int64_t)oh * W);
    float v[DM], d[DM];
    const float nrm = unit_blend<DM>(x, n, D, h, w, oh, ow, sh, sw, v);
    float t = 0.f;
#pragma unroll
    for (int c = 0; c < DM; ++c) {
      d[c] = 0.f;
      if (c < D) {
        d[c] = __ldg(dy + (n * D + c) * HW + p);
        v[c] = v[c] / nrm;
        t = fmaf(v[c], d[c], t);
      }
    }
#pragma unroll
    for (int c = 0; c < DM; ++c)
      if (c < D) g[(n * D + c) * HW + p] = (d[c] - v[c] * t) / nrm;
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

// The weight gradient's pixel slots, each with its own D*C + D floats of `part`: up to 512 slots of at least 16 pixels for the
// 512-channel trunk, 64 for the 2048-channel one, whose slots are 4x longer.
struct FcSlots { int max_slots, min_pixels; };
static FcSlots fc_slots(int C) { return C <= 512 ? FcSlots{512, 16} : FcSlots{64, 1}; }

size_t fc_part_floats(int C, int D) { return (size_t)fc_slots(C).max_slots * (D * C + D); }

// the kernels index one slot of `part` (D*C + D floats) with int
static bool fc_shape_ok(int C, int D) {
  return D >= 1 && D <= FC_MAXD && C > 0 && C % FC_CHUNK == 0 && (int64_t)D * C + D <= INT32_MAX;
}

static int check_fc(const float* feat, const __nv_bfloat16* feat_hi, int C, int D) {
  DDN_CHECK_ARG(feat || feat_hi, "fc: no feature tensor");
  DDN_CHECK_ARG(fc_shape_ok(C, D), "fc: need 1<=D<=32 and C a multiple of %d (got C=%d D=%d)", FC_CHUNK, C, D);
  return 0;
}

int launch_fc_forward(const float* feat, const __nv_bfloat16* feat_hi, const __nv_bfloat16* feat_lo, const float* w, const float* bias,
                      float* low, float* low_nhwc, int64_t Mimg, int N, int C, int D, cudaStream_t st) {
  DDN_TRY(check_fc(feat, feat_hi, C, D));
  const size_t smem = sizeof(float) * ((size_t)D * FC_CHUNK + (size_t)FC_TILE * D);
  const int blocks = (int)std::min<int64_t>(ceil_div((int64_t)N * Mimg, FC_TILE), (int64_t)num_sms() * 8);
#define CALL(DM)                                                                                                 \
  DDN_CUDA(cudaFuncSetAttribute(fc_forward_kernel<DM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));    \
  DDN_LAUNCH(fc_forward_kernel<DM>, blocks, 256, smem, st, feat, feat_hi, feat_lo, w, bias, low, low_nhwc, Mimg, N, C, D)
  FC_DISPATCH(D, CALL);
#undef CALL
  return 0;
}

int launch_fc_backward(const float* dlow, const float* feat, const __nv_bfloat16* feat_hi, const __nv_bfloat16* feat_lo, const float* w,
                       float* dfeat, float* dw, float* dbias, float* part, int64_t Mimg, int N, int C, int D, cudaStream_t st) {
  DDN_TRY(check_fc(feat, feat_hi, C, D));
  const int64_t total = (int64_t)N * Mimg;
  const size_t smem = sizeof(float) * (size_t)D * FC_CHUNK;
  const int chunks = C / FC_CHUNK;
  dim3 dgrid((unsigned)std::max<int64_t>(1, std::min<int64_t>(ceil_div(total * (FC_CHUNK / 4), 256), (int64_t)num_sms() * 8 / chunks)),
             (unsigned)chunks);
#define CALL(DM)                                                                                               \
  DDN_CUDA(cudaFuncSetAttribute(fc_dgrad_kernel<DM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));    \
  DDN_LAUNCH(fc_dgrad_kernel<DM>, dgrid, 256, smem, st, dlow, w, dfeat, Mimg, N, C, D)
  FC_DISPATCH(D, CALL);
#undef CALL
  const FcSlots fs = fc_slots(C);
  const int pps = (int)std::max<int64_t>(fs.min_pixels, ceil_div(total, fs.max_slots));
  const int slots = (int)ceil_div(total, pps);            // <= fs.max_slots
#define CALL(DM)                                                                                                            \
  {                                                                                                                         \
    constexpr int NQ = (DM) <= 8 ? 2 : 1;                                                                                   \
    DDN_LAUNCH((fc_wgrad_kernel<DM, NQ>), dim3((unsigned)slots, (unsigned)(C / (256 * NQ))), 256, 0, st, dlow, feat, feat_hi, \
               feat_lo, part, Mimg, N, C, D, pps);                                                                          \
  }
  FC_DISPATCH(D, CALL);
#undef CALL
  const int slot_len = D * C + D;
  DDN_LAUNCH(fc_part_reduce_kernel, (int)ceil_div(slot_len, 256), 256, 0, st, part, slots, slot_len, D * C, dw, dbias);
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

int launch_upsample_unit_fwd(const float* x, float* y, int N, int D, int h, int w, int H, int W, cudaStream_t st) {
  DDN_CHECK_ARG(D >= 1 && D <= FC_MAXD, "unit upsample: need 1 <= D <= %d (got %d)", FC_MAXD, D);
  const int64_t total = (int64_t)N * H * W;
  const float sh = ac_scale(h, H), sw = ac_scale(w, W);
#define CALL(DM) DDN_LAUNCH(upsample_unit_fwd_kernel<DM>, ew_blocks(total, 256), 256, 0, st, x, y, N, D, h, w, H, W, sh, sw)
  FC_DISPATCH(D, CALL);
#undef CALL
  return 0;
}

// g (N*D*H*W floats of scratch) = the cotangent through the normalisation, then dx = upsample^T(g)
int launch_upsample_unit_bwd(const float* x, const float* dy, float* dx, float* g, int N, int D, int h, int w, int H, int W, cudaStream_t st) {
  DDN_CHECK_ARG(D >= 1 && D <= FC_MAXD, "unit upsample: need 1 <= D <= %d (got %d)", FC_MAXD, D);
  const int64_t total = (int64_t)N * H * W;
  const float sh = ac_scale(h, H), sw = ac_scale(w, W);
#define CALL(DM) DDN_LAUNCH(unit_vjp_kernel<DM>, ew_blocks(total, 256), 256, 0, st, x, dy, g, N, D, h, w, H, W, sh, sw)
  FC_DISPATCH(D, CALL);
#undef CALL
  return launch_upsample_bwd(g, dx, N * D, h, w, H, W, st);
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

static int check_unit_upsample(int N, int D, int h, int w, int H, int W) {
  DDN_CHECK_ARG(N > 0 && D >= 1 && D <= FC_MAXD && h > 0 && w > 0 && H > 0 && W > 0 && (int64_t)N * D * H * W < (1LL << 40),
                "bad unit upsample arguments (N=%d D=%d h=%d w=%d H=%d W=%d; 1 <= D <= %d)", N, D, h, w, H, W, FC_MAXD);
  return 0;
}
extern "C" int ddn_upsample_bilinear_unit_forward(const float* x, float* y, int N, int D, int h, int w, int H, int W, void* stream) {
  DDN_CHECK_ARG(x && y, "null tensor");
  DDN_TRY(check_unit_upsample(N, D, h, w, H, W));
  return launch_upsample_unit_fwd(x, y, N, D, h, w, H, W, (cudaStream_t)stream);
}
extern "C" int ddn_upsample_bilinear_unit_backward(const float* x, const float* dy, float* dx, float* scratch, int N, int D, int h, int w,
                                                   int H, int W, void* stream) {
  DDN_CHECK_ARG(x && dy && dx && scratch, "null tensor");
  DDN_TRY(check_unit_upsample(N, D, h, w, H, W));
  return launch_upsample_unit_bwd(x, dy, dx, scratch, N, D, h, w, H, W, (cudaStream_t)stream);
}

extern "C" size_t ddn_fc_workspace_bytes(int C, int D) { return fc_shape_ok(C, D) ? sizeof(float) * fc_part_floats(C, D) : 0; }

static bool aligned16(const void* p) { return ((uintptr_t)p & 15u) == 0; }

// the checks both fc entries share: one feature source, the shape, and 16-byte alignment of what the kernels read as float4 /
// uint4 (every row of C channels then starts aligned, since C is a multiple of FC_CHUNK)
static int check_fc_entry(const float* feat, const void* feat_hi, const void* feat_lo, int64_t Mimg, int N, int C, int D) {
  DDN_CHECK_ARG(!feat != !feat_hi, "fc: exactly one feature source: feat, or the bf16 planes feat_hi (+ feat_lo)");
  DDN_CHECK_ARG(feat_hi || !feat_lo, "fc: feat_lo is the low plane of feat_hi");
  DDN_CHECK_ARG(Mimg >= 1 && N >= 1, "fc: need N >= 1 and Mimg >= 1 (got N=%d Mimg=%lld)", N, (long long)Mimg);
  DDN_CHECK_ARG(fc_shape_ok(C, D), "fc: need 1<=D<=32 and C a multiple of %d (got C=%d D=%d)", FC_CHUNK, C, D);
  DDN_CHECK_ARG(aligned16(feat) && aligned16(feat_hi) && aligned16(feat_lo), "fc: the feature tensors must be 16-byte aligned");
  return 0;
}

extern "C" int ddn_fc_forward(const float* feat, const void* feat_hi, const void* feat_lo, const float* w, const float* bias, float* low,
                              float* low_nhwc, int64_t Mimg, int N, int C, int D, void* stream) {
  DDN_CHECK_ARG(w && bias && low, "null tensor");
  DDN_TRY(check_fc_entry(feat, feat_hi, feat_lo, Mimg, N, C, D));
  return launch_fc_forward(feat, (const __nv_bfloat16*)feat_hi, (const __nv_bfloat16*)feat_lo, w, bias, low, low_nhwc, Mimg, N, C, D,
                           (cudaStream_t)stream);
}

extern "C" int ddn_fc_backward(const float* dlow, const float* feat, const void* feat_hi, const void* feat_lo, const float* w, float* dfeat,
                               float* dw, float* dbias, int64_t Mimg, int N, int C, int D, void* workspace, size_t workspace_bytes,
                               void* stream) {
  DDN_CHECK_ARG(dlow && w && dfeat && dw && dbias && workspace, "null tensor");
  DDN_TRY(check_fc_entry(feat, feat_hi, feat_lo, Mimg, N, C, D));
  DDN_CHECK_ARG(aligned16(dfeat), "fc: dfeat must be 16-byte aligned");
  DDN_CHECK_ARG(((uintptr_t)workspace & 3u) == 0 && workspace_bytes >= ddn_fc_workspace_bytes(C, D), "fc: workspace too small or misaligned");
  return launch_fc_backward(dlow, feat, (const __nv_bfloat16*)feat_hi, (const __nv_bfloat16*)feat_lo, w, dfeat, dw, dbias, (float*)workspace,
                            Mimg, N, C, D, (cudaStream_t)stream);
}
