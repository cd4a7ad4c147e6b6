// wgmma implicit-GEMM convolution for sm_90a: every convolution of Resnet34_8s (3x3 dilated / strided, 1x1, and the
// 7x7 stem as a patch GEMM), forward, data-gradient and weight-gradient, on the Hopper tensor cores.
//
//   D[128 pixels x BLOCK_N channels] (fp32, registers) += A[pixels x 64 ch] (smem) * B[BLOCK_N x 64 ch]^T (smem)
//
// * Activations are NHWC bf16 planes, cut into 4x16-pixel sub-tiles.  For filter tap (r,s) and 64-channel chunk c the A
//   rows of a sub-tile are ONE 4-D TMA box load at (c, w0+(s-1)*dil, h0+(r-1)*dil, n): TMA's out-of-bounds zero fill *is*
//   the convolution padding, so there is no im2col buffer and no halo logic.
// * Weights are [Cout][tap*Cin + ci] bf16 (K-major); a [BLOCK_N x 64] box per k-block.
// * Both operands land in shared memory in the 128-byte-swizzled K-major layout wgmma reads directly.
// * Precision: DDN_PRECISION_BF16X3 keeps fp32-equivalent results by splitting every operand x = hi + lo
//   (both bf16) and issuing hi*lo + lo*hi + hi*hi into the same fp32 accumulator (3 MMAs per k-step);
//   DDN_PRECISION_BF16 issues hi*hi only.
// * Warp roles (288 threads): warps 0-7 = two consumer warpgroups -- each issues wgmma.m64nNk16 for 64 of the 128 tile rows
//   (one sub-tile) into its own register accumulator and then runs the epilogue of those rows -- and warp 8 = TMA producer.
//   smem ring of kStages {A_hi,A_lo,B_hi,B_lo} slots with full/empty mbarriers; a slot is released once the wgmma group that
//   read it has completed (wgmma.wait_group).
// * Epilogue: each warp passes its accumulator fragment through a small shared-memory staging tile, after which 8 lanes hold
//   the 32 channels of one pixel and every global access is a whole 128-byte line of NHWC memory (fused addend / BatchNorm
//   statistics / folded inference BatchNorm / BatchNorm-backward column sums).
// * Kernels in this file: conv_tc_kernel (every conv), conv64_halo_kernel / wgrad64_halo_kernel (the 64-channel layer:
//   resident weights, one halo tile per 8x16 pixels, taps read in place), wgrad_tc_kernel (weight gradient, pixels as the K
//   dimension), operand preparation (stem patches, zero insertion, weight packs + their device-side validation).
// * Every kernel starts with griddepcontrol.launch_dependents / .wait (programmatic dependent launch, common.cuh).
//
// Reference op replaced: nn.Conv2d via conv3x3 (PSD/vision/torchvision/models/resnet.py:20-37,45,48) and the
// stride-1 1x1 downsample convs (resnet.py:210-214), plus their autograd data gradient.
#include <cuda.h>
#include <algorithm>
#include <cstring>
#include <functional>
#include <mutex>
#include <unordered_map>

#include "conv.cuh"
#include "conv_tc.cuh"

namespace ddn {

constexpr int TC_BLOCK_K = 64;                // bf16 elements per k-block = one 128-byte swizzle row
constexpr int TC_CONSUMERS = 256;             // two consumer warpgroups
constexpr int TC_THREADS = TC_CONSUMERS + 32; // + the TMA producer warp
constexpr int TC_PRODUCER_WARP = TC_CONSUMERS / 32;
constexpr int TC_WIDE_THREADS = TC_CONSUMERS + 128; // + a whole producer warpgroup that hands its registers to the consumers
constexpr int TC_A_BYTES = 128 * TC_BLOCK_K * 2;   // 16 KB

// ------------------------------------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t"
      "}\n" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_prefetch_l2_4d(const CUtensorMap* map, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.prefetch.tensor.4d.L2.global.tile [%0, {%1, %2, %3, %4}];" ::"l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

// wgmma shared-memory matrix descriptor, 128-byte swizzle (PTX ISA, "Matrix Descriptor Format"; cute::GmmaDescriptor):
//   [0,14) start >> 4 | [16,30) LBO >> 4 | [32,46) SBO >> 4 | [49,52) base offset = 0 | [62,64) layout = 1 (SWIZZLE_128B)
// K-major: SBO = byte distance between 8-row core-matrix groups along M/N (LBO unused).  MN-major: LBO = distance between
// 64-element atoms along M/N, SBO = distance between 8-row groups along K.  The swizzle is a function of the shared-memory
// address bits, as TMA writes it, so a descriptor may start at any 128-byte row of a staged 1024-byte-aligned tile (base
// offset 0) -- which is what lets the halo kernels read every filter tap of one staged tile in place.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFF) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) |
         ((uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ uint64_t gmma_desc_k(uint32_t smem_addr, uint32_t sbo_bytes = 1024) { return gmma_desc(smem_addr, 16, sbo_bytes); }

template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across wgmma issue and wait points (cute warpgroup_fence_operand)
template <int K>
__device__ __forceinline__ void fence_acc(float (&d)[K]) {
#pragma unroll
  for (int i = 0; i < K; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// wgmma.mma_async m64nNk16, bf16 x bf16 -> fp32 in registers.  TRANS = 0: both operands K-major; 1: both MN-major.
// Fragment of warp w of the warpgroup: d[4j + {0,1}] = (row 16w + lane/4, columns 8j + 2(lane%4) + {0,1}), d[4j + {2,3}] =
// the same columns of row 16w + lane/4 + 8.  scale_d = 0 overwrites the accumulator.
template <int N> struct Wgmma;
template <> struct Wgmma<32> {
  template <int TRANS>
  static __device__ __forceinline__ void mma(float (&d)[16], uint64_t a, uint64_t b, int scale_d) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
        "}, %16, %17, p, 1, 1, %19, %19;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TRANS));
  }
};
template <> struct Wgmma<64> {
  template <int TRANS>
  static __device__ __forceinline__ void mma(float (&d)[32], uint64_t a, uint64_t b, int scale_d) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, %32, %33, p, 1, 1, %35, %35;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TRANS));
  }
};
template <> struct Wgmma<128> {
  template <int TRANS>
  static __device__ __forceinline__ void mma(float (&d)[64], uint64_t a, uint64_t b, int scale_d) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, %64, %65, p, 1, 1, %67, %67;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TRANS));
  }
};

// NPROD products of one k16 step into `d`: bf16x3 = hi*lo + lo*hi + hi*hi (small terms first), bf16 = hi*hi
template <int N, int TRANS, int NPROD>
__device__ __forceinline__ void mma_k16(float (&d)[N / 2], uint64_t a_hi, uint64_t a_lo, uint64_t b_hi, uint64_t b_lo, int accumulate) {
  if (NPROD == 3) {
    Wgmma<N>::template mma<TRANS>(d, a_hi, b_lo, accumulate);
    Wgmma<N>::template mma<TRANS>(d, a_lo, b_hi, 1);
    Wgmma<N>::template mma<TRANS>(d, a_hi, b_hi, 1);
  } else {
    Wgmma<N>::template mma<TRANS>(d, a_hi, b_hi, accumulate);
  }
}
// The same with the two small products in their own accumulator `x` (added to `d` once, after the last k-step).  Hopper's
// tensor cores round the fp32 accumulator at every wgmma; three instructions per k-step into one accumulator made that
// rounding -- not the bf16 split -- the largest error of a deep contraction (K = 4608: 1.5e-5 relative vs 4.4e-6 for the
// exact bf16x3 products, measured on H100).  With the cross terms 2^-8 smaller, they barely add to it here.
template <int N, int TRANS, int NPROD>
__device__ __forceinline__ void mma_k16_x(float (&d)[N / 2], float (&x)[N / 2], uint64_t a_hi, uint64_t a_lo, uint64_t b_hi, uint64_t b_lo,
                                          int accumulate) {
  if (NPROD == 3) {
    Wgmma<N>::template mma<TRANS>(x, a_hi, b_lo, accumulate);
    Wgmma<N>::template mma<TRANS>(x, a_lo, b_hi, 1);
  }
  Wgmma<N>::template mma<TRANS>(d, a_hi, b_hi, accumulate);
}
template <int K>
__device__ __forceinline__ void add_cross(float (&d)[K], const float (&x)[K]) {
#pragma unroll
  for (int i = 0; i < K; ++i) d[i] += x[i];
}
// the first N columns of a wider accumulator (fragment index 4j + x covers columns 8j .. 8j + 7)
template <int N, int K>
__device__ __forceinline__ float (&acc_cols(float (&d)[K]))[N / 2] {
  static_assert(N / 2 <= K, "accumulator too narrow");
  return *reinterpret_cast<float(*)[N / 2]>(&d[0]);
}

// ------------------------------------------------------------------------------------------------ epilogue helpers
// A warp owns 16 accumulator rows.  stage_chunk() hands lane 8a+b the rows 4a .. 4a+3 of those 16, channel quad b of the
// 32-column chunk c, through the warp's staging tile: after it the 8 lanes of a group hold the 32 channels of ONE row, so a
// 128-bit load / store per lane moves whole 128-byte lines of NHWC memory and per-channel constants are one load per lane.
constexpr int EPI_ROWS = 4;                      // rows per lane group
constexpr int EPI_STRIDE = 40;                   // floats per staging row: conflict-free float2 writes and float4 reads
constexpr int EPI_WARP_FLOATS = 16 * EPI_STRIDE;

// the warp's 16 rows x columns 32c .. 32c + 31 of the accumulator -> st[row * EPI_STRIDE + column - 32c]
template <int K>
__device__ __forceinline__ void stage_write(const float (&acc)[K], int c, float* st, int lane) {
  const int r = lane >> 2, q = (lane & 3) * 2;
#pragma unroll
  for (int jj = 0; jj < 4; ++jj) {
    const int j = 4 * c + jj;                    // compile-time once the caller's chunk loop is unrolled
    *reinterpret_cast<float2*>(st + r * EPI_STRIDE + 8 * jj + q) = make_float2(acc[4 * j], acc[4 * j + 1]);
    *reinterpret_cast<float2*>(st + (r + 8) * EPI_STRIDE + 8 * jj + q) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
  }
  __syncwarp();
}

template <int K>
__device__ __forceinline__ void stage_chunk(const float (&acc)[K], int c, float* st, int lane, float4 (&v)[EPI_ROWS]) {
  stage_write(acc, c, st, lane);
  const int ga = lane >> 3, gb = lane & 7;
#pragma unroll
  for (int i = 0; i < EPI_ROWS; ++i) v[i] = *reinterpret_cast<const float4*>(st + (EPI_ROWS * ga + i) * EPI_STRIDE + 4 * gb);
  __syncwarp();                                  // the tile is rewritten by the next chunk
}

__device__ __forceinline__ uint32_t pack_bf16x2(__nv_bfloat16 a, __nv_bfloat16 b) {
  return (uint32_t)__bfloat16_as_ushort(a) | ((uint32_t)__bfloat16_as_ushort(b) << 16);
}

// The fused epilogue request of conv_tc_kernel and conv64_halo_kernel (built and validated by tc_epilogue_request).
struct TcEpilogueParams {
  float* out;            // [N,H,W,C] fp32 (may be null with the folded epilogue)
  const float* addend;   // optional, same shape
  int imgs_per_group;    // BatchNorm group of image n = n / imgs_per_group
  BnFwdFinal fin;        // fin.a.acc == nullptr: no statistics
  TcBwdStats bst;        // bst.fin.a.acc != nullptr (data gradient): column sums of the BatchNorm backward that consumes `out`
  // optional folded epilogue (inference): y = relu?(acc * ep_scale[c] + ep_shift[c] + addend)
  const float* ep_scale; const float* ep_shift; int ep_relu;
  __nv_bfloat16* out_hi; __nv_bfloat16* out_lo;
};

// The fused epilogue of a forward / data-gradient conv for EPI_ROWS pixels x 4 channels of one lane.  v[i] = accumulator of
// pixel i; `off` = element offset of pixel 0, channel `ch` in the NHWC output (C channels per pixel), `rs` = elements between
// pixel i and i + 1; only the first n_ok pixels exist (the others are neither stored nor summed).  Variants:
//   ep_scale (inference): eval-mode BatchNorm folded in, + addend, ReLU; written as fp32 and / or the next conv's bf16 planes;
//   bst (data gradient): out = acc + addend, and (s1, s2) += (sum g, sum g * xhat), g = out * relu mask -- what
//     bn_colsum_kernel<1> computes, on the gradient this kernel just wrote;
//   otherwise (training forward): out = acc + addend, and (s1, s2) += the column sum / sum of squares of acc.
__device__ __forceinline__ void conv_epilogue_rows(const TcEpilogueParams& p, const float4 (&v)[EPI_ROWS], size_t off, size_t rs, int n_ok, int ch,
                                                   int C, int grp, float4& s1, float4& s2) {
  // the addend (residual-branch gradient) first: its global-load latency overlaps the rest
  float4 adv[EPI_ROWS];
#pragma unroll
  for (int i = 0; i < EPI_ROWS; ++i)
    adv[i] = (p.addend && i < n_ok) ? __ldg(reinterpret_cast<const float4*>(p.addend + off + i * rs)) : make_float4(0.f, 0.f, 0.f, 0.f);
  if (p.ep_scale) {        // folded BatchNorm (+ residual, ReLU): the conv output never exists un-normalised
    const float4 sc = __ldg(reinterpret_cast<const float4*>(p.ep_scale + ch));
    const float4 sh = __ldg(reinterpret_cast<const float4*>(p.ep_shift + ch));
#pragma unroll
    for (int i = 0; i < EPI_ROWS; ++i) {
      float4 f = make_float4(fmaf(v[i].x, sc.x, sh.x) + adv[i].x, fmaf(v[i].y, sc.y, sh.y) + adv[i].y,
                             fmaf(v[i].z, sc.z, sh.z) + adv[i].z, fmaf(v[i].w, sc.w, sh.w) + adv[i].w);
      if (p.ep_relu) { f.x = fmaxf(f.x, 0.f); f.y = fmaxf(f.y, 0.f); f.z = fmaxf(f.z, 0.f); f.w = fmaxf(f.w, 0.f); }
      if (i < n_ok) {
        if (p.out) *reinterpret_cast<float4*>(p.out + off + i * rs) = f;
        if (p.out_hi) {
          const __nv_bfloat16 h0 = __float2bfloat16_rn(f.x), h1 = __float2bfloat16_rn(f.y), h2 = __float2bfloat16_rn(f.z), h3 = __float2bfloat16_rn(f.w);
          *reinterpret_cast<uint2*>(p.out_hi + off + i * rs) = make_uint2(pack_bf16x2(h0, h1), pack_bf16x2(h2, h3));
          if (p.out_lo)
            *reinterpret_cast<uint2*>(p.out_lo + off + i * rs) =
                make_uint2(pack_bf16x2(__float2bfloat16_rn(f.x - __bfloat162float(h0)), __float2bfloat16_rn(f.y - __bfloat162float(h1))),
                           pack_bf16x2(__float2bfloat16_rn(f.z - __bfloat162float(h2)), __float2bfloat16_rn(f.w - __bfloat162float(h3))));
        }
      }
    }
  } else if (p.bst.fin.a.acc) {
    // backward statistics: the pre-BatchNorm activation (and the sign plane of the block output) of the same elements
    float4 rw[EPI_ROWS];
    uint2 yh[EPI_ROWS];
#pragma unroll
    for (int i = 0; i < EPI_ROWS; ++i) {
      rw[i] = i < n_ok ? __ldg(reinterpret_cast<const float4*>(p.bst.raw + off + i * rs)) : make_float4(0.f, 0.f, 0.f, 0.f);
      if (p.bst.y_hi) yh[i] = i < n_ok ? __ldg(reinterpret_cast<const uint2*>(p.bst.y_hi + off + i * rs)) : make_uint2(0u, 0u);
    }
    const float4 mu = __ldg(reinterpret_cast<const float4*>(p.bst.mean + (size_t)grp * C + ch));
    const float4 is = __ldg(reinterpret_cast<const float4*>(p.bst.invstd + (size_t)grp * C + ch));
    float4 scl = make_float4(0.f, 0.f, 0.f, 0.f), be = scl;
    if (!p.bst.y_hi && p.bst.relu) {     // no residual in the forward: y > 0 <=> bn(x) > 0, the same fmaf as bn_apply_kernel
      const float4 gm = __ldg(reinterpret_cast<const float4*>(p.bst.gamma + ch));
      be = __ldg(reinterpret_cast<const float4*>(p.bst.beta + ch));
      scl = make_float4(gm.x * is.x, gm.y * is.y, gm.z * is.z, gm.w * is.w);
    }
#pragma unroll
    for (int i = 0; i < EPI_ROWS; ++i) {
      float4 g = make_float4(v[i].x + adv[i].x, v[i].y + adv[i].y, v[i].z + adv[i].z, v[i].w + adv[i].w);
      if (i < n_ok) *reinterpret_cast<float4*>(p.out + off + i * rs) = g;
      else g = make_float4(0.f, 0.f, 0.f, 0.f);
      if (p.bst.y_hi) {
        const uint2 hh = yh[i];
        if ((hh.x & 0x8000u) || !(hh.x & 0x7fffu)) g.x = 0.f;
        if ((hh.x & 0x80000000u) || !(hh.x & 0x7fff0000u)) g.y = 0.f;
        if ((hh.y & 0x8000u) || !(hh.y & 0x7fffu)) g.z = 0.f;
        if ((hh.y & 0x80000000u) || !(hh.y & 0x7fff0000u)) g.w = 0.f;
      } else if (p.bst.relu) {
        if (!(fmaf(rw[i].x - mu.x, scl.x, be.x) > 0.f)) g.x = 0.f;
        if (!(fmaf(rw[i].y - mu.y, scl.y, be.y) > 0.f)) g.y = 0.f;
        if (!(fmaf(rw[i].z - mu.z, scl.z, be.z) > 0.f)) g.z = 0.f;
        if (!(fmaf(rw[i].w - mu.w, scl.w, be.w) > 0.f)) g.w = 0.f;
      }
      s1.x += g.x; s1.y += g.y; s1.z += g.z; s1.w += g.w;
      s2.x = fmaf(g.x, (rw[i].x - mu.x) * is.x, s2.x); s2.y = fmaf(g.y, (rw[i].y - mu.y) * is.y, s2.y);
      s2.z = fmaf(g.z, (rw[i].z - mu.z) * is.z, s2.z); s2.w = fmaf(g.w, (rw[i].w - mu.w) * is.w, s2.w);
    }
  } else {
#pragma unroll
    for (int i = 0; i < EPI_ROWS; ++i) {
      // rows outside the image hold garbage (their shifted taps can read valid pixels): neither stored nor summed
      const float4 raw = i < n_ok ? v[i] : make_float4(0.f, 0.f, 0.f, 0.f);
      if (i < n_ok)
        *reinterpret_cast<float4*>(p.out + off + i * rs) = make_float4(raw.x + adv[i].x, raw.y + adv[i].y, raw.z + adv[i].z, raw.w + adv[i].w);
      s1.x += raw.x; s1.y += raw.y; s1.z += raw.z; s1.w += raw.w;
      s2.x = fmaf(raw.x, raw.x, s2.x); s2.y = fmaf(raw.y, raw.y, s2.y); s2.z = fmaf(raw.z, raw.z, s2.z); s2.w = fmaf(raw.w, raw.w, s2.w);
    }
  }
}

// Column sums of a warp's 16 rows: lane b of the first group ends up with channel quad b (the other rows sit in lanes b + 8,
// b + 16, b + 24).
__device__ __forceinline__ void colsum_lane_groups(float4& s1, float4& s2) {
#pragma unroll
  for (int off = 8; off < 32; off <<= 1) {
    s1.x += __shfl_xor_sync(0xffffffffu, s1.x, off); s1.y += __shfl_xor_sync(0xffffffffu, s1.y, off);
    s1.z += __shfl_xor_sync(0xffffffffu, s1.z, off); s1.w += __shfl_xor_sync(0xffffffffu, s1.w, off);
    s2.x += __shfl_xor_sync(0xffffffffu, s2.x, off); s2.y += __shfl_xor_sync(0xffffffffu, s2.y, off);
    s2.z += __shfl_xor_sync(0xffffffffu, s2.z, off); s2.w += __shfl_xor_sync(0xffffffffu, s2.w, off);
  }
}

__device__ __forceinline__ void named_barrier(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

// After a kernel's last item, in all TC_CONSUMERS consumer threads (named barrier `bar`): the CTA that arrives last turns the
// accumulated sums of C channels into mean / invstd / running statistics (forward), or into dgamma / dbeta and the per-group
// sums bn_bwd_apply_kernel reads (data gradient).
__device__ __forceinline__ void conv_epilogue_finalize(const TcEpilogueParams& p, int C, int* s_last, int bar) {
  if (p.fin.a.acc) {
    if (bn_last_cta(p.fin.a.ticket, gridDim.x, threadIdx.x == 0, s_last, [bar] { named_barrier(bar, TC_CONSUMERS); }))
      for (int c = threadIdx.x; c < C; c += TC_CONSUMERS) bn_fwd_finalize_channel(p.fin, c);
  } else if (p.bst.fin.a.acc) {
    if (bn_last_cta(p.bst.fin.a.ticket, gridDim.x, threadIdx.x == 0, s_last, [bar] { named_barrier(bar, TC_CONSUMERS); }))
      for (int c = threadIdx.x; c < C; c += TC_CONSUMERS) bn_bwd_finalize_channel(p.bst.fin, c);
  }
}

// ------------------------------------------------------------------------------------------------ the kernel
// One persistent, warp-specialised kernel serves every convolution forward and data gradient: a 128-pixel x BLOCK_N tile per
// work item, the two consumer warpgroups taking one 64-row sub-tile each.
//
// Pixels: the output is cut into 4x16-pixel SUB-TILES (one TMA box {64 ch, 16 w, 4 h, 1 n} each, 8 KB); a CTA's 128 MMA
// rows are two consecutive sub-tiles of the flattened (image, row, column) list, which may straddle image borders, so
// 60x80 feature maps lose nothing to tile rounding (8x16 tiles would waste 6.25 % of layers 3 and 4).
// Work items: `full_items` full-width tiles (spatial-major, co-slice minor: the CTAs working on the co-slices of one pixel
// tile share its A loads in L2), then the tiles of the last, partial wave cut along N into `tail_split` pieces of
// BLOCK_N / tail_split channels (own B tensor maps), so that the tail wave costs 1/tail_split of a tile time instead
// of a whole one.  Static round-robin over the items; producer and consumers walk the same sequence.
//
// Epilogue variants: training forward -- raw fp32 output + per-channel sum / sum of squares added to the BatchNorm
// accumulator (bn_stats.cuh), statistics finalized by the last CTA; inference -- eval-mode BN folded to
// relu(acc*scale + shift + residual), written as fp32 and / or the next conv's bf16 planes; data gradient -- + addend.
struct TcConvParams {
  TcEpilogueParams epi;
  int N, H, W, Cin, Cout;   // H, W: OUTPUT size
  int taps_w;            // 1 or 3 (k x k filter)
  int dil;
  int stride;            // 1, or 2 (forward only: the A tensor map then samples every other input pixel)
  int tiles_h, tiles_w;  // 4x16 sub-tiles per image
  int n_sub;             // N * tiles_h * tiles_w
  int n_co;              // Cout / BLOCK_N
  int full_items, tail_split, total_items;
};

constexpr int TC_SUB_H = 4, TC_SUB_W = 16;     // sub-tile = one TMA box = 64 MMA rows
constexpr int TC_SUB_BYTES = 64 * 128;         // 8 KB per plane

struct TcItem { int sp, co0, width; };
__device__ __forceinline__ TcItem tc_item(const TcConvParams& p, int idx, int block_n) {
  int tile = idx, piece = 0, width = block_n;
  if (idx >= p.full_items) {
    const int j = idx - p.full_items;
    tile = p.full_items + j / p.tail_split;
    piece = j - (j / p.tail_split) * p.tail_split;
    width = block_n / p.tail_split;
  }
  TcItem it;
  it.sp = tile / p.n_co;
  it.co0 = (tile - it.sp * p.n_co) * block_n + piece * width;
  it.width = width;
  return it;
}
struct TcSub { int n, h0, w0; bool valid; };
__device__ __forceinline__ TcSub tc_sub(const TcConvParams& p, int st) {
  TcSub s;
  s.valid = st < p.n_sub;
  const int tw = st % p.tiles_w; const int t = st / p.tiles_w;
  const int th = t % p.tiles_h;
  s.n = s.valid ? t / p.tiles_h : p.N;        // image index N is out of bounds for TMA: zero fill, no memory traffic
  s.h0 = th * TC_SUB_H; s.w0 = tw * TC_SUB_W;
  return s;
}

// The k-loop of one item whose tile is W channels wide (BLOCK_N, or a tail piece of 64 or 32 channels): acc / accx are the first
// W columns of the accumulators.  One instantiation per width keeps the accumulator registers of every wgmma in the loop fixed.
// TRANS = 0: K-major operands (a k16 step is 32 bytes along the swizzle row).  TRANS = 1: MN-major operands, the weight
// gradient's 64-pixel boxes of 64 channels (a k16 step is 16 pixel rows, LBO = the next box of 64 channels).
template <int W, int BLOCK_N, int NPROD, int STAGES, int TRANS = 0>
__device__ __forceinline__ void conv_tc_mainloop(float (&acc)[W / 2], float (&accx)[W / 2], int num_kb, uint32_t& g, const uint64_t* full_bar,
                                                 const uint64_t* empty_bar, const uint8_t* smem, int wg, int lane) {
  constexpr int NSPLIT = NPROD == 3 ? 2 : 1;
  constexpr int A_BYTES = 128 * TC_BLOCK_K * 2;
  constexpr int B_BYTES = BLOCK_N * TC_BLOCK_K * 2;
  constexpr int STAGE_BYTES = NSPLIT * (A_BYTES + B_BYTES);
  constexpr uint32_t LBO = TRANS ? TC_SUB_BYTES : 16;
  constexpr int K_STEP = TRANS ? 16 * 128 : 32;
  for (int kb = 0; kb < num_kb; ++kb, ++g) {
    const int s = g % STAGES;
    mbar_wait(smem_u32(&full_bar[s]), (g / STAGES) & 1);
    wgmma_fence();
    const uint32_t stg = smem_u32(smem + (size_t)s * STAGE_BYTES);
    const uint64_t a_hi = gmma_desc(stg + wg * TC_SUB_BYTES, LBO, 1024), a_lo = gmma_desc(stg + A_BYTES + wg * TC_SUB_BYTES, LBO, 1024);
    const uint64_t b_hi = gmma_desc(stg + NSPLIT * A_BYTES, LBO, 1024), b_lo = gmma_desc(stg + 2 * A_BYTES + B_BYTES, LBO, 1024);
#pragma unroll
    for (int k = 0; k < TC_BLOCK_K / 16; ++k) {
      const uint64_t adv = (uint64_t)((k * K_STEP) >> 4);
      mma_k16_x<W, TRANS, NPROD>(acc, accx, a_hi + adv, a_lo + adv, b_hi + adv, b_lo + adv, (kb | k) != 0);
    }
    wgmma_commit();
    wgmma_wait<1>();                                    // the previous k-block's MMAs are done: release its slot
    if (kb > 0 && lane == 0) mbar_arrive(smem_u32(&empty_bar[(g - 1) % STAGES]));
  }
  wgmma_wait<0>();
  fence_acc(acc);
  if (NPROD == 3) { fence_acc(accx); add_cross(acc, accx); }
  if (lane == 0) mbar_arrive(smem_u32(&empty_bar[(g - 1) % STAGES]));
}

template <int BLOCK_N, int NPROD>
__global__ void __launch_bounds__(TC_WIDE_THREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
               const __grid_constant__ CUtensorMap tm_b_hi, const __grid_constant__ CUtensorMap tm_b_lo,
               const __grid_constant__ CUtensorMap tm_bt_hi, const __grid_constant__ CUtensorMap tm_bt_lo,   // tail-width B boxes
               const TcConvParams p) {
  constexpr int NSPLIT = NPROD == 3 ? 2 : 1;
  constexpr int A_BYTES = 128 * TC_BLOCK_K * 2;                // 16 KB = two sub-tile boxes
  constexpr int B_BYTES = BLOCK_N * TC_BLOCK_K * 2;
  constexpr int STAGE_BYTES = NSPLIT * (A_BYTES + B_BYTES);
  constexpr int STAGES = (192 * 1024) / STAGE_BYTES >= 8 ? 8 : (192 * 1024) / STAGE_BYTES;
  static_assert(STAGES >= 2, "pipeline needs at least two stages");

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ __align__(8) uint64_t full_bar[STAGES];
  __shared__ __align__(8) uint64_t empty_bar[STAGES];
  __shared__ int s_last;
  __shared__ __align__(16) float s_stage[TC_CONSUMERS / 32][EPI_WARP_FLOATS];
  __shared__ __align__(16) float s_part[2][2][4][BLOCK_N];     // [warpgroup][sum | sum of squares][warp][column]

  pdl_trigger();
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  const int cin_chunks = p.Cin / TC_BLOCK_K;
  const int num_kb = p.taps_w * p.taps_w * cin_chunks;
  const int half = p.taps_w >> 1;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(smem_u32(&full_bar[s]), 1); mbar_init(smem_u32(&empty_bar[s]), TC_CONSUMERS / 32); }
    fence_barrier_init();
    tma_prefetch_desc(&tm_a_hi); tma_prefetch_desc(&tm_b_hi); tma_prefetch_desc(&tm_bt_hi);
    if (NSPLIT == 2) { tma_prefetch_desc(&tm_a_lo); tma_prefetch_desc(&tm_b_lo); tma_prefetch_desc(&tm_bt_lo); }
  }
  __syncthreads();
  pdl_wait();                      // everything above overlapped the previous kernel's tail; its results are visible from here

  if (warp >= TC_PRODUCER_WARP) {
    // ===== TMA producer: two sub-tiles of A + the B rows of the item's channel slice per k-block
    setmaxnreg_dec<40>();
    if (warp == TC_PRODUCER_WARP && lane == 0) {
      uint32_t g = 0;                                  // global k-block counter across items -> ring slot / phase
      for (int idx = blockIdx.x; idx < p.total_items; idx += gridDim.x) {
        const TcItem it = tc_item(p, idx, BLOCK_N);
        const bool tail = it.width != BLOCK_N;
        const uint32_t stage_tx = (uint32_t)(NSPLIT * (A_BYTES + it.width * TC_BLOCK_K * 2));
        const CUtensorMap* mb_hi = tail ? &tm_bt_hi : &tm_b_hi;
        const CUtensorMap* mb_lo = tail ? &tm_bt_lo : &tm_b_lo;
        const TcSub s0 = tc_sub(p, it.sp * 2), s1 = tc_sub(p, it.sp * 2 + 1);
        for (int kb = 0; kb < num_kb; ++kb, ++g) {
          const int s = g % STAGES;
          mbar_wait(smem_u32(&empty_bar[s]), ((g / STAGES) & 1) ^ 1);
          const int tap = kb / cin_chunks, cc = kb - tap * cin_chunks;
          const int r = tap / p.taps_w, sx = tap - r * p.taps_w;
          const int dh = (r - half) * p.dil, dw = (sx - half) * p.dil;
          uint8_t* stg = smem + (size_t)s * STAGE_BYTES;
          const uint32_t bar = smem_u32(&full_bar[s]);
          mbar_expect_tx(bar, stage_tx);
          tma_load_4d(smem_u32(stg), &tm_a_hi, bar, cc * TC_BLOCK_K, s0.w0 * p.stride + dw, s0.h0 * p.stride + dh, s0.n);
          tma_load_4d(smem_u32(stg + TC_SUB_BYTES), &tm_a_hi, bar, cc * TC_BLOCK_K, s1.w0 * p.stride + dw, s1.h0 * p.stride + dh, s1.n);
          tma_load_2d(smem_u32(stg + NSPLIT * A_BYTES), mb_hi, bar, kb * TC_BLOCK_K, it.co0);
          if (NSPLIT == 2) {
            tma_load_4d(smem_u32(stg + A_BYTES), &tm_a_lo, bar, cc * TC_BLOCK_K, s0.w0 * p.stride + dw, s0.h0 * p.stride + dh, s0.n);
            tma_load_4d(smem_u32(stg + A_BYTES + TC_SUB_BYTES), &tm_a_lo, bar, cc * TC_BLOCK_K, s1.w0 * p.stride + dw, s1.h0 * p.stride + dh, s1.n);
            tma_load_2d(smem_u32(stg + 2 * A_BYTES + B_BYTES), mb_lo, bar, kb * TC_BLOCK_K, it.co0);
          }
        }
      }
    }
  } else {
    // ===== consumer warpgroup wg: MMA rows 64wg .. 64wg+63 = sub-tile wg of the item; warp w of it owns rows 16w .. 16w+15 =
    // image row h0 + w of the sub-tile, and after stage_chunk lane group a holds its columns w0 + 4a .. w0 + 4a + 3
    setmaxnreg_inc<232>();
    const int wg = warp >> 2, w = warp & 3, e = threadIdx.x & 127;
    const int ga = lane >> 3, gb = lane & 7;
    const bool stats = p.epi.fin.a.acc != nullptr;
    const bool bstats = p.epi.bst.fin.a.acc != nullptr;
    double* const sum_acc = bstats ? p.epi.bst.fin.a.acc : p.epi.fin.a.acc;
    float* const st = s_stage[warp];
    float acc[BLOCK_N / 2], accx[BLOCK_N / 2];
    uint32_t g = 0;
    for (int idx = blockIdx.x; idx < p.total_items; idx += gridDim.x) {
      const TcItem it = tc_item(p, idx, BLOCK_N);
      // item widths: BLOCK_N, or a tail piece of 64 or 32 channels (tc_conv_planes never cuts below 32)
      if (it.width == BLOCK_N)
        conv_tc_mainloop<BLOCK_N, BLOCK_N, NPROD, STAGES>(acc, accx, num_kb, g, full_bar, empty_bar, smem, wg, lane);
      else if (BLOCK_N > 64 && it.width == 64)
        conv_tc_mainloop<64, BLOCK_N, NPROD, STAGES>(acc_cols<64>(acc), acc_cols<64>(accx), num_kb, g, full_bar, empty_bar, smem, wg, lane);
      else
        conv_tc_mainloop<32, BLOCK_N, NPROD, STAGES>(acc_cols<32>(acc), acc_cols<32>(accx), num_kb, g, full_bar, empty_bar, smem, wg, lane);

      const TcSub sb = tc_sub(p, it.sp * 2 + wg);
      const int h = sb.h0 + w, w4 = sb.w0 + EPI_ROWS * ga;
      const int n_ok = (sb.valid && h < p.H) ? min(EPI_ROWS, p.W - w4) : 0;          // valid pixels among the 4 (<= 0: none)
      const size_t pix = ((size_t)(n_ok > 0 ? sb.n : 0) * p.H + (n_ok > 0 ? h : 0)) * p.W + (n_ok > 0 ? w4 : 0);
      const size_t cbase = pix * p.Cout + it.co0 + gb * 4;                     // + i * Cout + c * 32
      const int grp = sb.valid ? sb.n / p.epi.imgs_per_group : 0;
#pragma unroll
      for (int c = 0; c < BLOCK_N / 32; ++c) {
        if (c < (it.width >> 5)) {
          float4 v[EPI_ROWS];
          stage_chunk(acc, c, st, lane, v);
          float4 s1 = make_float4(0.f, 0.f, 0.f, 0.f), s2 = s1;      // column sums of this lane's rows (4 channels)
          conv_epilogue_rows(p.epi, v, cbase + c * 32, (size_t)p.Cout, n_ok, it.co0 + c * 32 + gb * 4, p.Cout, grp, s1, s2);
          if (stats || bstats) {
            colsum_lane_groups(s1, s2);
            if (ga == 0) {
              *reinterpret_cast<float4*>(&s_part[wg][0][w][c * 32 + gb * 4]) = s1;
              *reinterpret_cast<float4*>(&s_part[wg][1][w][c * 32 + gb * 4]) = s2;
            }
          }
        }
      }
      if (stats || bstats) {
        named_barrier(1 + wg, 128);          // the 4 warps of this warpgroup
        if (sb.valid)
          for (int col = e; col < it.width; col += 128) {
#pragma unroll
            for (int k = 0; k < 2; ++k) {
              const float sum = s_part[wg][k][0][col] + s_part[wg][k][1][col] + s_part[wg][k][2][col] + s_part[wg][k][3][col];
              red_add_f64(sum_acc + (size_t)(grp * 2 + k) * p.Cout + it.co0 + col, (double)sum);
            }
          }
        named_barrier(1 + wg, 128);          // s_part is rewritten by the next item
      }
    }
    conv_epilogue_finalize(p.epi, p.Cout, &s_last, 3);
  }
}

// ------------------------------------------------------------------------------------------------ 64 -> 64 channels: halo tiles
// The 3x3 convolutions of layer1 (64 -> 64 channels on the 120x160 map) have the lowest arithmetic intensity of the network:
// with one TMA box per (tap, tile) every 128-pixel tile pulls 9 x 32 KB of activations and the whole 147 KB weight tensor
// through L2 -> shared memory, ~1 GB per convolution, and the kernel above runs at the L2-to-SM throughput cap.  This kernel
// loads every operand ONCE:
//   * the weights (9 taps x [64 co x 64 ci], hi and lo planes, 147 KB) stay resident in shared memory for the whole launch;
//   * a tile is 8 rows x 16 columns of output pixels; its 10 x 18 HALO (one TMA box per plane, out-of-bounds = padding) is
//     staged once and all 9 taps read it in place.  The tensor map has H and W swapped, so halo pixel (h, w) is shared-memory
//     row w * 10 + h: MMA row m = 8 * (m / 8) + m % 8 is output pixel (h0 + m % 8, w0 + m / 8), the 8 rows of a core-matrix
//     group are 8 consecutive halo rows, consecutive groups are 10 rows apart (SBO = 1280 B), and tap (r, s) is the same
//     window shifted by (s * 10 + r) rows (a descriptor may start at any 128-byte row, see gmma_desc).  Warpgroup wg takes
//     MMA rows 64wg .. 64wg + 63 = output columns w0 + 8wg .. w0 + 8wg + 7.
// bf16x3 order: first the 72 MMAs that read the hi plane of the tile (hi*lo + hi*hi), then the 36 that read the lo plane.
// The plane ring has 3 slots in bf16 and 2 in bf16x3 (the resident lo weights take the room of the third); the halos of the
// tiles two and three rounds ahead are pulled into L2 by prefetches that occupy no shared memory.
struct TcHaloParams {
  TcEpilogueParams epi;
  int N, H, W;
  int tiles_h, tiles_w, n_tiles;
};
constexpr int HALO_TH = 8, HALO_TW = 16;
constexpr int HALO_BH = HALO_TH + 2, HALO_BW = HALO_TW + 2;
constexpr int HALO_BOX_BYTES = HALO_BH * HALO_BW * 128;                      // 23,040
constexpr int HALO_SLOT = ((HALO_BOX_BYTES + 1023) / 1024) * 1024;           // 23,552
constexpr int HALO_B_TAP = 64 * 128;                                         // one tap: 64 co x 64 ci bf16
constexpr int HALO_B_PLANE = 9 * HALO_B_TAP;
__host__ __device__ constexpr int halo_slots(int nprod) { return nprod == 3 ? 2 : 3; }

template <int NPROD>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv64_halo_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
                   const __grid_constant__ CUtensorMap tm_b_hi, const __grid_constant__ CUtensorMap tm_b_lo, const TcHaloParams p) {
  constexpr int NSPLIT = NPROD == 3 ? 2 : 1;
  constexpr int SLOTS = halo_slots(NPROD);
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_b = smem;                                   // [plane][tap][64 x 128 B]
  uint8_t* smem_a = smem + NSPLIT * HALO_B_PLANE;           // SLOTS plane slots
  __shared__ __align__(8) uint64_t full_bar[SLOTS], empty_bar[SLOTS], b_full;
  __shared__ int s_last;
  __shared__ __align__(16) float s_stage[TC_CONSUMERS / 32][EPI_WARP_FLOATS];
  __shared__ __align__(16) float s_part[2][8][64];          // [sum | sum of squares][consumer warp][column]

  pdl_trigger();
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // provably warp-uniform
  if (threadIdx.x == 0) {
    for (int s = 0; s < SLOTS; ++s) { mbar_init(smem_u32(&full_bar[s]), 1); mbar_init(smem_u32(&empty_bar[s]), TC_CONSUMERS / 32); }
    mbar_init(smem_u32(&b_full), 1);
    fence_barrier_init();
    tma_prefetch_desc(&tm_a_hi); tma_prefetch_desc(&tm_b_hi);
    if (NSPLIT == 2) { tma_prefetch_desc(&tm_a_lo); tma_prefetch_desc(&tm_b_lo); }
  }
  __syncthreads();
  pdl_wait();

  auto tile_of = [&](int t, int& n, int& h0, int& w0) {
    const int tw = t % p.tiles_w; const int q = t / p.tiles_w;
    const int th = q % p.tiles_h; n = q / p.tiles_h;
    h0 = th * HALO_TH; w0 = tw * HALO_TW;
  };

  if (warp == TC_PRODUCER_WARP) {
    if (lane == 0) {
      const uint32_t bb = smem_u32(&b_full);
      mbar_expect_tx(bb, NSPLIT * HALO_B_PLANE);
#pragma unroll 1
      for (int tap = 0; tap < 9; ++tap) {
        tma_load_2d(smem_u32(smem_b + tap * HALO_B_TAP), &tm_b_hi, bb, tap * 64, 0);
        if (NSPLIT == 2) tma_load_2d(smem_u32(smem_b + HALO_B_PLANE + tap * HALO_B_TAP), &tm_b_lo, bb, tap * 64, 0);
      }
      uint32_t g = 0;
      constexpr int PF = 2;
      for (int j = 0; j < PF; ++j) {
        const int tp = blockIdx.x + j * gridDim.x;
        if (tp < p.n_tiles) {
          int n, h0, w0;
          tile_of(tp, n, h0, w0);
          tma_prefetch_l2_4d(&tm_a_hi, 0, h0 - 1, w0 - 1, n);
          if (NSPLIT == 2) tma_prefetch_l2_4d(&tm_a_lo, 0, h0 - 1, w0 - 1, n);
        }
      }
      for (int t = blockIdx.x; t < p.n_tiles; t += gridDim.x) {
        int n, h0, w0;
        {
          const int tp = t + PF * gridDim.x;
          if (tp < p.n_tiles) {
            tile_of(tp, n, h0, w0);
            tma_prefetch_l2_4d(&tm_a_hi, 0, h0 - 1, w0 - 1, n);
            if (NSPLIT == 2) tma_prefetch_l2_4d(&tm_a_lo, 0, h0 - 1, w0 - 1, n);
          }
        }
        tile_of(t, n, h0, w0);
#pragma unroll
        for (int pl = 0; pl < NSPLIT; ++pl, ++g) {
          const int s = g % SLOTS;
          mbar_wait(smem_u32(&empty_bar[s]), ((g / SLOTS) & 1) ^ 1);
          const uint32_t bar = smem_u32(&full_bar[s]);
          mbar_expect_tx(bar, HALO_BOX_BYTES);
          tma_load_4d(smem_u32(smem_a + s * HALO_SLOT), pl == 0 ? &tm_a_hi : &tm_a_lo, bar, 0, h0 - 1, w0 - 1, n);   // map dims: {c, h, w, n}
        }
      }
    }
  } else {
    const int wg = warp >> 2, w = warp & 3;
    const int ga = lane >> 3, gb = lane & 7;
    const bool stats = p.epi.fin.a.acc != nullptr;
    const bool bstats = p.epi.bst.fin.a.acc != nullptr;     // data gradient: column sums of the BatchNorm backward that consumes `out`
    double* const sum_acc = bstats ? p.epi.bst.fin.a.acc : p.epi.fin.a.acc;
    float* const st = s_stage[warp];
    mbar_wait(smem_u32(&b_full), 0);
    const uint64_t bd_hi = gmma_desc_k(smem_u32(smem_b));
    const uint64_t bd_lo = gmma_desc_k(smem_u32(smem_b + HALO_B_PLANE));
    const uint32_t a_wg = (uint32_t)(8 * wg * HALO_BH * 128);      // this warpgroup's 8 output columns
    float acc[32], accx[32];                           // hi*hi | the two small products (see mma_k16_x)
    uint32_t g = 0;
    for (int t = blockIdx.x; t < p.n_tiles; t += gridDim.x) {
      int n, h0, w0;
      tile_of(t, n, h0, w0);
      // descriptors below are `base + compile-time constant` (taps and k-steps fully unrolled)
      const int s_hi = g % SLOTS;
      {   // plane hi of the tile: hi*lo + hi*hi (bf16x3) or hi*hi
        mbar_wait(smem_u32(&full_bar[s_hi]), (g / SLOTS) & 1);
        wgmma_fence();
        const uint64_t a0 = gmma_desc_k(smem_u32(smem_a + s_hi * HALO_SLOT) + a_wg, HALO_BH * 128);
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const uint64_t ad = a0 + (uint64_t)((((tap % 3) * HALO_BH + tap / 3) * 128 + k * 32) >> 4);
            const uint64_t boff = (uint64_t)((tap * HALO_B_TAP + k * 32) >> 4);
            if (NPROD == 3) Wgmma<64>::mma<0>(accx, ad, bd_lo + boff, (tap | k) != 0);
            Wgmma<64>::mma<0>(acc, ad, bd_hi + boff, (tap | k) != 0);
          }
        }
        wgmma_commit();
        ++g;
      }
      if (NPROD == 3) {   // plane lo: lo*hi
        const int s = g % SLOTS;
        mbar_wait(smem_u32(&full_bar[s]), (g / SLOTS) & 1);
        const uint64_t a0 = gmma_desc_k(smem_u32(smem_a + s * HALO_SLOT) + a_wg, HALO_BH * 128);
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
#pragma unroll
          for (int k = 0; k < 4; ++k)
            Wgmma<64>::mma<0>(accx, a0 + (uint64_t)((((tap % 3) * HALO_BH + tap / 3) * 128 + k * 32) >> 4),
                              bd_hi + (uint64_t)((tap * HALO_B_TAP + k * 32) >> 4), 1);
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (lane == 0) mbar_arrive(smem_u32(&empty_bar[s_hi]));
        ++g;
      }
      wgmma_wait<0>();
      fence_acc(acc);
      if (NPROD == 3) { fence_acc(accx); add_cross(acc, accx); }
      if (lane == 0) mbar_arrive(smem_u32(&empty_bar[(g - 1) % SLOTS]));

      // warp w holds MMA rows 64wg + 16w .. + 15 = output column w0 + 8wg + 2w + (ga >> 1), rows h0 + 4(ga & 1) + i after the
      // staging (the tiles are whole: H % 8 == 0, W % 16 == 0)
      const size_t pix0 = ((size_t)n * p.H + h0 + EPI_ROWS * (ga & 1)) * p.W + (w0 + 8 * wg + 2 * w + (ga >> 1));
      const size_t row_stride = (size_t)p.W * 64;      // floats between (h, w) and (h + 1, w)
      const int grp = n / p.epi.imgs_per_group;        // a tile lies inside one image
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        float4 v[EPI_ROWS];
        stage_chunk(acc, c, st, lane, v);
        float4 s1 = make_float4(0.f, 0.f, 0.f, 0.f), s2 = s1;
        conv_epilogue_rows(p.epi, v, pix0 * 64 + gb * 4 + c * 32, row_stride, EPI_ROWS, c * 32 + gb * 4, 64, grp, s1, s2);
        if (stats || bstats) {
          colsum_lane_groups(s1, s2);
          if (ga == 0) {
            *reinterpret_cast<float4*>(&s_part[0][warp][c * 32 + gb * 4]) = s1;
            *reinterpret_cast<float4*>(&s_part[1][warp][c * 32 + gb * 4]) = s2;
          }
        }
      }
      if (stats || bstats) {
        named_barrier(3, TC_CONSUMERS);
        if (threadIdx.x < 128) {
          const int col = threadIdx.x & 63, k = threadIdx.x >> 6;     // 128 threads = 64 columns x {sum, sum of squares}
          float s8 = 0.f;
#pragma unroll
          for (int q = 0; q < 8; ++q) s8 += s_part[k][q][col];
          red_add_f64(sum_acc + (size_t)(grp * 2 + k) * 64 + col, (double)s8);
        }
        named_barrier(3, TC_CONSUMERS);                // s_part is rewritten by the next tile
      }
    }
    conv_epilogue_finalize(p.epi, 64, &s_last, 3);
  }
}

// ------------------------------------------------------------------------------------------------ weight gradient
// dW[co][tap][ci] = sum_pixels dY[pixel][co] * X[pixel + offset(tap)][ci]  as a wgmma GEMM with the PIXELS as the K
// dimension.  Both operands are the same NHWC bf16 planes the forward reads, consumed as MN-MAJOR operands
// (channels contiguous, pixels = K rows), so no transposed copy exists anywhere:
//   A = dY patch: 64 pixels (4x16) x 128 output channels = two TMA boxes {64 c, 16 w, 4 h, 1 n}, 8 KB each
//   B = X  patch: the 64 pixels shifted by the tap x BN input channels = BN/64 boxes at (w0+(s-1)dil, h0+(r-1)dil); OOB zero
//                 fill is the padding, the shift only touches the W/H coordinates
// In shared memory a box is 64 rows (pixels) of 128 swizzled bytes (64 channels): the canonical MN-major SWIZZLE_128B
// layout with SBO = 1024 B (next 8 pixels) and LBO = 8192 B (next 64 channels = next box).  The stage ring {A_hi, A_lo, B_hi,
// B_lo} and the k-loop are conv_tc_kernel's (conv_tc_mainloop, TRANS = 1): consumer warpgroup wg issues wgmma.m64nBNk16 for
// output channels co0 + 64wg .. + 63, the two small bf16x3 products into their own accumulator.
// A tile is 128 co x BN ci x ONE tap (BN = 128 when Cin % 128 == 0, else 64), so 3x3 and 1x1 convolutions share one path.
// Work item = (pixel chunk c, tile), numbered chunk-major (item = c * n_tiles + tile) and dealt round-robin to a persistent
// grid: the CTAs running at one time walk the same pixel range, so the tiles that read a k-block find it in L2.  The host
// picks the chunk count (tc_wgrad_chunks).  At the end of an item each warp adds its fp32 partial into dwp[tap][co][ci] with
// fp64 reds, staged through shared memory so that one red instruction covers 32 consecutive doubles of a row; the producer
// meanwhile loads the next item's stages.  dwp is fp64 and zero-filled: the partial sums arrive in any order and still round
// to the same fp32 gradient, so a step computes the same weight gradients every run.
struct TcWgradParams {
  double* dwp;           // [taps][Cout][Cin] fp64, zero-filled by the caller
  int N, H, W, Cin, Cout;   // H, W: OUTPUT (dY) size
  int taps_w, dil, stride;
  int tiles_h, tiles_w;  // 4x16 (output-)pixel patches per image
  int total_kb;          // N * tiles_h * tiles_w
  int n_co, n_ci, n_tiles;   // n_tiles = n_co * n_ci * taps
  int chunks;            // pixel chunks: chunk c holds k-blocks [c * total_kb / chunks, (c + 1) * total_kb / chunks)
};

struct WgradItem { int co0, ci0, tap, kb0, kb1; };
__device__ __forceinline__ WgradItem wgrad_item(const TcWgradParams& p, int idx, int bn) {
  const int c = idx / p.n_tiles;
  int t = idx - c * p.n_tiles;
  WgradItem it;
  it.co0 = (t % p.n_co) * 128; t /= p.n_co;
  it.ci0 = (t % p.n_ci) * bn;
  it.tap = t / p.n_ci;
  it.kb0 = (int)((int64_t)c * p.total_kb / p.chunks);
  it.kb1 = (int)((int64_t)(c + 1) * p.total_kb / p.chunks);
  return it;
}

template <int BN, int NPROD>
__global__ void __launch_bounds__(TC_WIDE_THREADS, 1)
wgrad_tc_kernel(const __grid_constant__ CUtensorMap tm_dy_hi, const __grid_constant__ CUtensorMap tm_dy_lo,
                const __grid_constant__ CUtensorMap tm_x_hi, const __grid_constant__ CUtensorMap tm_x_lo,
                const TcWgradParams p) {
  constexpr int NSPLIT = NPROD == 3 ? 2 : 1;
  constexpr int B_BYTES = BN * TC_BLOCK_K * 2;
  constexpr int STAGE_BYTES = NSPLIT * (TC_A_BYTES + B_BYTES);
  constexpr int STAGES = (192 * 1024) / STAGE_BYTES >= 8 ? 8 : (192 * 1024) / STAGE_BYTES;
  static_assert(STAGES >= 2, "pipeline needs at least two stages");

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ __align__(8) uint64_t full_bar[STAGES];
  __shared__ __align__(8) uint64_t empty_bar[STAGES];
  __shared__ __align__(16) float s_stage[TC_CONSUMERS / 32][EPI_WARP_FLOATS];

  pdl_trigger();
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  const int total_items = p.chunks * p.n_tiles;
  const int half = p.taps_w >> 1;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(smem_u32(&full_bar[s]), 1); mbar_init(smem_u32(&empty_bar[s]), TC_CONSUMERS / 32); }
    fence_barrier_init();
    tma_prefetch_desc(&tm_dy_hi); tma_prefetch_desc(&tm_x_hi);
    if (NSPLIT == 2) { tma_prefetch_desc(&tm_dy_lo); tma_prefetch_desc(&tm_x_lo); }
  }
  __syncthreads();
  pdl_wait();

  if (warp >= TC_PRODUCER_WARP) {
    // ===== TMA producer: 128 channels of dY + BN channels of X (shifted by the item's tap) per 64-pixel k-block
    setmaxnreg_dec<40>();
    if (warp == TC_PRODUCER_WARP && lane == 0) {
      uint32_t g = 0;                                  // global k-block counter across items -> ring slot / phase
      for (int idx = blockIdx.x; idx < total_items; idx += gridDim.x) {
        const WgradItem it = wgrad_item(p, idx, BN);
        const int r = it.tap / p.taps_w, sx = it.tap - r * p.taps_w;
        const int dh = (r - half) * p.dil, dw = (sx - half) * p.dil;
        for (int kb = it.kb0; kb < it.kb1; ++kb, ++g) {
          const int s = g % STAGES;
          mbar_wait(smem_u32(&empty_bar[s]), ((g / STAGES) & 1) ^ 1);
          const int tw = kb % p.tiles_w, q = kb / p.tiles_w;
          const int th = q % p.tiles_h, n = q / p.tiles_h;
          const int h0 = th * TC_SUB_H, w0 = tw * TC_SUB_W;
          const int hh = h0 * p.stride + dh, ww = w0 * p.stride + dw;
          uint8_t* stg = smem + (size_t)s * STAGE_BYTES;
          const uint32_t bar = smem_u32(&full_bar[s]);
          mbar_expect_tx(bar, STAGE_BYTES);
#pragma unroll
          for (int hf = 0; hf < 2; ++hf) {      // channels co0+64..127 of a 64-channel tensor are out of bounds = zeros
            tma_load_4d(smem_u32(stg + hf * TC_SUB_BYTES), &tm_dy_hi, bar, it.co0 + 64 * hf, w0, h0, n);
            if (NSPLIT == 2) tma_load_4d(smem_u32(stg + TC_A_BYTES + hf * TC_SUB_BYTES), &tm_dy_lo, bar, it.co0 + 64 * hf, w0, h0, n);
          }
#pragma unroll
          for (int part = 0; part < BN / 64; ++part) {
            tma_load_4d(smem_u32(stg + NSPLIT * TC_A_BYTES + part * TC_SUB_BYTES), &tm_x_hi, bar, it.ci0 + 64 * part, ww, hh, n);
            if (NSPLIT == 2)
              tma_load_4d(smem_u32(stg + 2 * TC_A_BYTES + B_BYTES + part * TC_SUB_BYTES), &tm_x_lo, bar, it.ci0 + 64 * part, ww, hh, n);
          }
        }
      }
    }
  } else {
    // ===== consumer warpgroup wg: accumulator rows = output channels co0 + 64wg + 16w + lane/4 (+ 8), columns = input channels
    setmaxnreg_inc<232>();
    const int wg = warp >> 2, w = warp & 3;
    float* const st = s_stage[warp];
    float acc[BN / 2], accx[BN / 2];
    uint32_t g = 0;
    for (int idx = blockIdx.x; idx < total_items; idx += gridDim.x) {
      const WgradItem it = wgrad_item(p, idx, BN);
      if (it.co0 + 64 * wg >= p.Cout) {               // a 64-channel dY leaves the second warpgroup nothing to do
        for (int kb = it.kb0; kb < it.kb1; ++kb, ++g) {
          mbar_wait(smem_u32(&full_bar[g % STAGES]), (g / STAGES) & 1);
          if (lane == 0) mbar_arrive(smem_u32(&empty_bar[g % STAGES]));
        }
      } else {
        conv_tc_mainloop<BN, BN, NPROD, STAGES, 1>(acc, accx, it.kb1 - it.kb0, g, full_bar, empty_bar, smem, wg, lane);
        // lane l adds column 32c + l of the warp's 16 rows: 32 consecutive doubles per red instruction
        double* const dst = p.dwp + ((size_t)it.tap * p.Cout + it.co0 + 64 * wg + 16 * w) * p.Cin + it.ci0 + lane;
#pragma unroll
        for (int c = 0; c < BN / 32; ++c) {
          stage_write(acc, c, st, lane);
#pragma unroll
          for (int i = 0; i < 16; ++i) red_add_f64(dst + (size_t)i * p.Cin + 32 * c, (double)st[i * EPI_STRIDE + lane]);
          __syncwarp();                                 // the tile is rewritten by the next chunk
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ 64 -> 64 weight gradient: halo tiles
// The kernel above gives a 64 x 64 convolution (layer1) half-empty tiles (128 co rows for 64 output channels) and, with one X box
// per (tap, 64 pixels), ~1.1 GB of L2 -> shared-memory traffic per weight gradient: it runs at the L2 throughput cap.  Here a
// CTA walks 8 x 16-pixel tiles (the geometry and the H/W-swapped tensor maps of conv64_halo_kernel); per tile it stages the
// 10 x 18 halo of X and the 8 x 16 tile of dY ONCE, and
//   * the roles are swapped: the M side is X, shifted by the tap (an MN-major descriptor starting at the tap's halo row), the
//     N side is dY (64 output channels); K = pixels, 16 per MMA = two columns of 8 rows (SBO = 10 halo rows for X, 8 for dY);
//   * three consumer warpgroups, one per filter row r, each keep the [64 ci] x [64 co] fp32 accumulators of taps (r, 0..2) in
//     registers for the whole launch.
// At the end each CTA adds its partial dW into dwp[tap][co][ci] (fp64 reds, see wgrad_tc_kernel).
struct TcWgradHaloParams {
  double* dwp;           // [9][64][64] fp64, zero-filled by the caller
  int N, H, W;
  int tiles_h, tiles_w, n_tiles;
};
constexpr int WGH_CONSUMERS = 384;                       // three warpgroups
constexpr int WGH_THREADS = WGH_CONSUMERS + 32;
constexpr int WGH_X_SLOT = HALO_SLOT;                    // 10 x 18 halo of X, one plane
constexpr int WGH_DY_BYTES = 128 * 128;                  // 8 x 16 pixels x 64 channels, one plane
__host__ __device__ constexpr int wgh_off(int tap) { return (tap % 3) * HALO_BH + tap / 3; }       // halo row of tap (r, s) = s * 10 + r

template <int NPROD>
__global__ void __launch_bounds__(WGH_THREADS, 1)
wgrad64_halo_kernel(const __grid_constant__ CUtensorMap tm_x_hi, const __grid_constant__ CUtensorMap tm_x_lo,
                    const __grid_constant__ CUtensorMap tm_dy_hi, const __grid_constant__ CUtensorMap tm_dy_lo, const TcWgradHaloParams p) {
  constexpr int NSPLIT = NPROD == 3 ? 2 : 1;
  constexpr int STAGE = NSPLIT * (WGH_X_SLOT + WGH_DY_BYTES);
  constexpr int STAGES = 2;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ __align__(8) uint64_t full_bar[STAGES], empty_bar[STAGES];

  pdl_trigger();
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(smem_u32(&full_bar[s]), 1); mbar_init(smem_u32(&empty_bar[s]), WGH_CONSUMERS / 32); }
    fence_barrier_init();
    tma_prefetch_desc(&tm_x_hi); tma_prefetch_desc(&tm_dy_hi);
    if (NSPLIT == 2) { tma_prefetch_desc(&tm_x_lo); tma_prefetch_desc(&tm_dy_lo); }
  }
  __syncthreads();
  pdl_wait();
  const int my_tiles = p.n_tiles > (int)blockIdx.x ? (p.n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
  if (my_tiles == 0) return;

  if (warp == WGH_CONSUMERS / 32) {
    if (lane == 0) {
      int i = 0;
      for (int t = blockIdx.x; t < p.n_tiles; t += gridDim.x, ++i) {
        const int tw = t % p.tiles_w; const int q = t / p.tiles_w;
        const int th = q % p.tiles_h, n = q / p.tiles_h;
        const int h0 = th * HALO_TH, w0 = tw * HALO_TW;
        const int s = i % STAGES;
        mbar_wait(smem_u32(&empty_bar[s]), ((i / STAGES) & 1) ^ 1);
        const uint32_t bar = smem_u32(&full_bar[s]);
        mbar_expect_tx(bar, NSPLIT * (HALO_BOX_BYTES + WGH_DY_BYTES));
        uint8_t* stg = smem + (size_t)s * STAGE;
        tma_load_4d(smem_u32(stg), &tm_x_hi, bar, 0, h0 - 1, w0 - 1, n);                               // map dims {c, h, w, n}
        tma_load_4d(smem_u32(stg + NSPLIT * WGH_X_SLOT), &tm_dy_hi, bar, 0, h0, w0, n);
        if (NSPLIT == 2) {
          tma_load_4d(smem_u32(stg + WGH_X_SLOT), &tm_x_lo, bar, 0, h0 - 1, w0 - 1, n);
          tma_load_4d(smem_u32(stg + NSPLIT * WGH_X_SLOT + WGH_DY_BYTES), &tm_dy_lo, bar, 0, h0, w0, n);
        }
      }
    }
  } else {
    const int r = warp >> 2, w = warp & 3;              // warpgroup r: taps (r, 0), (r, 1), (r, 2)
    float acc[3][32];
    for (int i = 0; i < my_tiles; ++i) {
      const int s = i % STAGES;
      mbar_wait(smem_u32(&full_bar[s]), (i / STAGES) & 1);
      wgmma_fence();
      const uint32_t stg = smem_u32(smem + (size_t)s * STAGE);
      const uint32_t x_hi = stg, x_lo = stg + WGH_X_SLOT;
      const uint32_t d_hi = stg + NSPLIT * WGH_X_SLOT, d_lo = d_hi + WGH_DY_BYTES;
      const uint64_t b_hi0 = gmma_desc(d_hi, 1024, 1024);
      const uint64_t b_lo0 = gmma_desc(d_lo, 1024, 1024);
#pragma unroll
      for (int sx = 0; sx < 3; ++sx) {
        const int oa = wgh_off(r * 3 + sx);
        const uint64_t a_hi0 = gmma_desc(x_hi + oa * 128, 1024, HALO_BH * 128);
        const uint64_t a_lo0 = gmma_desc(x_lo + oa * 128, 1024, HALO_BH * 128);
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {                    // 16 pixels: columns 2kk, 2kk + 1 of the tile
          const uint64_t a_adv = (uint64_t)((2 * kk * HALO_BH * 128) >> 4);
          const uint64_t b_adv = (uint64_t)((kk * 16 * 128) >> 4);
          mma_k16<64, 1, NPROD>(acc[sx], a_hi0 + a_adv, a_lo0 + a_adv, b_hi0 + b_adv, b_lo0 + b_adv, (i | kk) != 0);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (i > 0 && lane == 0) mbar_arrive(smem_u32(&empty_bar[(i - 1) % STAGES]));
    }
    wgmma_wait<0>();
#pragma unroll
    for (int sx = 0; sx < 3; ++sx) fence_acc(acc[sx]);
    // accumulator row = input channel 16w + lane/4 (+ 8), column = output channel 8j + 2(lane % 4) (+ 1)
    const int ci = 16 * w + (lane >> 2), co = 2 * (lane & 3);
#pragma unroll
    for (int sx = 0; sx < 3; ++sx) {
      double* dst = p.dwp + (size_t)(r * 3 + sx) * 64 * 64;    // [tap][co][ci]
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        red_add_f64(dst + (size_t)(co + 8 * j) * 64 + ci, (double)acc[sx][4 * j]);
        red_add_f64(dst + (size_t)(co + 8 * j + 1) * 64 + ci, (double)acc[sx][4 * j + 1]);
        red_add_f64(dst + (size_t)(co + 8 * j) * 64 + ci + 8, (double)acc[sx][4 * j + 2]);
        red_add_f64(dst + (size_t)(co + 8 * j + 1) * 64 + ci + 8, (double)acc[sx][4 * j + 3]);
      }
    }
  }
}

// dwp[tap][co][ci] -> dw[co][ci][r][s]
__global__ void unpack_wgrad_tc_kernel(const double* __restrict__ dwp, float* __restrict__ dw, int Cout, int Cin, int taps) {
  pdl_prologue();
  const int64_t total = (int64_t)Cout * Cin * taps;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int tap = (int)(i % taps); int64_t q = i / taps;
    int ci = (int)(q % Cin); int co = (int)(q / Cin);
    dw[i] = (float)dwp[((int64_t)tap * Cout + co) * Cin + ci];
  }
}

// The same for many convolutions in ONE launch (blockIdx.y = table entry): the network backward leaves every conv's
// [taps][Cout][Cin] accumulator in one scratch array and converts a whole gradient bucket (a residual layer) at once.
// kind 1 = stem: dW'[co][192] (k = (r*7+s)*3 + c) -> conv1.weight gradient [64][3][7][7].
__global__ void unpack_wgrad_batched_kernel(const double* __restrict__ dwp_base, float* __restrict__ grads_base, TcUnpackTable t) {
  pdl_prologue();
  const TcUnpackEntry en = t.e[blockIdx.y];
  const double* __restrict__ dwp = dwp_base + en.src_off;
  float* __restrict__ dw = grads_base + en.dst_off;
  if (en.kind == 1) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < 64 * 147; i += gridDim.x * blockDim.x) {
      const int rs = i % 49, c = (i / 49) % 3, co = i / 147;
      dw[i] = (float)dwp[co * 192 + rs * 3 + c];
    }
    return;
  }
  const int64_t total = (int64_t)en.Cout * en.Cin * en.taps;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int tap = (int)(i % en.taps); int64_t q = i / en.taps;
    int ci = (int)(q % en.Cin); int co = (int)(q / en.Cin);
    dw[i] = (float)dwp[((int64_t)tap * en.Cout + co) * en.Cin + ci];
  }
}

// ------------------------------------------------------------------------------------------------ operand preparation
// x fp32 -> hi = bf16(x), lo = bf16(x - hi)      (n multiple of 4)
__global__ void split_bf16_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                                  int64_t n4, int want_lo) {
  pdl_prologue();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
    __nv_bfloat16 h0 = __float2bfloat16_rn(v.x), h1 = __float2bfloat16_rn(v.y), h2 = __float2bfloat16_rn(v.z), h3 = __float2bfloat16_rn(v.w);
    __nv_bfloat162 a = __halves2bfloat162(h0, h1), b = __halves2bfloat162(h2, h3);
    uint2 ho; ho.x = *reinterpret_cast<uint32_t*>(&a); ho.y = *reinterpret_cast<uint32_t*>(&b);
    reinterpret_cast<uint2*>(hi)[i] = ho;
    if (want_lo) {
      __nv_bfloat162 c = __halves2bfloat162(__float2bfloat16_rn(v.x - __bfloat162float(h0)), __float2bfloat16_rn(v.y - __bfloat162float(h1)));
      __nv_bfloat162 d = __halves2bfloat162(__float2bfloat16_rn(v.z - __bfloat162float(h2)), __float2bfloat16_rn(v.w - __bfloat162float(h3)));
      uint2 lo2; lo2.x = *reinterpret_cast<uint32_t*>(&c); lo2.y = *reinterpret_cast<uint32_t*>(&d);
      reinterpret_cast<uint2*>(lo)[i] = lo2;
    }
  }
}

// w [Cout][Cin][k][k] fp32 ->  fwd:   B[co][(r*k+s)*Cin + ci]
//                             dgrad: B[ci][(r'*k+s')*Cout + co]  with (r,s) = (k-1-r', k-1-s')
__global__ void pack_weights_tc_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                                       int Cout, int Cin, int k, int dgrad, int want_lo) {
  pdl_prologue();
  const int64_t total = (int64_t)Cout * Cin * k * k;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int co, ci, r, s;
    if (!dgrad) {
      ci = (int)(i % Cin); int64_t q = i / Cin;
      s = (int)(q % k); q /= k;
      r = (int)(q % k); co = (int)(q / k);
    } else {
      co = (int)(i % Cout); int64_t q = i / Cout;
      s = k - 1 - (int)(q % k); q /= k;
      r = k - 1 - (int)(q % k); ci = (int)(q / k);
    }
    float v = w[(((int64_t)co * Cin + ci) * k + r) * k + s];
    __nv_bfloat16 h = __float2bfloat16_rn(v);
    hi[i] = h;
    if (want_lo) lo[i] = __float2bfloat16_rn(v - __bfloat162float(h));
  }
}


// dY fp32 [N,Ho,Wo,C] -> zero-inserted bf16 planes [N,2Ho,2Wo,C]: value at (2ho,2wo), zeros at the other three positions.
// The data gradient of a stride-2 convolution is then an ordinary stride-1 convolution over these planes.
__global__ void upsample_zero_split_kernel(const float* __restrict__ dy, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                                           int N, int Ho, int Wo, int C, int want_lo) {
  pdl_prologue();
  const int q = C >> 2;
  const int64_t total = (int64_t)N * Ho * Wo * q;
  const uint2 z = make_uint2(0u, 0u);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int c4 = (int)(i % q); int64_t t = i / q;
    int wo = (int)(t % Wo); t /= Wo;
    int ho = (int)(t % Ho); int n = (int)(t / Ho);
    float4 v = __ldg(reinterpret_cast<const float4*>(dy) + i);
    __nv_bfloat16 h0 = __float2bfloat16_rn(v.x), h1 = __float2bfloat16_rn(v.y), h2 = __float2bfloat16_rn(v.z), h3 = __float2bfloat16_rn(v.w);
    __nv_bfloat162 a = __halves2bfloat162(h0, h1), b = __halves2bfloat162(h2, h3);
    uint2 hv; hv.x = *reinterpret_cast<uint32_t*>(&a); hv.y = *reinterpret_cast<uint32_t*>(&b);
    uint2 lv = z;
    if (want_lo) {
      __nv_bfloat162 c = __halves2bfloat162(__float2bfloat16_rn(v.x - __bfloat162float(h0)), __float2bfloat16_rn(v.y - __bfloat162float(h1)));
      __nv_bfloat162 d = __halves2bfloat162(__float2bfloat16_rn(v.z - __bfloat162float(h2)), __float2bfloat16_rn(v.w - __bfloat162float(h3)));
      lv.x = *reinterpret_cast<uint32_t*>(&c); lv.y = *reinterpret_cast<uint32_t*>(&d);
    }
    const int64_t W2 = 2 * Wo;
    const int64_t base = (((int64_t)n * 2 * Ho + 2 * ho) * W2 + 2 * wo) * q + c4;
    uint2* H = reinterpret_cast<uint2*>(hi); uint2* L = reinterpret_cast<uint2*>(lo);
    H[base] = hv; H[base + q] = z; H[base + W2 * q] = z; H[base + W2 * q + q] = z;
    if (want_lo) { L[base] = lv; L[base + q] = z; L[base + W2 * q] = z; L[base + W2 * q + q] = z; }
  }
}

// Stem: x fp32 NCHW [N,3,H,W] -> 7x7/2 patch planes [N,H1,W1,192] bf16 (k = (r*7+s)*3 + c for k < 147, zero above), so
// that conv1 becomes a GEMM with K = 192 on the tensor cores.  One block = one output row x 64 output columns: the 7 input
// rows x 133 input columns x 3 channels it needs are staged in shared memory with coalesced loads, then written out as
// 384-byte (hi) + 384-byte (lo) rows per output pixel.
constexpr int STEM_TW = 64;
constexpr int STEM_COLS = 2 * STEM_TW + 5;
__global__ void __launch_bounds__(256)
stem_patch_split_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                        int N, int H, int W, int H1, int W1, int want_lo) {
  pdl_prologue();
  __shared__ float tile[3 * 7 * (STEM_COLS + 1) + 4];
  __shared__ int koff[192];          // k -> offset of (c, r, s) inside `tile` (the + 2*px part is added per pixel); -1 = zero padding
  const int wt = blockIdx.x, ho = blockIdx.y, n = blockIdx.z;
  const int wo0 = wt * STEM_TW;
  const int h_base = 2 * ho - 3, w_base = 2 * wo0 - 3;
  for (int k = threadIdx.x; k < 192; k += blockDim.x) {
    int off = -1;
    if (k < 147) { const int c = k % 3, rs = k / 3, r = rs / 7, sx = rs - r * 7; off = (c * 7 + r) * (STEM_COLS + 1) + sx; }
    koff[k] = off;
  }
  for (int i = threadIdx.x; i < 3 * 7 * STEM_COLS; i += blockDim.x) {
    int col = i % STEM_COLS, rc = i / STEM_COLS;
    int r = rc % 7, c = rc / 7;
    int h = h_base + r, w = w_base + col;
    float v = 0.f;
    if (h >= 0 && h < H && w >= 0 && w < W) v = __ldg(x + (((int64_t)n * 3 + c) * H + h) * W + w);
    tile[(c * 7 + r) * (STEM_COLS + 1) + col] = v;
  }
  __syncthreads();
  const int npix = min(STEM_TW, W1 - wo0);
  // thread -> a fixed group of 4 consecutive k (its four tile offsets live in registers), looping over the pixels
  const int kq = threadIdx.x % 48, px0 = threadIdx.x / 48;
  const int pstep = blockDim.x / 48;            // 256 threads: 5 pixels per sweep (16 threads idle)
  if (px0 < pstep) {
    const int o0 = koff[kq * 4], o1 = koff[kq * 4 + 1], o2 = koff[kq * 4 + 2], o3 = koff[kq * 4 + 3];
    for (int px = px0; px < npix; px += pstep) {
      const int b2 = 2 * px;
      float v[4];
      v[0] = o0 >= 0 ? tile[o0 + b2] : 0.f; v[1] = o1 >= 0 ? tile[o1 + b2] : 0.f;
      v[2] = o2 >= 0 ? tile[o2 + b2] : 0.f; v[3] = o3 >= 0 ? tile[o3 + b2] : 0.f;
      const int64_t o = (((int64_t)n * H1 + ho) * W1 + wo0 + px) * 48 + kq;
      __nv_bfloat16 h0 = __float2bfloat16_rn(v[0]), h1 = __float2bfloat16_rn(v[1]), h2 = __float2bfloat16_rn(v[2]), h3 = __float2bfloat16_rn(v[3]);
      __nv_bfloat162 a = __halves2bfloat162(h0, h1), b = __halves2bfloat162(h2, h3);
      uint2 hv; hv.x = *reinterpret_cast<uint32_t*>(&a); hv.y = *reinterpret_cast<uint32_t*>(&b);
      reinterpret_cast<uint2*>(hi)[o] = hv;
      if (want_lo) {
        __nv_bfloat162 c2 = __halves2bfloat162(__float2bfloat16_rn(v[0] - __bfloat162float(h0)), __float2bfloat16_rn(v[1] - __bfloat162float(h1)));
        __nv_bfloat162 d2 = __halves2bfloat162(__float2bfloat16_rn(v[2] - __bfloat162float(h2)), __float2bfloat16_rn(v[3] - __bfloat162float(h3)));
        uint2 lv; lv.x = *reinterpret_cast<uint32_t*>(&c2); lv.y = *reinterpret_cast<uint32_t*>(&d2);
        reinterpret_cast<uint2*>(lo)[o] = lv;
      }
    }
  }
}

// conv1.weight [64][3][7][7] fp32 -> B[co][k] bf16 hi/lo with k = (r*7+s)*3 + c, zero for k in [147,192)
__global__ void stem_pack_weights_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, int want_lo) {
  pdl_prologue();
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 64 * 192) return;
  int k = i % 192, co = i / 192;
  float v = 0.f;
  if (k < 147) { int c = k % 3, rs = k / 3; v = w[(co * 3 + c) * 49 + rs]; }
  __nv_bfloat16 h = __float2bfloat16_rn(v);
  hi[i] = h;
  if (want_lo) lo[i] = __float2bfloat16_rn(v - __bfloat162float(h));
}

// ------------------------------------------------------------------------------------------------ weight-pack cache
// The packed bf16 weights of every conv (forward and data-gradient layouts) live in a caller-owned cache that must never be
// stale.  Staleness is decided ON THE DEVICE: every forward fingerprints the whole fp32 parameter array (two 64-bit sums
// over the raw words, one of them position-weighted: an 85 MB read, ~15 us) and the batched pack kernel re-packs only when
// the fingerprint differs from the one the packs were made from -- so a write through `.data`, a raw pointer, an optimizer
// or NCCL is caught without any host-side version bookkeeping, and an unchanged array costs three tiny launches.
__global__ void __launch_bounds__(256)
param_fingerprint_kernel(const uint32_t* __restrict__ w, int64_t n, unsigned long long* __restrict__ fp) {
  pdl_prologue();
  unsigned long long s1 = 0, s2 = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long v = __ldg(w + i);
    s1 += v;
    s2 += v * (0x9E3779B97F4A7C15ull * (unsigned long long)(i + 1) | 1ull);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
  if ((threadIdx.x & 31) == 0) { atomicAdd(fp, s1); atomicAdd(fp + 1, s2); }
}

// blockIdx.y = table entry; packs entry's conv unless the fingerprint is unchanged (fp_new == fp_old) and !force
__global__ void __launch_bounds__(256)
pack_all_kernel(const float* __restrict__ params, char* __restrict__ cache, TcPackTable t, const unsigned long long* __restrict__ fp_new,
                const unsigned long long* __restrict__ fp_old, int force, int want_lo) {
  pdl_prologue();
  if (!force && fp_new[0] == fp_old[0] && fp_new[1] == fp_old[1]) return;
  const TcPackEntry en = t.e[blockIdx.y];
  const float* __restrict__ w = params + en.w_off;
  __nv_bfloat16* __restrict__ hi = reinterpret_cast<__nv_bfloat16*>(cache + en.dst_off);
  if (en.kind == 1) {          // stem: conv1.weight [64][3][7][7] -> B[co][k], k = (r*7+s)*3 + c, zero for k in [147,192)
    __nv_bfloat16* __restrict__ lo = hi + 64 * 192;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < 64 * 192; i += gridDim.x * blockDim.x) {
      const int k = i % 192, co = i / 192;
      float v = 0.f;
      if (k < 147) { const int c = k % 3, rs = k / 3; v = w[(co * 3 + c) * 49 + rs]; }
      const __nv_bfloat16 h = __float2bfloat16_rn(v);
      hi[i] = h;
      if (want_lo) lo[i] = __float2bfloat16_rn(v - __bfloat162float(h));
    }
    return;
  }
  const int Cout = en.Cout, Cin = en.Cin, k = en.k;
  const int64_t total = (int64_t)Cout * Cin * k * k;
  __nv_bfloat16* __restrict__ lo = hi + total;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int co, ci, r, s;
    if (!en.dgrad) {
      ci = (int)(i % Cin); int64_t q = i / Cin;
      s = (int)(q % k); q /= k;
      r = (int)(q % k); co = (int)(q / k);
    } else {
      co = (int)(i % Cout); int64_t q = i / Cout;
      s = k - 1 - (int)(q % k); q /= k;
      r = k - 1 - (int)(q % k); ci = (int)(q / k);
    }
    const float v = w[(((int64_t)co * Cin + ci) * k + r) * k + s];
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    hi[i] = h;
    if (want_lo) lo[i] = __float2bfloat16_rn(v - __bfloat162float(h));
  }
}

__global__ void commit_fingerprint_kernel(unsigned long long* fp_new, unsigned long long* fp_old) {
  pdl_prologue();
  if (threadIdx.x < 2) { fp_old[threadIdx.x] = fp_new[threadIdx.x]; fp_new[threadIdx.x] = 0ull; }
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

// Encoded tensor maps are cached: a training step encodes the same few hundred (pointer, shape, box) combinations over and
// over (the workspace plan and the weight cache keep every operand at a fixed address), ~1 us of driver time each.
struct MapKey {
  const void* base; int d0, d1, d2, d3, b0, b1, b2, sample;
  bool operator==(const MapKey& o) const {
    return base == o.base && d0 == o.d0 && d1 == o.d1 && d2 == o.d2 && d3 == o.d3 && b0 == o.b0 && b1 == o.b1 && b2 == o.b2 && sample == o.sample;
  }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    size_t h = std::hash<const void*>()(k.base);
    for (int v : {k.d0, k.d1, k.d2, k.d3, k.b0, k.b1, k.b2, k.sample}) h = h * 1000003u ^ (size_t)v;
    return h;
  }
};
static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_maps;
static std::mutex g_maps_mu;

// `sample` = traversal stride in W and H (elementStrides): a box then spans box*sample input pixels and delivers every
// sample-th one, which is how a stride-2 convolution reads its input without a strided copy.
static int make_act_map(CUtensorMap* m, const void* base, int N, int H, int W, int C, int sample = 1) {
  const MapKey key = {base, C, W, H, N, TC_BLOCK_K, TC_SUB_W, TC_SUB_H, sample};
  {
    std::lock_guard<std::mutex> lk(g_maps_mu);
    auto it = g_maps.find(key);
    if (it != g_maps.end()) { *m = it->second; return 0; }
  }
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) { set_error("cuTensorMapEncodeTiled is unavailable (driver too old?)"); return DDN_EUNSUPPORTED; }
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  cuuint32_t box[4] = {(cuuint32_t)TC_BLOCK_K, (cuuint32_t)(TC_SUB_W * sample), (cuuint32_t)(TC_SUB_H * sample), 1};
  cuuint32_t es[4] = {1, (cuuint32_t)sample, (cuuint32_t)sample, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(activations) failed: %d", (int)r); return DDN_EINVAL; }
  std::lock_guard<std::mutex> lk(g_maps_mu);
  if (g_maps.size() > 8192) g_maps.clear();
  g_maps[key] = *m;
  return 0;
}
// Halo boxes of conv64_halo_kernel: the same NHWC planes with H and W swapped in the map, {c, h, w, n}, so that a box lands in
// shared memory as [w][h][64 c] (8 consecutive rows of a pixel column form one wgmma core-matrix group).
static int make_act_map_hw(CUtensorMap* m, const void* base, int N, int H, int W, int C, int box_h, int box_w) {
  const MapKey key = {base, C, H, W, N, TC_BLOCK_K, box_h, box_w, -2};
  {
    std::lock_guard<std::mutex> lk(g_maps_mu);
    auto it = g_maps.find(key);
    if (it != g_maps.end()) { *m = it->second; return 0; }
  }
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) { set_error("cuTensorMapEncodeTiled is unavailable (driver too old?)"); return DDN_EUNSUPPORTED; }
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)H, (cuuint64_t)W, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)W * C * 2, (cuuint64_t)C * 2, (cuuint64_t)H * W * C * 2};
  cuuint32_t box[4] = {(cuuint32_t)TC_BLOCK_K, (cuuint32_t)box_h, (cuuint32_t)box_w, 1};
  cuuint32_t es[4] = {1, 1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(halo activations) failed: %d", (int)r); return DDN_EINVAL; }
  std::lock_guard<std::mutex> lk(g_maps_mu);
  if (g_maps.size() > 8192) g_maps.clear();
  g_maps[key] = *m;
  return 0;
}
static int make_act_map_halo(CUtensorMap* m, const void* base, int N, int H, int W, int C) {
  return make_act_map_hw(m, base, N, H, W, C, HALO_BH, HALO_BW);
}
static int make_weight_map(CUtensorMap* m, const void* base, int rows, int K, int box_rows) {
  const MapKey key = {base, K, rows, 0, 0, TC_BLOCK_K, box_rows, 0, -1};
  {
    std::lock_guard<std::mutex> lk(g_maps_mu);
    auto it = g_maps.find(key);
    if (it != g_maps.end()) { *m = it->second; return 0; }
  }
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) { set_error("cuTensorMapEncodeTiled is unavailable (driver too old?)"); return DDN_EUNSUPPORTED; }
  cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)K * 2};
  cuuint32_t box[2] = {(cuuint32_t)TC_BLOCK_K, (cuuint32_t)box_rows};
  cuuint32_t es[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(weights) failed: %d", (int)r); return DDN_EINVAL; }
  std::lock_guard<std::mutex> lk(g_maps_mu);
  if (g_maps.size() > 8192) g_maps.clear();
  g_maps[key] = *m;
  return 0;
}

template <int BN, int NPROD>
static int launch_wgrad_tc(const CUtensorMap& dy_hi, const CUtensorMap& dy_lo, const CUtensorMap& x_hi, const CUtensorMap& x_lo,
                           const TcWgradParams& p, int workers, cudaStream_t st) {
  constexpr int NSPLIT = NPROD == 3 ? 2 : 1;
  constexpr int STAGE_BYTES = NSPLIT * (TC_A_BYTES + BN * TC_BLOCK_K * 2);
  constexpr int STAGES = (192 * 1024) / STAGE_BYTES >= 8 ? 8 : (192 * 1024) / STAGE_BYTES;
  const size_t smem = (size_t)STAGES * STAGE_BYTES + 1024;
  static bool configured = false;
  if (!configured) {
    DDN_CUDA(cudaFuncSetAttribute(wgrad_tc_kernel<BN, NPROD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = true;
  }
  DDN_LAUNCH((wgrad_tc_kernel<BN, NPROD>), workers, TC_WIDE_THREADS, smem, st, dy_hi, dy_lo, x_hi, x_lo, p);
  return 0;
}

// Pixel chunks of a weight gradient with `tiles` tiles over `total_kb` k-blocks on `workers` persistent CTAs: the smallest
// count S whose round-robin makespan is within 2 % of an even split of the work, else the one with the smallest makespan.
// The makespan is bounded by (items of the busiest CTA) x (longest chunk) = ceil(S * tiles / workers) * ceil(total_kb / S).
// Fewer chunks mean fewer fp64 reds of partial tiles; chunks keep at least 4 k-blocks.
static int tc_wgrad_chunks(int tiles, int total_kb, int workers) {
  const double even = (double)tiles * total_kb / workers;
  const int max_s = std::max(1, total_kb / 4);
  int best = 1;
  double best_span = 1e300;
  for (int s = 1; s <= max_s; ++s) {
    const double span = (double)ceil_div((int64_t)s * tiles, workers) * (double)ceil_div(total_kb, s);
    if (span <= 1.02 * even) return s;
    if (span < best_span) { best_span = span; best = s; }
  }
  return best;
}

// dwp[taps][Cout][Cin] += the weight gradient from the bf16 planes of x [N,H,W,Cin] and dy [N,Ho,Wo,Cout] (Ho = H/stride).
// dw != nullptr: dwp is scratch -- zero-filled here, converted to dw[Cout][Cin][k][k] (overwritten) afterwards.
// dw == nullptr: the caller zero-filled dwp and converts it later (tc_unpack_wgrads: one launch for many convs).
int tc_wgrad_planes(TcPlanes x, TcPlanes dy, float* dw, int N, int H, int W, int Cin, int Cout, int k, int stride, int dil,
                    int precision, double* dwp, cudaStream_t st) {
  const int want_lo = precision == DDN_PRECISION_BF16X3;
  const int taps = k * k;
  const int Ho = H / stride, Wo = W / stride;
  if (dw) DDN_TRY(launch_fill_zero(dwp, sizeof(double) * (size_t)taps * Cout * Cin, st));
  if (k == 3 && Cin == 64 && Cout == 64 && stride == 1 && dil == 1 && H % HALO_TH == 0 && W % HALO_TW == 0) {
    // layer1: one halo tile of X + one tile of dY per 8x16 pixels, every tap read in place (wgrad64_halo_kernel)
    TcWgradHaloParams hp;
    hp.dwp = dwp; hp.N = N; hp.H = H; hp.W = W; hp.tiles_h = H / HALO_TH; hp.tiles_w = W / HALO_TW; hp.n_tiles = N * hp.tiles_h * hp.tiles_w;
    CUtensorMap mx_hi, mx_lo, md_hi, md_lo;
    DDN_TRY(make_act_map_halo(&mx_hi, x.hi, N, H, W, 64));
    DDN_TRY(make_act_map_halo(&mx_lo, want_lo ? x.lo : x.hi, N, H, W, 64));
    DDN_TRY(make_act_map_hw(&md_hi, dy.hi, N, H, W, 64, HALO_TH, HALO_TW));
    DDN_TRY(make_act_map_hw(&md_lo, want_lo ? dy.lo : dy.hi, N, H, W, 64, HALO_TH, HALO_TW));
    const int nsplit = want_lo ? 2 : 1;
    const size_t smem = (size_t)2 * nsplit * (WGH_X_SLOT + WGH_DY_BYTES) + 1024;
    const int grid = std::min(hp.n_tiles, tc_worker_sms());
    {
      ProfScope ps(PROF_CONV_WGRAD_TC, 2.0 * N * H * W * 64.0 * 9 * 64, st);
      if (want_lo) {
        static bool configured = false;
        if (!configured) { DDN_CUDA(cudaFuncSetAttribute(wgrad64_halo_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); configured = true; }
        DDN_LAUNCH((wgrad64_halo_kernel<3>), grid, WGH_THREADS, smem, st, mx_hi, mx_lo, md_hi, md_lo, hp);
      } else {
        static bool configured = false;
        if (!configured) { DDN_CUDA(cudaFuncSetAttribute(wgrad64_halo_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); configured = true; }
        DDN_LAUNCH((wgrad64_halo_kernel<1>), grid, WGH_THREADS, smem, st, mx_hi, mx_lo, md_hi, md_lo, hp);
      }
    }
    if (dw) {
      int blocks = (int)std::min<int64_t>(ceil_div((int64_t)taps * Cout * Cin, 256), 4096);
      DDN_LAUNCH(unpack_wgrad_tc_kernel, blocks, 256, 0, st, dwp, dw, Cout, Cin, taps);
    }
    return 0;
  }
  const int bn = Cin % 128 == 0 ? 128 : 64;
  CUtensorMap m_dy_hi, m_dy_lo, m_x_hi, m_x_lo;
  DDN_TRY(make_act_map(&m_dy_hi, dy.hi, N, Ho, Wo, Cout));
  DDN_TRY(make_act_map(&m_dy_lo, want_lo ? dy.lo : dy.hi, N, Ho, Wo, Cout));
  DDN_TRY(make_act_map(&m_x_hi, x.hi, N, H, W, Cin, stride));
  DDN_TRY(make_act_map(&m_x_lo, want_lo ? x.lo : x.hi, N, H, W, Cin, stride));
  TcWgradParams p;
  p.dwp = dwp; p.N = N; p.H = Ho; p.W = Wo; p.Cin = Cin; p.Cout = Cout; p.taps_w = k; p.dil = dil; p.stride = stride;
  p.tiles_h = (int)ceil_div(Ho, TC_SUB_H); p.tiles_w = (int)ceil_div(Wo, TC_SUB_W);
  p.total_kb = N * p.tiles_h * p.tiles_w;
  p.n_co = (int)ceil_div(Cout, 128); p.n_ci = Cin / bn; p.n_tiles = p.n_co * p.n_ci * taps;
  const int sms = tc_worker_sms();
  p.chunks = tc_wgrad_chunks(p.n_tiles, p.total_kb, sms);
  const int workers = std::min(p.chunks * p.n_tiles, sms);
  const double fl = 2.0 * N * Ho * Wo * (double)Cout * taps * Cin;
  {
    ProfScope ps(PROF_CONV_WGRAD_TC, fl, st);
    if (bn == 128) DDN_TRY((want_lo ? launch_wgrad_tc<128, 3>(m_dy_hi, m_dy_lo, m_x_hi, m_x_lo, p, workers, st)
                                    : launch_wgrad_tc<128, 1>(m_dy_hi, m_dy_lo, m_x_hi, m_x_lo, p, workers, st)));
    else DDN_TRY((want_lo ? launch_wgrad_tc<64, 3>(m_dy_hi, m_dy_lo, m_x_hi, m_x_lo, p, workers, st)
                          : launch_wgrad_tc<64, 1>(m_dy_hi, m_dy_lo, m_x_hi, m_x_lo, p, workers, st)));
  }
  if (dw) {
    int blocks = (int)std::min<int64_t>(ceil_div((int64_t)taps * Cout * Cin, 256), 4096);
    DDN_LAUNCH(unpack_wgrad_tc_kernel, blocks, 256, 0, st, dwp, dw, Cout, Cin, taps);
  }
  return 0;
}

int tc_unpack_wgrads(const TcUnpackEntry* entries, int n, const double* dwp_base, float* grads_base, cudaStream_t st) {
  for (int i0 = 0; i0 < n; i0 += TC_UNPACK_MAX) {
    TcUnpackTable t; t.n = std::min(TC_UNPACK_MAX, n - i0);
    int64_t biggest = 0;
    for (int i = 0; i < t.n; ++i) { t.e[i] = entries[i0 + i]; biggest = std::max<int64_t>(biggest, (int64_t)t.e[i].Cout * t.e[i].Cin * t.e[i].taps); }
    dim3 grid((unsigned)std::min<int64_t>(ceil_div(biggest, 256 * 4), 1024), (unsigned)t.n);
    DDN_LAUNCH(unpack_wgrad_batched_kernel, grid, 256, 0, st, dwp_base, grads_base, t);
  }
  return 0;
}

// forward / weight-gradient coverage: 3x3 (pad == dil) or 1x1 (pad 0), stride 1 -- or stride 2 with dil 1 on even sizes
bool tc_conv_supported(int Cin, int Cout, int k, int stride, int pad, int dil, int H, int W) {
  if (Cin % 64 || Cout % 64) return false;
  if (stride == 2) { if (dil != 1 || (H & 1) || (W & 1)) return false; }
  else if (stride != 1) return false;
  if (k == 3) return pad == dil;
  if (k == 1) return pad == 0;
  return false;
}

static const size_t kMaxWeightElems = (size_t)9 * 512 * 512;
size_t tc_max_weight_elems() { return kMaxWeightElems; }
size_t tc_weight_ws_bytes() { return 2 * align_up(kMaxWeightElems * 2, 1024) + 2048; }

int tc_split(const float* x, __nv_bfloat16* hi, __nv_bfloat16* lo, int64_t n, int precision, cudaStream_t st) {
  DDN_CHECK_ARG(n % 4 == 0, "split: element count must be a multiple of 4");
  int64_t n4 = n / 4;
  int blocks = (int)std::min<int64_t>(ceil_div(n4, 256), (int64_t)num_sms() * 8);
  DDN_LAUNCH(split_bf16_kernel, blocks, 256, 0, st, x, hi, lo, n4, precision == DDN_PRECISION_BF16X3 ? 1 : 0);
  return 0;
}

int tc_upsample_zero_split(const float* dy, __nv_bfloat16* hi, __nv_bfloat16* lo, int N, int Ho, int Wo, int C, int precision,
                           cudaStream_t st) {
  int64_t total = (int64_t)N * Ho * Wo * (C / 4);
  int blocks = (int)std::min<int64_t>(ceil_div(total, 256), (int64_t)num_sms() * 8);
  DDN_LAUNCH(upsample_zero_split_kernel, blocks, 256, 0, st, dy, hi, lo, N, Ho, Wo, C, precision == DDN_PRECISION_BF16X3 ? 1 : 0);
  return 0;
}

int tc_stem_patches(const float* x_nchw, __nv_bfloat16* hi, __nv_bfloat16* lo, int N, int H, int W, int precision, cudaStream_t st) {
  const int H1 = (H - 1) / 2 + 1, W1 = (W - 1) / 2 + 1;
  DDN_CHECK_ARG(N <= 65535 && H1 <= 65535, "stem: batch / height too large for the launch grid");
  dim3 grid((unsigned)ceil_div(W1, STEM_TW), (unsigned)H1, (unsigned)N);
  DDN_LAUNCH(stem_patch_split_kernel, grid, 256, 0, st, x_nchw, hi, lo, N, H, W, H1, W1, precision == DDN_PRECISION_BF16X3 ? 1 : 0);
  return 0;
}

template <int BLOCK_N, int NPROD>
static int launch_conv_tc(const CUtensorMap& a_hi, const CUtensorMap& a_lo, const CUtensorMap& b_hi, const CUtensorMap& b_lo,
                          const CUtensorMap& bt_hi, const CUtensorMap& bt_lo, const TcConvParams& p, int workers, cudaStream_t st) {
  constexpr int NSPLIT = NPROD == 3 ? 2 : 1;
  constexpr int STAGE_BYTES = NSPLIT * (128 * TC_BLOCK_K * 2 + BLOCK_N * TC_BLOCK_K * 2);
  constexpr int STAGES = (192 * 1024) / STAGE_BYTES >= 8 ? 8 : (192 * 1024) / STAGE_BYTES;
  const size_t smem = (size_t)STAGES * STAGE_BYTES + 1024;
  static bool configured = false;
  if (!configured) {
    DDN_CUDA(cudaFuncSetAttribute(conv_tc_kernel<BLOCK_N, NPROD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = true;
  }
  DDN_LAUNCH((conv_tc_kernel<BLOCK_N, NPROD>), workers, TC_WIDE_THREADS, smem, st, a_hi, a_lo, b_hi, b_lo, bt_hi, bt_lo, p);
  return 0;
}

template <int NPROD>
static int launch_conv64_halo(const CUtensorMap& a_hi, const CUtensorMap& a_lo, const CUtensorMap& b_hi, const CUtensorMap& b_lo,
                              const TcHaloParams& p, cudaStream_t st) {
  constexpr int NSPLIT = NPROD == 3 ? 2 : 1;
  const size_t smem = (size_t)NSPLIT * HALO_B_PLANE + (size_t)halo_slots(NPROD) * HALO_SLOT + 1024;
  static bool configured = false;
  if (!configured) {
    DDN_CUDA(cudaFuncSetAttribute(conv64_halo_kernel<NPROD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = true;
  }
  const int grid = std::min(p.n_tiles, tc_worker_sms());
  DDN_LAUNCH((conv64_halo_kernel<NPROD>), grid, TC_THREADS, smem, st, a_hi, a_lo, b_hi, b_lo, p);
  return 0;
}

// The epilogue request of one conv, for either kernel: `out` (+ `addend`) and at most one of the forward BatchNorm statistics
// (`stats`), the data gradient's BatchNorm-backward column sums (`bst`) and the folded inference epilogue (`ep`).  A
// BatchNorm request covers the gout channels the conv writes.
static int tc_epilogue_request(TcEpilogueParams* e, float* out, const float* addend, const BnFwdFinal* stats, const TcBwdStats* bst,
                               const TcFoldedEpilogue* ep, int N, int gout, int dgrad, int want_lo) {
  memset(e, 0, sizeof(*e));
  e->out = out; e->addend = addend; e->imgs_per_group = N;
  if (stats) {
    DDN_CHECK_ARG(!dgrad && !ep && stats->G >= 1 && stats->G <= BN_MAX_GROUPS && N % stats->G == 0 && stats->C == gout,
                  "bad BatchNorm statistics request");
    e->fin = *stats;
    e->imgs_per_group = N / stats->G;
  }
  if (bst) {
    DDN_CHECK_ARG(dgrad && !ep && !stats && bst->raw && bst->mean && bst->invstd && bst->fin.a.acc && bst->fin.G >= 1 &&
                  bst->fin.G <= BN_MAX_GROUPS && N % bst->fin.G == 0 && bst->fin.C == gout && (bst->y_hi || !bst->relu || (bst->gamma && bst->beta)),
                  "bad BatchNorm backward-statistics request");
    e->bst = *bst;
    e->imgs_per_group = N / bst->fin.G;
  }
  if (ep) {
    DDN_CHECK_ARG(!dgrad && !stats && !bst && ep->scale && ep->shift && (out || ep->out_hi), "folded epilogue: forward only, needs scale/shift and an output");
    e->ep_scale = ep->scale; e->ep_shift = ep->shift; e->ep_relu = ep->relu; e->out_hi = ep->out_hi; e->out_lo = want_lo ? ep->out_lo : nullptr;
  } else {
    DDN_CHECK_ARG(out != nullptr, "conv output pointer is null");
  }
  return 0;
}

// out[N,Ho,Wo,gout] = conv(planes of in[N,H,W,gin]) (+ addend).
//   dgrad = 0: forward (gin = Cin, gout = Cout, Ho = H/stride).
//   dgrad = 1: data gradient, stride 1 only (`in` = dY planes with Cout channels, out = dX with Cin channels; Cin/Cout are
//              those of the ORIGINAL conv).
//   wpk != nullptr: weights are already packed [gout][k*k*gin] bf16 hi/lo; else they are packed from w_oihw into `wws`.
//   stats (forward only): per-channel sum / sum of squares of the output go to stats->a, and the kernel's last CTA writes
//              the BatchNorm statistics described by *stats; groups = BatchNorm groups in the batch.
//   bst (data gradient only): the gradient written to `out` is the dY of a BatchNorm whose column sums (sum g, sum g*xhat,
//              g = dY * relu mask) are accumulated by the epilogue; the last CTA finalizes them like bn_colsum_kernel<1>.
int tc_conv_planes(TcPlanes in, const float* w_oihw, const TcPlanes* wpk, float* out, const float* addend, const BnFwdFinal* stats,
                   int N, int H, int W, int Cin, int Cout, int k, int stride, int dil, int dgrad, int precision,
                   void* wws, size_t wws_bytes, cudaStream_t st, const TcFoldedEpilogue* ep, const TcBwdStats* bst) {
  DDN_CHECK_ARG(stride == 1 || !dgrad, "the strided data gradient goes through zero-inserted planes (stride 1 here)");
  const int Ho = H / stride, Wo = W / stride;
  const double fl = 2.0 * N * Ho * Wo * (double)Cout * k * k * Cin;
  const int gin = dgrad ? Cout : Cin, gout = dgrad ? Cin : Cout;
  const int want_lo = precision == DDN_PRECISION_BF16X3;
  TcEpilogueParams epi;
  DDN_TRY(tc_epilogue_request(&epi, out, addend, stats, bst, ep, N, gout, dgrad, want_lo));
  const __nv_bfloat16* b_hi; const __nv_bfloat16* b_lo;
  if (wpk) {
    b_hi = wpk->hi; b_lo = wpk->lo;
  } else {
    const size_t wel = (size_t)Cout * Cin * k * k;
    const size_t w_b = align_up(kMaxWeightElems * 2, 1024);
    DDN_CHECK_ARG(wws != nullptr && wel <= kMaxWeightElems, "tc weight staging missing or weight tensor too large");
    char* base = reinterpret_cast<char*>(align_up(reinterpret_cast<uintptr_t>(wws), 1024));
    if ((size_t)(base - (char*)wws) + 2 * w_b > wws_bytes) { set_error("tensor-core weight staging too small"); return DDN_EWORKSPACE; }
    __nv_bfloat16* ph = (__nv_bfloat16*)base; __nv_bfloat16* pl = (__nv_bfloat16*)(base + w_b);
    int wblocks = (int)std::min<int64_t>(ceil_div((int64_t)wel, 256), 4096);
    DDN_LAUNCH(pack_weights_tc_kernel, wblocks, 256, 0, st, w_oihw, ph, pl, Cout, Cin, k, dgrad, want_lo);
    b_hi = ph; b_lo = pl;
  }
  if (k == 3 && gin == 64 && gout == 64 && stride == 1 && dil == 1 && Ho % HALO_TH == 0 && Wo % HALO_TW == 0) {
    // 64 -> 64 channels (layer1): resident weights + one halo tile per 8x16 output pixels (conv64_halo_kernel)
    TcHaloParams hp;
    memset(&hp, 0, sizeof(hp));
    hp.epi = epi; hp.N = N; hp.H = Ho; hp.W = Wo;
    hp.tiles_h = Ho / HALO_TH; hp.tiles_w = Wo / HALO_TW; hp.n_tiles = N * hp.tiles_h * hp.tiles_w;
    CUtensorMap ma_hi, ma_lo, mb_hi, mb_lo;
    DDN_TRY(make_act_map_halo(&ma_hi, in.hi, N, H, W, 64));
    DDN_TRY(make_act_map_halo(&ma_lo, want_lo ? in.lo : in.hi, N, H, W, 64));
    DDN_TRY(make_weight_map(&mb_hi, b_hi, 64, 9 * 64, 64));
    DDN_TRY(make_weight_map(&mb_lo, want_lo ? b_lo : b_hi, 64, 9 * 64, 64));
    ProfScope ps(dgrad ? PROF_CONV_DGRAD_TC : PROF_CONV_FWD_TC, fl, st);
    return want_lo ? launch_conv64_halo<3>(ma_hi, ma_lo, mb_hi, mb_lo, hp, st) : launch_conv64_halo<1>(ma_hi, ma_lo, mb_hi, mb_lo, hp, st);
  }
  const int block_n = gout % 128 == 0 ? 128 : 64;
  TcConvParams p;
  memset(&p, 0, sizeof(p));
  p.epi = epi; p.N = N; p.H = Ho; p.W = Wo; p.Cin = gin; p.Cout = gout; p.taps_w = k; p.dil = dil;
  p.stride = stride;
  p.tiles_h = (int)ceil_div(Ho, TC_SUB_H); p.tiles_w = (int)ceil_div(Wo, TC_SUB_W);
  p.n_sub = N * p.tiles_h * p.tiles_w;
  p.n_co = gout / block_n;
  const int tiles = (int)ceil_div(p.n_sub, 2) * p.n_co;
  const int workers_max = tc_worker_sms();
  // the tiles of the last, partial wave are cut along N so that the tail costs a fraction of a tile time
  const int rem = tiles % workers_max;
  int split = 1;
  if (rem)
    while (split * 2 <= 8 && block_n / (split * 2) >= 32 && rem * split * 2 <= workers_max) split *= 2;
  p.full_items = tiles - rem; p.tail_split = split; p.total_items = p.full_items + rem * split;
  if (split == 1) { p.full_items = tiles; p.total_items = tiles; }
  const int workers = std::min(p.total_items, workers_max);
  const int b_rows = block_n;
  const int bt_rows = b_rows / split;
  CUtensorMap ma_hi, ma_lo, mb_hi, mb_lo, mt_hi, mt_lo;
  DDN_TRY(make_act_map(&ma_hi, in.hi, N, H, W, gin, stride));
  DDN_TRY(make_act_map(&ma_lo, want_lo ? in.lo : in.hi, N, H, W, gin, stride));
  DDN_TRY(make_weight_map(&mb_hi, b_hi, gout, k * k * gin, b_rows));
  DDN_TRY(make_weight_map(&mb_lo, want_lo ? b_lo : b_hi, gout, k * k * gin, b_rows));
  DDN_TRY(make_weight_map(&mt_hi, b_hi, gout, k * k * gin, bt_rows));
  DDN_TRY(make_weight_map(&mt_lo, want_lo ? b_lo : b_hi, gout, k * k * gin, bt_rows));
  ProfScope ps(dgrad ? PROF_CONV_DGRAD_TC : PROF_CONV_FWD_TC, fl, st);   // times the MMA kernel only
#define CONV_TC(BN)                                                                                                           \
  (want_lo ? launch_conv_tc<BN, 3>(ma_hi, ma_lo, mb_hi, mb_lo, mt_hi, mt_lo, p, workers, st)                                   \
           : launch_conv_tc<BN, 1>(ma_hi, ma_lo, mb_hi, mb_lo, mt_hi, mt_lo, p, workers, st))
  if (block_n == 128) return CONV_TC(128);
  return CONV_TC(64);
#undef CONV_TC
}

// data gradient of a stride-2 conv: zero-insert dY [N,H/2,W/2,Cout] into `up` planes [N,H,W,Cout], then a stride-1 dgrad
int tc_dgrad_strided(const float* dy_f32, TcPlanes up, const float* w_oihw, const TcPlanes* w_packed, float* dx, const float* addend,
                     int N, int H, int W, int Cin, int Cout, int k, int precision, void* wws, size_t wws_bytes, cudaStream_t st,
                     const TcBwdStats* bst) {
  DDN_TRY(tc_upsample_zero_split(dy_f32, const_cast<__nv_bfloat16*>(up.hi), const_cast<__nv_bfloat16*>(up.lo), N, H / 2, W / 2, Cout,
                                 precision, st));
  return tc_conv_planes(up, w_oihw, w_packed, dx, addend, nullptr, N, H, W, Cin, Cout, k, 1, 1, 1, precision, wws, wws_bytes, st, nullptr, bst);
}

// ---- stem (conv1 7x7/2, Cin = 3) as a K = 192 GEMM over patch planes
int tc_stem_pack_weights(const float* w_conv1, __nv_bfloat16* hi, __nv_bfloat16* lo, int precision, cudaStream_t st) {
  DDN_LAUNCH(stem_pack_weights_kernel, (64 * 192 + 255) / 256, 256, 0, st, w_conv1, hi, lo, precision == DDN_PRECISION_BF16X3 ? 1 : 0);
  return 0;
}
int tc_stem_forward(TcPlanes patches, const float* w_conv1, const TcPlanes* w_packed, float* raw, const BnFwdFinal* stats, int N, int H1,
                    int W1, int precision, void* wws, size_t wws_bytes, cudaStream_t st) {
  TcPlanes wpk;
  if (w_packed) wpk = *w_packed;
  else {
    char* base = reinterpret_cast<char*>(align_up(reinterpret_cast<uintptr_t>(wws), 1024));
    DDN_CHECK_ARG((size_t)(base - (char*)wws) + 2 * 64 * 192 * 2 + 1024 <= wws_bytes, "weight staging too small");
    __nv_bfloat16* ph = (__nv_bfloat16*)base; __nv_bfloat16* pl = (__nv_bfloat16*)(base + align_up((size_t)64 * 192 * 2, 1024));
    DDN_TRY(tc_stem_pack_weights(w_conv1, ph, pl, precision, st));
    wpk.hi = ph; wpk.lo = pl;
  }
  return tc_conv_planes(patches, nullptr, &wpk, raw, nullptr, stats, N, H1, W1, 192, 64, 1, 1, 1, 0, precision, wws, wws_bytes, st);
}

// d conv1.weight from the patch planes and the planes of d(raw stem output), accumulated into the pre-zeroed fp64 [64][192]
// `dwp`, which tc_unpack_wgrads converts to [64][3][7][7] (a kind-1 entry).
int tc_stem_wgrad(TcPlanes patches, TcPlanes dy, int N, int H1, int W1, int precision, double* dwp, cudaStream_t st) {
  return tc_wgrad_planes(patches, dy, nullptr, N, H1, W1, 192, 64, 1, 1, 1, precision, dwp, st);
}

// (re)packs every table entry into `cache` when the device-side fingerprint of params[0..n_params) differs from the one
// stored at `fp_old` (or `force`): three launches, no host synchronisation.  fp_new / fp_old: 2 x uint64 each, fp_new zero.
int tc_pack_all(const float* params, int64_t n_params, char* cache, const TcPackEntry* entries, int n, unsigned long long* fp_new,
                unsigned long long* fp_old, int force, int precision, cudaStream_t st) {
  DDN_CHECK_ARG(n >= 1, "empty pack table");
  DDN_LAUNCH(param_fingerprint_kernel, num_sms() * 2, 256, 0, st, reinterpret_cast<const uint32_t*>(params), n_params, fp_new);
  for (int i0 = 0; i0 < n; i0 += TC_PACK_MAX) {     // a table longer than one launch's parameter block: one launch per slice
    TcPackTable t; t.n = std::min(TC_PACK_MAX, n - i0);
    for (int i = 0; i < t.n; ++i) t.e[i] = entries[i0 + i];
    dim3 grid(32, (unsigned)t.n);
    DDN_LAUNCH(pack_all_kernel, grid, 256, 0, st, params, cache, t, fp_new, fp_old, force, precision == DDN_PRECISION_BF16X3 ? 1 : 0);
  }
  DDN_LAUNCH(commit_fingerprint_kernel, 1, 32, 0, st, fp_new, fp_old);
  return 0;
}

// ---- fp32-tensor wrappers (single-operator C ABI): split into the staging region, then run the plane kernels
// staging layout: [weights hi|lo][x hi|lo][dy hi|lo][zero-inserted dy hi|lo (stride 2 only)]
size_t tc_workspace_bytes(size_t max_act_elems) { return tc_weight_ws_bytes() + 6 * align_up(max_act_elems * 2, 1024) + 4096; }

int stage_planes(void* ws, size_t ws_bytes, size_t x_el, size_t dy_el, size_t up_el, void** wws, TcPlanes* x, TcPlanes* dy,
                 TcPlanes* up) {
  char* base = reinterpret_cast<char*>(align_up(reinterpret_cast<uintptr_t>(ws), 1024));
  const size_t wb = align_up(tc_weight_ws_bytes(), 1024), xb = align_up(x_el * 2, 1024), yb = align_up(dy_el * 2, 1024),
               ub = align_up(up_el * 2, 1024);
  if ((size_t)(base - (char*)ws) + wb + 2 * xb + 2 * yb + 2 * ub > ws_bytes) { set_error("tensor-core staging workspace too small"); return DDN_EWORKSPACE; }
  *wws = base;
  char* q = base + wb;
  x->hi = (__nv_bfloat16*)q; x->lo = (__nv_bfloat16*)(q + xb);
  dy->hi = (__nv_bfloat16*)(q + 2 * xb); dy->lo = (__nv_bfloat16*)(q + 2 * xb + yb);
  up->hi = (__nv_bfloat16*)(q + 2 * xb + 2 * yb); up->lo = (__nv_bfloat16*)(q + 2 * xb + 2 * yb + ub);
  return 0;
}

int tc_conv_forward(const float* x, const float* w, float* y, int N, int H, int W, int Cin, int Cout, int k, int stride, int pad, int dil,
                    int precision, void* ws, size_t ws_bytes, cudaStream_t st) {
  (void)pad;
  void* wws; TcPlanes px, pdy, pup;
  DDN_TRY(stage_planes(ws, ws_bytes, (size_t)N * H * W * Cin, 0, 0, &wws, &px, &pdy, &pup));
  DDN_TRY(tc_split(x, const_cast<__nv_bfloat16*>(px.hi), const_cast<__nv_bfloat16*>(px.lo), (int64_t)N * H * W * Cin, precision, st));
  return tc_conv_planes(px, w, nullptr, y, nullptr, nullptr, N, H, W, Cin, Cout, k, stride, dil, 0, precision, wws, tc_weight_ws_bytes(), st);
}

int tc_conv_backward(const float* x, const float* w, const float* dy, float* dx, const float* dx_addend, float* dw,
                     int N, int H, int W, int Cin, int Cout, int k, int stride, int pad, int dil, int precision,
                     void* ws, size_t ws_bytes, double* dwp_scratch, cudaStream_t st) {
  (void)pad;
  const int Ho = H / stride, Wo = W / stride;
  void* wws; TcPlanes px, pdy, pup;
  DDN_TRY(stage_planes(ws, ws_bytes, (size_t)N * H * W * Cin, (size_t)N * Ho * Wo * Cout, stride == 2 ? (size_t)N * H * W * Cout : 0,
                       &wws, &px, &pdy, &pup));
  DDN_TRY(tc_split(x, const_cast<__nv_bfloat16*>(px.hi), const_cast<__nv_bfloat16*>(px.lo), (int64_t)N * H * W * Cin, precision, st));
  DDN_TRY(tc_split(dy, const_cast<__nv_bfloat16*>(pdy.hi), const_cast<__nv_bfloat16*>(pdy.lo), (int64_t)N * Ho * Wo * Cout, precision, st));
  DDN_TRY(tc_wgrad_planes(px, pdy, dw, N, H, W, Cin, Cout, k, stride, dil, precision, dwp_scratch, st));
  if (dx) {
    if (stride == 2)
      DDN_TRY(tc_dgrad_strided(dy, pup, w, nullptr, dx, dx_addend, N, H, W, Cin, Cout, k, precision, wws, tc_weight_ws_bytes(), st));
    else
      DDN_TRY(tc_conv_planes(pdy, w, nullptr, dx, dx_addend, nullptr, N, H, W, Cin, Cout, k, 1, dil, 1, precision, wws, tc_weight_ws_bytes(), st));
  }
  return 0;
}

}  // namespace ddn
