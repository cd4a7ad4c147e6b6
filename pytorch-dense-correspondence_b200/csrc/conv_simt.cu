// fp32 implicit-GEMM convolution on CUDA cores (DDN_PRECISION_FP32_SIMT), NHWC activations.
//
// One "gather-form" kernel serves forward and data-gradient:
//     out[n,ho,wo,co] = sum_{r,s,ci} in[n, (ho*S - pad + r*dil)/U, (wo*S - pad + s*dil)/U, ci] * Wp[(r,s,ci), co]
// (terms whose numerator is negative, not divisible by U, or past the edge are zero).  Forward uses
// U=1; the data gradient of a stride-S conv uses S=1, U=stride, flipped/transposed weights and
// pad' = dil*(k-1) - pad.  The weight-gradient kernel contracts the same gathered operand against dY.
//
// These kernels are the exact-fp32 class of the oracle (cuDNN/MKLDNN fp32 in the reference:
// nn.Conv2d at PSD/vision/torchvision/models/resnet.py:36,136,210); they also carry the convs the
// tensor-core path does not cover (7x7/2 stem with Cin=3, the two stride-2 convs of layer2).
#include "conv.cuh"

namespace ddn {

// ------------------------------------------------------------------------------------------------
// weight repacking
// w [Cout][Cin][KH][KW]  ->  fwd:   wp[(r*KW+s)*CinP + ci][Cout]
//                           dgrad:  wp[(r*KW+s)*Cout + co][CinP]  with (r,s) flipped
__global__ void pack_weights_kernel(const float* __restrict__ w, float* __restrict__ wp,
                                    int Cout, int Cin, int CinP, int KH, int KW, int dgrad) {
  pdl_prologue();
  int64_t total = dgrad ? (int64_t)KH * KW * Cout * CinP : (int64_t)KH * KW * CinP * Cout;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int co, ci, r, s;
    if (!dgrad) {
      co = (int)(i % Cout); int64_t q = i / Cout;
      ci = (int)(q % CinP); q /= CinP;
      s = (int)(q % KW); r = (int)(q / KW);
    } else {
      ci = (int)(i % CinP); int64_t q = i / CinP;
      co = (int)(q % Cout); q /= Cout;
      s = KW - 1 - (int)(q % KW); r = KH - 1 - (int)(q / KW);
    }
    float v = 0.f;
    if (ci < Cin) v = w[(((int64_t)co * Cin + ci) * KH + r) * KW + s];
    wp[i] = v;
  }
}

// dwp[(r*KW+s)*CinP + ci][Cout] -> dw[Cout][Cin][KH][KW]
__global__ void unpack_wgrad_kernel(const float* __restrict__ dwp, float* __restrict__ dw,
                                    int Cout, int Cin, int CinP, int KH, int KW) {
  pdl_prologue();
  int64_t total = (int64_t)Cout * Cin * KH * KW;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int s = (int)(i % KW); int64_t q = i / KW;
    int r = (int)(q % KH); q /= KH;
    int ci = (int)(q % Cin); int co = (int)(q / Cin);
    dw[i] = dwp[((int64_t)(r * KW + s) * CinP + ci) * Cout + co];
  }
}

// ------------------------------------------------------------------------------------------------
// gather-form conv:  C[M = N*Ho*Wo][Cout] = A[M][K = KH*KW*Cin] * Wp[K][Cout]  (+ addend)
template <int BM, int BN, int BK, int TM, int TN>
__global__ void __launch_bounds__((BM / TM) * (BN / TN))
conv_gather_f32_kernel(const float* __restrict__ in, const float* __restrict__ wp, const float* __restrict__ addend,
                       float* __restrict__ out, ConvGeom g) {
  pdl_prologue();
  constexpr int THREADS = (BM / TM) * (BN / TN);
  constexpr int A_F4 = BM * BK / 4;            // float4 loads per A tile
  constexpr int B_F4 = BK * BN / 4;
  constexpr int A_PER_T = A_F4 / THREADS;
  constexpr int B_PER_T = B_F4 / THREADS;
  static_assert(A_F4 % THREADS == 0 && B_F4 % THREADS == 0, "tile/threads mismatch");
  constexpr int KQ = BK / 4;                   // float4 columns per A row
  __shared__ __align__(16) float As[2][BK][BM + 4];
  __shared__ __align__(16) float Bs[2][BK][BN];

  const int tid = threadIdx.x;
  const int64_t M = (int64_t)g.N * g.Hout * g.Wout;
  const int K = g.KH * g.KW * g.Cin;
  const int64_t m0 = (int64_t)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;

  // per-thread A-load rows: fixed across the k loop
  int a_row[A_PER_T], a_kq[A_PER_T], a_hb[A_PER_T], a_wb[A_PER_T];
  const float* a_base[A_PER_T];
  bool a_ok[A_PER_T];
#pragma unroll
  for (int i = 0; i < A_PER_T; ++i) {
    int f = tid + i * THREADS;
    a_row[i] = f / KQ;
    a_kq[i] = (f % KQ) * 4;
    int64_t m = m0 + a_row[i];
    a_ok[i] = m < M;
    int64_t mm = a_ok[i] ? m : 0;
    int wo = (int)(mm % g.Wout); int64_t q = mm / g.Wout;
    int ho = (int)(q % g.Hout); int n = (int)(q / g.Hout);
    a_hb[i] = ho * g.stride - g.pad;
    a_wb[i] = wo * g.stride - g.pad;
    a_base[i] = in + (int64_t)n * g.Hin * g.Win * g.Cin;
  }
  const int cin_shift = g.cin_log2;

  float4 a_reg[A_PER_T], b_reg[B_PER_T];
  auto load_tiles = [&](int k0) {
#pragma unroll
    for (int i = 0; i < A_PER_T; ++i) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      int k = k0 + a_kq[i];
      if (a_ok[i] && k < K) {
        int tap = k >> cin_shift;
        int ci = k & (g.Cin - 1);
        int r = tap / g.KW, s = tap - r * g.KW;
        int hn = a_hb[i] + r * g.dil, wn = a_wb[i] + s * g.dil;
        bool ok = hn >= 0 && wn >= 0;
        int hi = hn, wi = wn;
        if (g.ups > 1) {
          ok = ok && (hn % g.ups == 0) && (wn % g.ups == 0);
          hi = hn / g.ups; wi = wn / g.ups;
        }
        ok = ok && hi < g.Hin && wi < g.Win;
        if (ok) v = __ldg(reinterpret_cast<const float4*>(a_base[i] + ((int64_t)hi * g.Win + wi) * g.Cin + ci));
      }
      a_reg[i] = v;
    }
#pragma unroll
    for (int i = 0; i < B_PER_T; ++i) {
      int f = tid + i * THREADS;
      int kr = f / (BN / 4), c4 = (f % (BN / 4)) * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (k0 + kr < K) v = __ldg(reinterpret_cast<const float4*>(wp + (int64_t)(k0 + kr) * g.Cout + n0 + c4));
      b_reg[i] = v;
    }
  };
  auto store_tiles = [&](int buf) {
#pragma unroll
    for (int i = 0; i < A_PER_T; ++i) {
      As[buf][a_kq[i] + 0][a_row[i]] = a_reg[i].x;
      As[buf][a_kq[i] + 1][a_row[i]] = a_reg[i].y;
      As[buf][a_kq[i] + 2][a_row[i]] = a_reg[i].z;
      As[buf][a_kq[i] + 3][a_row[i]] = a_reg[i].w;
    }
#pragma unroll
    for (int i = 0; i < B_PER_T; ++i) {
      int f = tid + i * THREADS;
      int kr = f / (BN / 4), c4 = (f % (BN / 4)) * 4;
      *reinterpret_cast<float4*>(&Bs[buf][kr][c4]) = b_reg[i];
    }
  };

  const int tx = tid % (BN / TN), ty = tid / (BN / TN);
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  const int nk = (K + BK - 1) / BK;
  load_tiles(0);
  store_tiles(0);
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    int buf = kt & 1;
    if (kt + 1 < nk) load_tiles((kt + 1) * BK);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; i += 4) {
        float4 v = *reinterpret_cast<const float4*>(&As[buf][kk][ty * TM + i]);
        a[i] = v.x; a[i + 1] = v.y; a[i + 2] = v.z; a[i + 3] = v.w;
      }
#pragma unroll
      for (int j = 0; j < TN; j += 4) {
        float4 v = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * TN + j]);
        b[j] = v.x; b[j + 1] = v.y; b[j + 2] = v.z; b[j + 3] = v.w;
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < nk) {
      store_tiles(buf ^ 1);
      __syncthreads();
    }
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    int64_t m = m0 + ty * TM + i;
    if (m >= M) continue;
    float* o = out + m * g.Cout + n0 + tx * TN;
#pragma unroll
    for (int j = 0; j < TN; j += 4) {
      float4 v = make_float4(acc[i][j], acc[i][j + 1], acc[i][j + 2], acc[i][j + 3]);
      if (addend) {
        float4 ad = __ldg(reinterpret_cast<const float4*>(addend + m * g.Cout + n0 + tx * TN + j));
        v.x += ad.x; v.y += ad.y; v.z += ad.z; v.w += ad.w;
      }
      *reinterpret_cast<float4*>(o + j) = v;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// weight gradient:  dWp[K][Cout] += sum_{m in split} A[m][K]^T * dY[m][Cout]      (fp32 atomics across splits)
template <int BKR, int BN, int BP, int TM, int TN>   // BKR rows of K, BN cols of Cout, BP pixels per step
__global__ void __launch_bounds__((BKR / TM) * (BN / TN))
conv_wgrad_f32_kernel(const float* __restrict__ in, const float* __restrict__ dy, float* __restrict__ dwp,
                      ConvGeom g, int pixels_per_split) {
  pdl_prologue();
  constexpr int THREADS = (BKR / TM) * (BN / TN);
  constexpr int A_F4 = BP * BKR / 4, B_F4 = BP * BN / 4;
  constexpr int A_PER_T = A_F4 / THREADS, B_PER_T = B_F4 / THREADS;
  static_assert(A_F4 % THREADS == 0 && B_F4 % THREADS == 0, "tile/threads mismatch");
  __shared__ __align__(16) float As[2][BP][BKR];
  __shared__ __align__(16) float Bs[2][BP][BN];

  const int tid = threadIdx.x;
  const int64_t M = (int64_t)g.N * g.Hout * g.Wout;
  const int K = g.KH * g.KW * g.Cin;
  const int k0 = blockIdx.x * BKR;
  const int n0 = blockIdx.y * BN;
  const int64_t m_begin = (int64_t)blockIdx.z * pixels_per_split;
  const int64_t m_end = min(M, m_begin + pixels_per_split);
  if (m_begin >= m_end) return;

  // A loads: thread -> (pixel slot, k quad); the k quad (tap, ci) is fixed across the pixel loop
  int a_p[A_PER_T], a_k[A_PER_T], a_r[A_PER_T], a_s[A_PER_T], a_ci[A_PER_T];
  bool a_kok[A_PER_T];
#pragma unroll
  for (int i = 0; i < A_PER_T; ++i) {
    int f = tid + i * THREADS;
    a_p[i] = f / (BKR / 4);
    a_k[i] = (f % (BKR / 4)) * 4;
    int k = k0 + a_k[i];
    a_kok[i] = k < K;
    int kk = a_kok[i] ? k : 0;
    int tap = kk >> g.cin_log2;
    a_ci[i] = kk & (g.Cin - 1);
    a_r[i] = tap / g.KW; a_s[i] = tap - a_r[i] * g.KW;
  }
  float4 a_reg[A_PER_T], b_reg[B_PER_T];
  auto load_tiles = [&](int64_t mb) {
#pragma unroll
    for (int i = 0; i < A_PER_T; ++i) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      int64_t m = mb + a_p[i];
      if (a_kok[i] && m < m_end) {
        int wo = (int)(m % g.Wout); int64_t q = m / g.Wout;
        int ho = (int)(q % g.Hout); int n = (int)(q / g.Hout);
        int hn = ho * g.stride - g.pad + a_r[i] * g.dil, wn = wo * g.stride - g.pad + a_s[i] * g.dil;
        if (hn >= 0 && wn >= 0 && hn < g.Hin && wn < g.Win)
          v = __ldg(reinterpret_cast<const float4*>(in + (((int64_t)n * g.Hin + hn) * g.Win + wn) * g.Cin + a_ci[i]));
      }
      a_reg[i] = v;
    }
#pragma unroll
    for (int i = 0; i < B_PER_T; ++i) {
      int f = tid + i * THREADS;
      int p = f / (BN / 4), c4 = (f % (BN / 4)) * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      int64_t m = mb + p;
      if (m < m_end) v = __ldg(reinterpret_cast<const float4*>(dy + m * g.Cout + n0 + c4));
      b_reg[i] = v;
    }
  };
  auto store_tiles = [&](int buf) {
#pragma unroll
    for (int i = 0; i < A_PER_T; ++i) *reinterpret_cast<float4*>(&As[buf][a_p[i]][a_k[i]]) = a_reg[i];
#pragma unroll
    for (int i = 0; i < B_PER_T; ++i) {
      int f = tid + i * THREADS;
      int p = f / (BN / 4), c4 = (f % (BN / 4)) * 4;
      *reinterpret_cast<float4*>(&Bs[buf][p][c4]) = b_reg[i];
    }
  };
  const int tx = tid % (BN / TN), ty = tid / (BN / TN);
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  const int nsteps = (int)((m_end - m_begin + BP - 1) / BP);
  load_tiles(m_begin);
  store_tiles(0);
  __syncthreads();
  for (int st = 0; st < nsteps; ++st) {
    int buf = st & 1;
    if (st + 1 < nsteps) load_tiles(m_begin + (int64_t)(st + 1) * BP);
#pragma unroll
    for (int p = 0; p < BP; ++p) {
      float a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; i += 4) {
        float4 v = *reinterpret_cast<const float4*>(&As[buf][p][ty * TM + i]);
        a[i] = v.x; a[i + 1] = v.y; a[i + 2] = v.z; a[i + 3] = v.w;
      }
#pragma unroll
      for (int j = 0; j < TN; j += 4) {
        float4 v = *reinterpret_cast<const float4*>(&Bs[buf][p][tx * TN + j]);
        b[j] = v.x; b[j + 1] = v.y; b[j + 2] = v.z; b[j + 3] = v.w;
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (st + 1 < nsteps) {
      store_tiles(buf ^ 1);
      __syncthreads();
    }
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    int k = k0 + ty * TM + i;
    if (k >= K) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) atomicAdd(dwp + (int64_t)k * g.Cout + n0 + tx * TN + j, acc[i][j]);
  }
}

// ------------------------------------------------------------------------------------------------
static int ilog2_exact(int v) {
  int l = 0;
  while ((1 << l) < v) ++l;
  return (1 << l) == v ? l : -1;
}

int conv_geom_init(ConvGeom* g, int N, int Hin, int Win, int Cin, int Hout, int Wout, int Cout,
                   int KH, int KW, int stride, int ups, int pad, int dil) {
  g->N = N; g->Hin = Hin; g->Win = Win; g->Cin = Cin; g->Hout = Hout; g->Wout = Wout; g->Cout = Cout;
  g->KH = KH; g->KW = KW; g->stride = stride; g->ups = ups; g->pad = pad; g->dil = dil;
  g->cin_log2 = ilog2_exact(Cin);
  DDN_CHECK_ARG(g->cin_log2 >= 2, "SIMT conv needs Cin a power of two >= 4 (got %d)", Cin);
  DDN_CHECK_ARG(Cout % 64 == 0, "SIMT conv needs Cout %% 64 == 0 (got %d)", Cout);
  return 0;
}

int launch_pack_weights(const float* w, float* wp, int Cout, int Cin, int CinP, int KH, int KW, int dgrad, cudaStream_t st) {
  int64_t total = (int64_t)KH * KW * CinP * Cout;
  int blocks = (int)std::min<int64_t>(ceil_div(total, 256), 4096);
  DDN_LAUNCH(pack_weights_kernel, blocks, 256, 0, st, w, wp, Cout, Cin, CinP, KH, KW, dgrad);
  return 0;
}

int launch_unpack_wgrad(const float* dwp, float* dw, int Cout, int Cin, int CinP, int KH, int KW, cudaStream_t st) {
  int64_t total = (int64_t)Cout * Cin * KH * KW;
  int blocks = (int)std::min<int64_t>(ceil_div(total, 256), 4096);
  DDN_LAUNCH(unpack_wgrad_kernel, blocks, 256, 0, st, dwp, dw, Cout, Cin, CinP, KH, KW);
  return 0;
}

int launch_conv_gather_f32(const float* in, const float* wp, const float* addend, float* out, const ConvGeom& g, cudaStream_t st) {
  int64_t M = (int64_t)g.N * g.Hout * g.Wout;
  if (g.Cout % 128 == 0) {
    dim3 grid((unsigned)ceil_div(M, 128), g.Cout / 128);
    DDN_LAUNCH((conv_gather_f32_kernel<128, 128, 8, 8, 8>), grid, 256, 0, st, in, wp, addend, out, g);
  } else {
    dim3 grid((unsigned)ceil_div(M, 128), g.Cout / 64);
    DDN_LAUNCH((conv_gather_f32_kernel<128, 64, 16, 8, 4>), grid, 256, 0, st, in, wp, addend, out, g);
  }
  return 0;
}

// dwp must be zero-filled by the caller (split-K atomics accumulate into it).
int launch_conv_wgrad_f32(const float* in, const float* dy, float* dwp, const ConvGeom& g, cudaStream_t st) {
  int64_t M = (int64_t)g.N * g.Hout * g.Wout;
  int K = g.KH * g.KW * g.Cin;
  constexpr int BKR = 128, BN = 64, BP = 16;
  int tiles = (int)ceil_div(K, BKR) * (g.Cout / BN);
  int want = num_sms() * 4;
  int splits = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(want, tiles), ceil_div(M, 256)));
  int pps = (int)(ceil_div(ceil_div(M, splits), BP) * BP);
  splits = (int)ceil_div(M, pps);
  dim3 grid((unsigned)ceil_div(K, BKR), g.Cout / BN, splits);
  DDN_LAUNCH((conv_wgrad_f32_kernel<BKR, BN, BP, 8, 4>), grid, 256, 0, st, in, dy, dwp, g, pps);
  return 0;
}

}  // namespace ddn
