// Device-resident training frames: one launch gathers the frames B image pairs need from a FrameStore
// (pdc_b200/frames.py) into the producers' input layout (within_scene_batch / across_scene_batch /
// synthetic_multi_object_batch): rgb uint8 [B, H, W, 3] and mask uint8 [B, H, W] copied, depth uint16 -> float32
// millimetres [B, H, W] (exact: every uint16 is a float32).  Contract: include/ddn_b200.h (ddn_frames_gather).
//
// The store's pointers are read through UVA, so the same kernel reads a store in device memory or in pinned host memory
// (zero-copy over the host link).  The frame indices travel as kernel parameters: no host-to-device copy, no sync.
#include "common.cuh"

namespace ddn {

struct FramesGatherArgs {
  const uint8_t* rgb; const uint16_t* depth; const uint8_t* mask;        // the store, [F, H, W, 3] / [F, H, W] / [F, H, W]
  uint8_t* rgb_out[2]; float* depth_out[2]; uint8_t* mask_out[2];        // [side] -> [B, ...]; depth_out may be null
  int64_t P;                                                            // H * W
  int32_t idx[2][DDN_FRAMES_MAX_PAIRS];                                 // [side][pair] frame index
};

// n bytes s -> d: 16-byte vectors once d is aligned, if s is then aligned too; scalar head and tail
__device__ __forceinline__ void gather_bytes(const uint8_t* __restrict__ s, uint8_t* __restrict__ d, int64_t n, int64_t t,
                                             int64_t nt) {
  int64_t head = (int64_t)((16 - ((uintptr_t)d & 15)) & 15); if (head > n) head = n;
  if ((((uintptr_t)s + head) & 15) != 0) head = n;          // s and d differ in alignment: bytes only
  const int64_t nv = (n - head) >> 4;
  const uint4* sv = reinterpret_cast<const uint4*>(s + head);
  uint4* dv = reinterpret_cast<uint4*>(d + head);
  for (int64_t i = t; i < nv; i += nt) dv[i] = sv[i];
  for (int64_t i = t; i < head; i += nt) d[i] = s[i];
  for (int64_t i = head + (nv << 4) + t; i < n; i += nt) d[i] = s[i];
}

// n uint16 s -> float32 d: 8 values (one 16-byte load, two 16-byte stores) at a time where both line up
__device__ __forceinline__ void gather_depth(const uint16_t* __restrict__ s, float* __restrict__ d, int64_t n, int64_t t,
                                             int64_t nt) {
  int64_t head = (int64_t)(((16 - ((uintptr_t)s & 15)) & 15) >> 1); if (head > n) head = n;
  if (((uintptr_t)(d + head) & 15) != 0) head = n;
  const int64_t nv = (n - head) >> 3;
  const uint4* sv = reinterpret_cast<const uint4*>(s + head);
  float4* dv = reinterpret_cast<float4*>(d + head);
  for (int64_t i = t; i < nv; i += nt) {
    const uint4 v = sv[i];
    dv[2 * i] = make_float4((float)(v.x & 0xffffu), (float)(v.x >> 16), (float)(v.y & 0xffffu), (float)(v.y >> 16));
    dv[2 * i + 1] = make_float4((float)(v.z & 0xffffu), (float)(v.z >> 16), (float)(v.w & 0xffffu), (float)(v.w >> 16));
  }
  for (int64_t i = t; i < head; i += nt) d[i] = (float)s[i];
  for (int64_t i = head + (nv << 3) + t; i < n; i += nt) d[i] = (float)s[i];
}

// grid (chunks, B, 2 sides): chunk x of every plane of output frame (side, pair)
__global__ void __launch_bounds__(256) frames_gather_kernel(const __grid_constant__ FramesGatherArgs a) {
  pdl_prologue();
  const int side = blockIdx.z, b = blockIdx.y;
  const int64_t f = a.idx[side][b], P = a.P;
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, nt = (int64_t)gridDim.x * blockDim.x;
  gather_bytes(a.rgb + f * P * 3, a.rgb_out[side] + b * P * 3, P * 3, t, nt);
  gather_bytes(a.mask + f * P, a.mask_out[side] + b * P, P, t, nt);
  if (a.depth_out[side]) gather_depth(a.depth + f * P, a.depth_out[side] + b * P, P, t, nt);
}

}  // namespace ddn

using namespace ddn;

extern "C" int ddn_frames_gather(const uint8_t* rgb, const uint16_t* depth, const uint8_t* mask, int64_t F, int H, int W,
                                 const int32_t* idx_a_host, const int32_t* idx_b_host, int B, uint8_t* rgb_a, uint8_t* rgb_b,
                                 float* depth_a, float* depth_b, uint8_t* mask_a, uint8_t* mask_b, void* stream) {
  DDN_CHECK_ARG(B >= 1 && B <= DDN_FRAMES_MAX_PAIRS, "ddn_frames_gather: B must be in [1, %d] (got %d)", DDN_FRAMES_MAX_PAIRS, B);
  DDN_CHECK_ARG(F >= 1 && H >= 1 && W >= 1 && (int64_t)H * W < (1ll << 40) / 4, "ddn_frames_gather: bad store shape F=%lld H=%d W=%d",
                (long long)F, H, W);
  DDN_CHECK_ARG(rgb && mask && idx_a_host && idx_b_host && rgb_a && rgb_b && mask_a && mask_b, "ddn_frames_gather: null argument");
  DDN_CHECK_ARG((depth_a == nullptr) == (depth_b == nullptr), "ddn_frames_gather: depth_a and depth_b must both be given or both null");
  DDN_CHECK_ARG(depth || !depth_a, "ddn_frames_gather: depth output requested from a null depth store");
  FramesGatherArgs a = {};
  for (int s = 0; s < 2; ++s) {
    const int32_t* idx = s ? idx_b_host : idx_a_host;
    for (int b = 0; b < B; ++b) {
      DDN_CHECK_ARG(idx[b] >= 0 && idx[b] < F, "ddn_frames_gather: frame index %d of side %c pair %d is outside [0, %lld)",
                    idx[b], s ? 'b' : 'a', b, (long long)F);
      a.idx[s][b] = idx[b];
    }
  }
  a.rgb = rgb; a.depth = depth; a.mask = mask;
  a.rgb_out[0] = rgb_a; a.rgb_out[1] = rgb_b; a.depth_out[0] = depth_a; a.depth_out[1] = depth_b;
  a.mask_out[0] = mask_a; a.mask_out[1] = mask_b;
  a.P = (int64_t)H * W;
  // enough blocks to keep every SM busy whatever B is; a block's threads each move 16 bytes per plane per pass
  const int64_t per_frame = ceil_div(a.P * 3, 16 * 256);
  const int chunks = (int)std::max<int64_t>(1, std::min<int64_t>(per_frame, ceil_div(4 * num_sms(), 2 * B)));
  DDN_LAUNCH(frames_gather_kernel, dim3(chunks, B, 2), 256, 0, (cudaStream_t)stream, a);
  return 0;
}
