// Pre-split bf16 planes of an activation tensor (sm_90a): x = hi + lo with hi = bf16(x), lo = bf16(x - hi).
//
// The plane-gather convolution kernels (k_conv_pl in conv_tc.cu, k_wgrad_pl in wgrad_tc.cu) read their gathered
// operand from these planes with 16-byte cp.async copies, so the split (and, optionally, the BatchNorm affine +
// activation of the layer that produced x) is done ONCE per tensor here instead of once per kernel offset inside the
// gather.  HBM-bound: reads 4 B and writes 4 B (2 B in bf16 mode) per element.
#include "common.cuh"
#include "gmma.cuh"

using namespace pasco;
using namespace gmma;

namespace {

// fp32 [N, C] (row pitch `pitch`) → bf16 planes hi (and lo = bf16(y − hi)) of y = act(x*scale + shift)
__global__ void k_split_planes(const float* __restrict__ x, int64_t n, int C, int64_t pitch, const float* __restrict__ scale,
                               const float* __restrict__ shift, int act, __nv_bfloat16* __restrict__ hi,
                               __nv_bfloat16* __restrict__ lo) {
  const int cv = C >> 3;                      // 8 channels (two float4 in, one uint4 out per plane) per thread step
  const int64_t total = n * cv;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / cv;
    const int c = (int)(t - r * cv) << 3;
    float4 v0 = __ldg(reinterpret_cast<const float4*>(x + r * pitch + c));
    float4 v1 = __ldg(reinterpret_cast<const float4*>(x + r * pitch + c + 4));
    if (scale) {
      const float4 s0 = __ldg(reinterpret_cast<const float4*>(scale + c)), s1 = __ldg(reinterpret_cast<const float4*>(scale + c + 4));
      const float4 h0 = __ldg(reinterpret_cast<const float4*>(shift + c)), h1 = __ldg(reinterpret_cast<const float4*>(shift + c + 4));
      v0.x = fmaf(v0.x, s0.x, h0.x); v0.y = fmaf(v0.y, s0.y, h0.y); v0.z = fmaf(v0.z, s0.z, h0.z); v0.w = fmaf(v0.w, s0.w, h0.w);
      v1.x = fmaf(v1.x, s1.x, h1.x); v1.y = fmaf(v1.y, s1.y, h1.y); v1.z = fmaf(v1.z, s1.z, h1.z); v1.w = fmaf(v1.w, s1.w, h1.w);
    }
    if (act == 1) {
      v0.x = fmaxf(v0.x, 0.f); v0.y = fmaxf(v0.y, 0.f); v0.z = fmaxf(v0.z, 0.f); v0.w = fmaxf(v0.w, 0.f);
      v1.x = fmaxf(v1.x, 0.f); v1.y = fmaxf(v1.y, 0.f); v1.z = fmaxf(v1.z, 0.f); v1.w = fmaxf(v1.w, 0.f);
    } else if (act == 2) {
      v0.x = v0.x > 0.f ? v0.x : 0.01f * v0.x; v0.y = v0.y > 0.f ? v0.y : 0.01f * v0.y;
      v0.z = v0.z > 0.f ? v0.z : 0.01f * v0.z; v0.w = v0.w > 0.f ? v0.w : 0.01f * v0.w;
      v1.x = v1.x > 0.f ? v1.x : 0.01f * v1.x; v1.y = v1.y > 0.f ? v1.y : 0.01f * v1.y;
      v1.z = v1.z > 0.f ? v1.z : 0.01f * v1.z; v1.w = v1.w > 0.f ? v1.w : 0.01f * v1.w;
    }
    if (lo) {
      uint2 h0, l0, h1, l1;
      split4(v0, h0, l0);
      split4(v1, h1, l1);
      *reinterpret_cast<uint4*>(hi + r * C + c) = make_uint4(h0.x, h0.y, h1.x, h1.y);
      *reinterpret_cast<uint4*>(lo + r * C + c) = make_uint4(l0.x, l0.y, l1.x, l1.y);
    } else {
      const uint2 h0 = to_bf16x4(v0), h1 = to_bf16x4(v1);
      *reinterpret_cast<uint4*>(hi + r * C + c) = make_uint4(h0.x, h0.y, h1.x, h1.y);
    }
  }
}

}  // namespace

extern "C" int pasco_split_planes(const float* x, int64_t n, int32_t C, int64_t pitch, const float* scale, const float* shift,
                                  int32_t act, void* hi, void* lo, pasco_stream_t s) {
  PASCO_CHECK_ARG(C % 8 == 0 && (pitch == 0 || pitch % 4 == 0), "pasco_split_planes: C must be a multiple of 8, pitch of 4");
  PASCO_CHECK_ARG((scale == nullptr) == (shift == nullptr), "pasco_split_planes: scale and shift come together");
  PASCO_CHECK_ARG((((uintptr_t)x | (uintptr_t)hi | (uintptr_t)lo) & 15) == 0, "pasco_split_planes: pointers must be 16-byte aligned");
  if (n == 0) return 0;
  k_split_planes<<<grid_for(n * (C / 8), 256), 256, 0, (cudaStream_t)s>>>(x, n, C, pitch > 0 ? pitch : C, scale, shift, act,
                                                                        (__nv_bfloat16*)hi, (__nv_bfloat16*)lo);
  PASCO_CHECK_LAUNCH("pasco_split_planes");
  return 0;
}
