// Shared helpers for libpasco_sm100 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <mutex>
#include "../../include/pasco_sm100.h"

namespace pasco {

void set_error(const char* fmt, ...);

#define PASCO_CHECK_ARG(cond, ...)            \
  do {                                        \
    if (!(cond)) {                            \
      ::pasco::set_error(__VA_ARGS__);        \
      return -2;                              \
    }                                         \
  } while (0)

#define PASCO_CHECK_LAUNCH(name)                                                         \
  do {                                                                                   \
    cudaError_t e__ = cudaGetLastError();                                                \
    if (e__ != cudaSuccess) {                                                            \
      ::pasco::set_error("%s: CUDA launch failed: %s", name, cudaGetErrorString(e__));   \
      return -1;                                                                         \
    }                                                                                    \
  } while (0)

constexpr int kCoordBias = 32768;
constexpr uint64_t kEmptyKey = 0xFFFFFFFFFFFFFFFFull;

__host__ __device__ __forceinline__ uint64_t pack_key(int b, int x, int y, int z) {
  return ((uint64_t)(uint16_t)(b + kCoordBias) << 48) | ((uint64_t)(uint16_t)(x + kCoordBias) << 32) |
         ((uint64_t)(uint16_t)(y + kCoordBias) << 16) | (uint64_t)(uint16_t)(z + kCoordBias);
}

__device__ __forceinline__ uint32_t hash_key(uint64_t k) {  // murmur3 finaliser
  k ^= k >> 33;
  k *= 0xff51afd7ed558ccdull;
  k ^= k >> 33;
  k *= 0xc4ceb9fe1a85ec53ull;
  k ^= k >> 33;
  return (uint32_t)k;
}

__device__ __forceinline__ int table_find(const uint64_t* __restrict__ keys, const int32_t* __restrict__ vals,
                                          uint32_t mask, uint64_t key) {
  uint32_t slot = hash_key(key) & mask;
  while (true) {
    uint64_t k = __ldg(keys + slot);
    if (k == key) return __ldg(vals + slot);
    if (k == kEmptyKey) return -1;
    slot = (slot + 1) & mask;
  }
}

// activations: 0 none, 1 ReLU, 2 LeakyReLU(0.01) — the row kernels (reduce.cu) and the convolution's inference epilogue
// (conv_tc.cu) share this one definition, so a fused epilogue computes bit for bit what the row pass computes
__device__ __forceinline__ float act_fwd(float z, int act) {
  if (act == 1) return fmaxf(z, 0.f);
  if (act == 2) return z > 0.f ? z : 0.01f * z;
  return z;
}

__host__ __device__ __forceinline__ int floor_div(int a, int s) {
  int q = a / s;
  return (a % s != 0 && ((a < 0) != (s < 0))) ? q - 1 : q;
}

inline int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

// stream-ordered workspace of a call (freed with cudaFreeAsync on the same stream), from a memory pool of the library's
// own per device.  The pool keeps freed blocks (release threshold = unlimited) instead of returning them to the driver
// at every synchronisation, so a per-call workspace costs no re-mapping from one training step to the next; it holds
// at most the largest workspace in flight and lives as long as the process.  The default pool is left untouched.
inline cudaError_t ws_alloc(void** p, size_t bytes, cudaStream_t st) {
  static std::mutex mu;
  static cudaMemPool_t pools[64] = {};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
  cudaMemPool_t pool;
  {
    std::lock_guard<std::mutex> lock(mu);
    if (!pools[dev]) {
      cudaMemPoolProps props = {};
      props.allocType = cudaMemAllocationTypePinned;
      props.location.type = cudaMemLocationTypeDevice;
      props.location.id = dev;
      e = cudaMemPoolCreate(&pools[dev], &props);
      if (e != cudaSuccess) {
        pools[dev] = nullptr;
        return e;
      }
      uint64_t keep = ~0ull;
      cudaMemPoolSetAttribute(pools[dev], cudaMemPoolAttrReleaseThreshold, &keep);
    }
    pool = pools[dev];
  }
  return cudaMallocFromPoolAsync(p, bytes, pool, st);
}

inline int grid_for(int64_t work, int block, int waves = 8) {
  int64_t g = (work + block - 1) / block;
  int64_t cap = (int64_t)num_sms() * waves;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace pasco
