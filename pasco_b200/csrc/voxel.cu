// Point voxeliser grouping and the MIMO subnet merge on packed coordinate keys.
//
//   pasco_voxel_group / _order      torch.unique(rows, dim=0, return_inverse=True) for int (b, x, y, z) rows
//                                   (pasco/models/unet3d_sparse_v2.py:72-75): hash dedup of the packed keys, then one
//                                   radix sort of the unique keys only.  The bias-packed key orders as the signed rows
//                                   do, so the sorted keys are torch.unique's ascending lexicographic order.
//   pasco_mimo_merge_cells / _forward / _backward
//                                   Augmenter.merge (pasco/models/augmenter.py:13-27) without its dense volume: the
//                                   union of the subnets' (x, y, z) cells, rows whose M·f features are all ±0 dropped as
//                                   ME.to_sparse drops them, in ascending (x, y, z) order; pure data movement.
//
// Integer and copy work only: every result is exact, and independent of the order the atomics land in (the unique
// keys are collected in any order and then sorted).
#include <cub/device/device_radix_sort.cuh>
#include "common.cuh"

using namespace pasco;

namespace {

template <typename T>
__device__ __forceinline__ bool in_key_range(T v) {
  return v >= -(T)kCoordBias && v < (T)kCoordBias;
}

// insert `key` (never kEmptyKey) and return its slot
__device__ __forceinline__ uint32_t insert_slot(unsigned long long* keys, uint32_t mask, uint64_t key) {
  uint32_t slot = hash_key(key) & mask;
  while (true) {
    unsigned long long prev = atomicCAS(keys + slot, (unsigned long long)kEmptyKey, (unsigned long long)key);
    if (prev == kEmptyKey || prev == key) return slot;
    slot = (slot + 1) & mask;
  }
}

__device__ __forceinline__ uint32_t find_slot(const uint64_t* __restrict__ keys, uint32_t mask, uint64_t key) {
  uint32_t slot = hash_key(key) & mask;
  while (__ldg(keys + slot) != key) slot = (slot + 1) & mask;
  return slot;
}

// one (b, x, y, z) row of int32 or int64 components; bad = a component outside the packable range
template <typename T>
__device__ __forceinline__ uint64_t row_key(const T* __restrict__ rows, int64_t i, bool& bad) {
  const T b = rows[4 * i], x = rows[4 * i + 1], y = rows[4 * i + 2], z = rows[4 * i + 3];
  bad = !(in_key_range(b) && in_key_range(x) && in_key_range(y) && in_key_range(z));
  const uint64_t key = pack_key((int)b, (int)x, (int)y, (int)z);
  bad |= key == kEmptyKey;
  return key;
}

template <typename T>
__global__ void k_vox_insert(const T* __restrict__ rows, int64_t n, unsigned long long* keys, uint32_t mask,
                             int32_t* __restrict__ err) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    bool bad;
    const uint64_t key = row_key(rows, i, bad);
    if (bad) {
      *err = 1;                            // nothing of this row is inserted; the caller discards the call
      continue;
    }
    insert_slot(keys, mask, key);
  }
}

// Augmenter.merge's cells: key (0, x, y, z) of every row; vals[slot] |= 1 where the row has a feature that is not ±0
// (NaN included: ME.to_sparse keeps a row whose |F| sum is not exactly 0).  stats[1] = max batch index, stats[2] = err.
__global__ void k_merge_insert(const int4* __restrict__ coords, const float* __restrict__ F, int64_t n, int f,
                               unsigned long long* keys, int32_t* vals, uint32_t mask, int32_t* __restrict__ stats) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int4 c = __ldg(coords + i);
    if (c.x < 0 || !(in_key_range(c.y) && in_key_range(c.z) && in_key_range(c.w))) {
      stats[2] = 1;
      continue;
    }
    atomicMax(stats + 1, c.x);
    const uint32_t slot = insert_slot(keys, mask, pack_key(0, c.y, c.z, c.w));
    const float* row = F + i * f;
    uint32_t any = 0;
    for (int k = 0; k < f; ++k) any |= __float_as_uint(__ldg(row + k)) & 0x7FFFFFFFu;
    if (any) atomicOr(vals + slot, 1);
  }
}

// the occupied slots' keys → ukeys[0 .. stats[0]) in any order (one atomic per warp).  flagged: only slots with
// vals != 0 are taken; the others get vals = −1 ("no output row").
__global__ void k_collect(const uint64_t* __restrict__ keys, int32_t* vals, int64_t cap, int flagged,
                          uint64_t* __restrict__ ukeys, int32_t* __restrict__ count) {
  const int lane = threadIdx.x & 31;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i0 = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) & ~(int64_t)31; i0 < cap; i0 += stride) {
    const int64_t i = i0 + lane;
    uint64_t key = kEmptyKey;
    bool take = false;
    if (i < cap) {
      key = keys[i];
      if (key != kEmptyKey) {
        take = !flagged || vals[i] != 0;
        if (!take) vals[i] = -1;
      }
    }
    const unsigned ballot = __ballot_sync(0xFFFFFFFFu, take);
    if (!ballot) continue;
    int base = 0;
    if (lane == 0) base = atomicAdd(count, __popc(ballot));
    base = __shfl_sync(0xFFFFFFFFu, base, 0);
    if (take) ukeys[base + __popc(ballot & ((1u << lane) - 1))] = key;
  }
}

// sorted key r → vals[slot] = r, and the unpacked row
template <typename T>
__global__ void k_rank(const uint64_t* __restrict__ sorted, int64_t U, const uint64_t* __restrict__ keys,
                       int32_t* vals, uint32_t mask, T* __restrict__ rows) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < U; r += (int64_t)gridDim.x * blockDim.x) {
    const uint64_t key = sorted[r];
    vals[find_slot(keys, mask, key)] = (int32_t)r;
    rows[4 * r] = (T)((int)((key >> 48) & 0xFFFF) - kCoordBias);
    rows[4 * r + 1] = (T)((int)((key >> 32) & 0xFFFF) - kCoordBias);
    rows[4 * r + 2] = (T)((int)((key >> 16) & 0xFFFF) - kCoordBias);
    rows[4 * r + 3] = (T)((int)(key & 0xFFFF) - kCoordBias);
  }
}

template <typename T>
__global__ void k_vox_inverse(const T* __restrict__ rows, int64_t n, const uint64_t* __restrict__ keys,
                              const int32_t* __restrict__ vals, uint32_t mask, int64_t* __restrict__ inverse) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    bool bad;
    const uint64_t key = row_key(rows, i, bad);
    inverse[i] = __ldg(vals + find_slot(keys, mask, key));
  }
}

__global__ void k_merge_rows(const int4* __restrict__ coords, int64_t n, const uint64_t* __restrict__ keys,
                             const int32_t* __restrict__ vals, uint32_t mask, int32_t* __restrict__ row_of) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int4 c = __ldg(coords + i);
    row_of[i] = __ldg(vals + find_slot(keys, mask, pack_key(0, c.y, c.z, c.w)));
  }
}

// out[row_of[i], b_i·f + k] = F[i, k]   (out zeroed first)
__global__ void k_merge_copy(const int4* __restrict__ coords, const int32_t* __restrict__ row_of,
                             const float* __restrict__ F, int64_t n, int f, int M, float* __restrict__ out) {
  const int64_t total = n * f;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = e / f;
    const int k = (int)(e - i * f);
    const int r = __ldg(row_of + i);
    if (r >= 0) out[(int64_t)r * M * f + (int64_t)__ldg(&coords[i].x) * f + k] = __ldg(F + e);
  }
}

// gin[i, k] = g[row_of[i], b_i·f + k], 0 for a dropped cell.  For M > 1 the dense path's gradient is the sum of the M
// per-subnet slices' zero-filled gradients, i.e. g + 0.0f (a −0.0 gradient becomes +0.0): added here too, bit for bit.
__global__ void k_merge_grad(const int4* __restrict__ coords, const int32_t* __restrict__ row_of,
                             const float* __restrict__ g, int64_t n, int f, int M, float* __restrict__ gin) {
  const int64_t total = n * f;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = e / f;
    const int k = (int)(e - i * f);
    const int r = __ldg(row_of + i);
    float v = r >= 0 ? __ldg(g + (int64_t)r * M * f + (int64_t)__ldg(&coords[i].x) * f + k) : 0.f;
    gin[e] = M > 1 ? __fadd_rn(v, 0.f) : v;
  }
}

bool pow2(int64_t v) { return v > 0 && (v & (v - 1)) == 0; }

// ukeys[0 .. U) sorted ascending over key bits [0, end_bit) into a workspace buffer; *sorted is freed by the caller
// with cudaFreeAsync on `st`
int sort_keys(const uint64_t* ukeys, int64_t U, int end_bit, uint64_t** sorted, cudaStream_t st, const char* name) {
  size_t tmp_bytes = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, tmp_bytes, ukeys, (uint64_t*)nullptr, (int)U, 0, end_bit, st);
  const size_t keys_bytes = ((size_t)U * sizeof(uint64_t) + 255) & ~(size_t)255;
  void* ws = nullptr;
  if (ws_alloc(&ws, keys_bytes + tmp_bytes, st) != cudaSuccess) {
    set_error("%s: workspace allocation of %zu bytes failed", name, keys_bytes + tmp_bytes);
    return -1;
  }
  *sorted = (uint64_t*)ws;
  if (cub::DeviceRadixSort::SortKeys((char*)ws + keys_bytes, tmp_bytes, ukeys, *sorted, (int)U, 0, end_bit, st) !=
      cudaSuccess) {
    cudaFreeAsync(ws, st);
    set_error("%s: radix sort failed", name);
    return -1;
  }
  return 0;
}

}  // namespace

extern "C" int pasco_voxel_group(const void* rows, int32_t is_i64, int64_t n, uint64_t* table_keys, int64_t capacity,
                                 uint64_t* ukeys, int32_t* stats, pasco_stream_t s) {
  PASCO_CHECK_ARG(pow2(capacity) && capacity >= 2 * n && capacity <= (1ll << 31),
                  "pasco_voxel_group: capacity %lld must be a power of two >= 2n (n=%lld)", (long long)capacity,
                  (long long)n);
  if (n == 0) return 0;
  cudaStream_t st = (cudaStream_t)s;
  const uint32_t mask = (uint32_t)(capacity - 1);
  if (is_i64)
    k_vox_insert<<<grid_for(n, 256), 256, 0, st>>>((const int64_t*)rows, n, (unsigned long long*)table_keys, mask,
                                                    stats + 1);
  else
    k_vox_insert<<<grid_for(n, 256), 256, 0, st>>>((const int32_t*)rows, n, (unsigned long long*)table_keys, mask,
                                                    stats + 1);
  k_collect<<<grid_for(capacity, 256), 256, 0, st>>>(table_keys, nullptr, capacity, 0, ukeys, stats);
  PASCO_CHECK_LAUNCH("pasco_voxel_group");
  return 0;
}

extern "C" int pasco_voxel_group_order(const void* rows, int32_t is_i64, int64_t n, const uint64_t* table_keys,
                                       int32_t* table_vals, int64_t capacity, const uint64_t* ukeys, int64_t U,
                                       void* unique_rows, int64_t* inverse, pasco_stream_t s) {
  PASCO_CHECK_ARG(pow2(capacity) && U <= n && U < (1ll << 31), "pasco_voxel_group_order: bad sizes");
  if (n == 0) return 0;
  cudaStream_t st = (cudaStream_t)s;
  const uint32_t mask = (uint32_t)(capacity - 1);
  uint64_t* sorted = nullptr;
  if (sort_keys(ukeys, U, 64, &sorted, st, "pasco_voxel_group_order")) return -1;
  if (is_i64) {
    k_rank<<<grid_for(U, 256), 256, 0, st>>>(sorted, U, table_keys, table_vals, mask, (int64_t*)unique_rows);
    k_vox_inverse<<<grid_for(n, 256), 256, 0, st>>>((const int64_t*)rows, n, table_keys, table_vals, mask, inverse);
  } else {
    k_rank<<<grid_for(U, 256), 256, 0, st>>>(sorted, U, table_keys, table_vals, mask, (int32_t*)unique_rows);
    k_vox_inverse<<<grid_for(n, 256), 256, 0, st>>>((const int32_t*)rows, n, table_keys, table_vals, mask, inverse);
  }
  cudaFreeAsync(sorted, st);
  PASCO_CHECK_LAUNCH("pasco_voxel_group_order");
  return 0;
}

extern "C" int pasco_mimo_merge_cells(const int32_t* coords, const float* F, int64_t n, int32_t f,
                                      uint64_t* table_keys, int32_t* table_vals, int64_t capacity, uint64_t* ukeys,
                                      int32_t* stats, pasco_stream_t s) {
  PASCO_CHECK_ARG(pow2(capacity) && capacity >= 2 * n && capacity <= (1ll << 31) && f > 0,
                  "pasco_mimo_merge_cells: capacity %lld must be a power of two >= 2n (n=%lld), f > 0",
                  (long long)capacity, (long long)n);
  if (n == 0) return 0;
  cudaStream_t st = (cudaStream_t)s;
  const uint32_t mask = (uint32_t)(capacity - 1);
  k_merge_insert<<<grid_for(n, 256), 256, 0, st>>>((const int4*)coords, F, n, f, (unsigned long long*)table_keys,
                                                    table_vals, mask, stats);
  k_collect<<<grid_for(capacity, 256), 256, 0, st>>>(table_keys, table_vals, capacity, 1, ukeys, stats);
  PASCO_CHECK_LAUNCH("pasco_mimo_merge_cells");
  return 0;
}

extern "C" int pasco_mimo_merge_forward(const int32_t* coords, const float* F, int64_t n, int32_t f, int32_t M,
                                        const uint64_t* table_keys, int32_t* table_vals, int64_t capacity,
                                        const uint64_t* ukeys, int64_t U, int32_t* out_coords, float* out_F,
                                        int32_t* row_of, pasco_stream_t s) {
  PASCO_CHECK_ARG(pow2(capacity) && U <= n && M >= 1 && f > 0 && U < (1ll << 31),
                  "pasco_mimo_merge_forward: bad sizes");
  if (n == 0) return 0;
  cudaStream_t st = (cudaStream_t)s;
  const uint32_t mask = (uint32_t)(capacity - 1);
  if (U > 0) {
    uint64_t* sorted = nullptr;
    if (sort_keys(ukeys, U, 48, &sorted, st, "pasco_mimo_merge_forward")) return -1;   // batch bits are 0x8000
    k_rank<<<grid_for(U, 256), 256, 0, st>>>(sorted, U, table_keys, table_vals, mask, out_coords);
    cudaFreeAsync(sorted, st);
    cudaMemsetAsync(out_F, 0, (size_t)U * M * f * sizeof(float), st);
  }
  k_merge_rows<<<grid_for(n, 256), 256, 0, st>>>((const int4*)coords, n, table_keys, table_vals, mask, row_of);
  k_merge_copy<<<grid_for(n * f, 256), 256, 0, st>>>((const int4*)coords, row_of, F, n, f, M, out_F);
  PASCO_CHECK_LAUNCH("pasco_mimo_merge_forward");
  return 0;
}

extern "C" int pasco_mimo_merge_backward(const int32_t* coords, const int32_t* row_of, int64_t n, int32_t f,
                                         int32_t M, const float* g, float* gin, pasco_stream_t s) {
  PASCO_CHECK_ARG(M >= 1 && f > 0, "pasco_mimo_merge_backward: bad sizes");
  if (n == 0) return 0;
  cudaStream_t st = (cudaStream_t)s;
  k_merge_grad<<<grid_for(n * f, 256), 256, 0, st>>>((const int4*)coords, row_of, g, n, f, M, gin);
  PASCO_CHECK_LAUNCH("pasco_mimo_merge_backward");
  return 0;
}
