// Coordinate maps, kernel maps, row compaction, row gather/scatter, dense<->sparse.
// All HBM-bound integer/byte work: coalesced grid-stride kernels, grids sized in multiples of the SM count.
#include <stdarg.h>
#include "common.cuh"

namespace pasco {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
}  // namespace pasco

using namespace pasco;

extern "C" const char* pasco_last_error(void) { return pasco::g_err; }
extern "C" int pasco_abi_version(void) { return 3; }
extern "C" int pasco_device_info(int* sm_count, int* smem_optin, int* cc) {
  int dev = 0, v = 0, maj = 0, min = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    set_error("pasco_device_info: no CUDA device");
    return -1;
  }
  cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
  if (sm_count) *sm_count = v;
  cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  if (smem_optin) *smem_optin = v;
  cudaDeviceGetAttribute(&maj, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&min, cudaDevAttrComputeCapabilityMinor, dev);
  if (cc) *cc = maj * 10 + min;
  return 0;
}

// ------------------------------------------------------------------------------------------------
// hash table
// ------------------------------------------------------------------------------------------------
__global__ void k_hash_insert(const int4* __restrict__ coords, int64_t n, unsigned long long* keys, int* vals,
                              uint32_t mask, int* __restrict__ err) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int4 c = __ldg(coords + i);
    // keys pack 16 bits per component (bias 2^15): a component outside [-32768, 32767] would alias another voxel, and
    // (32767,32767,32767,32767) is the empty-slot marker.  Flag it (the host raises) instead of mapping silently.
    const bool bad = ((unsigned)(c.x + kCoordBias) | (unsigned)(c.y + kCoordBias) | (unsigned)(c.z + kCoordBias) |
                      (unsigned)(c.w + kCoordBias)) > 0xFFFFu;
    if (err && (bad || pack_key(c.x, c.y, c.z, c.w) == kEmptyKey)) *err = 2;
    uint64_t key = pack_key(c.x, c.y, c.z, c.w);
    uint32_t slot = hash_key(key) & mask;
    while (true) {
      unsigned long long prev = atomicCAS(keys + slot, (unsigned long long)kEmptyKey, (unsigned long long)key);
      if (prev == kEmptyKey || prev == key) {
        atomicMin(vals + slot, (int)i);
        break;
      }
      slot = (slot + 1) & mask;
    }
  }
}

__global__ void k_hash_lookup(const int4* __restrict__ q, int64_t n, const uint64_t* __restrict__ keys,
                              const int32_t* __restrict__ vals, uint32_t mask, int32_t* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int4 c = __ldg(q + i);
    out[i] = table_find(keys, vals, mask, pack_key(c.x, c.y, c.z, c.w));
  }
}

__global__ void k_hash_remap(int32_t* vals, int64_t cap, const int32_t* __restrict__ new_row) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < cap; i += (int64_t)gridDim.x * blockDim.x) {
    int v = vals[i];
    if (v != 0x7F7F7F7F && v >= 0) vals[i] = __ldg(new_row + v);
  }
}

static bool is_pow2(int64_t v) { return v > 0 && (v & (v - 1)) == 0; }

extern "C" int pasco_hash_insert(const int32_t* coords, int64_t n, uint64_t* table_keys, int32_t* table_vals,
                                 int64_t capacity, int32_t* first_row, int32_t* err_flag, pasco_stream_t s) {
  PASCO_CHECK_ARG(is_pow2(capacity) && capacity >= 2 * n && capacity <= (1ll << 31),
                  "pasco_hash_insert: capacity %lld must be a power of two >= 2n (n=%lld)", (long long)capacity,
                  (long long)n);
  PASCO_CHECK_ARG(n < 0x7F7F7F7F, "pasco_hash_insert: too many rows");
  if (n == 0) return 0;
  cudaStream_t st = (cudaStream_t)s;
  k_hash_insert<<<grid_for(n, 256), 256, 0, st>>>((const int4*)coords, n, (unsigned long long*)table_keys,
                                                   table_vals, (uint32_t)(capacity - 1), err_flag);
  if (first_row)
    k_hash_lookup<<<grid_for(n, 256), 256, 0, st>>>((const int4*)coords, n, table_keys, table_vals,
                                                     (uint32_t)(capacity - 1), first_row);
  PASCO_CHECK_LAUNCH("pasco_hash_insert");
  return 0;
}

extern "C" int pasco_hash_remap(int32_t* table_vals, int64_t capacity, const int32_t* new_row, pasco_stream_t s) {
  k_hash_remap<<<grid_for(capacity, 256), 256, 0, (cudaStream_t)s>>>(table_vals, capacity, new_row);
  PASCO_CHECK_LAUNCH("pasco_hash_remap");
  return 0;
}

extern "C" int pasco_hash_lookup(const int32_t* query, int64_t nq, const uint64_t* table_keys,
                                 const int32_t* table_vals, int64_t capacity, int32_t* out_row, pasco_stream_t s) {
  PASCO_CHECK_ARG(is_pow2(capacity), "pasco_hash_lookup: capacity must be a power of two");
  if (nq == 0) return 0;
  k_hash_lookup<<<grid_for(nq, 256), 256, 0, (cudaStream_t)s>>>((const int4*)query, nq, table_keys, table_vals,
                                                                 (uint32_t)(capacity - 1), out_row);
  PASCO_CHECK_LAUNCH("pasco_hash_lookup");
  return 0;
}

// ------------------------------------------------------------------------------------------------
// coordinate generation
// ------------------------------------------------------------------------------------------------
__global__ void k_coords_floor(const int4* __restrict__ in, int64_t n, int sx, int sy, int sz, int4* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int4 c = __ldg(in + i);
    out[i] = make_int4(c.x, floor_div(c.y, sx) * sx, floor_div(c.z, sy) * sy, floor_div(c.w, sz) * sz);
  }
}

extern "C" int pasco_coords_floor(const int32_t* coords, int64_t n, int32_t sx, int32_t sy, int32_t sz, int32_t* out,
                                  pasco_stream_t s) {
  PASCO_CHECK_ARG(sx > 0 && sy > 0 && sz > 0, "pasco_coords_floor: stride must be positive");
  if (n == 0) return 0;
  k_coords_floor<<<grid_for(n, 256), 256, 0, (cudaStream_t)s>>>((const int4*)coords, n, sx, sy, sz, (int4*)out);
  PASCO_CHECK_LAUNCH("pasco_coords_floor");
  return 0;
}

__global__ void k_coords_generate_k2(const int4* __restrict__ in, int64_t n, int sx, int sy, int sz,
                                     int4* __restrict__ out) {
  int64_t total = n * 8;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    int64_t p = t >> 3;
    int k = (int)(t & 7);
    int4 c = __ldg(in + p);
    out[t] = make_int4(c.x, c.y + (k & 1) * sx, c.z + ((k >> 1) & 1) * sy, c.w + ((k >> 2) & 1) * sz);
  }
}

extern "C" int pasco_coords_generate_k2(const int32_t* coords, int64_t n, int32_t out_sx, int32_t out_sy,
                                        int32_t out_sz, int32_t* out, pasco_stream_t s) {
  if (n == 0) return 0;
  k_coords_generate_k2<<<grid_for(n * 8, 256), 256, 0, (cudaStream_t)s>>>((const int4*)coords, n, out_sx, out_sy,
                                                                          out_sz, (int4*)out);
  PASCO_CHECK_LAUNCH("pasco_coords_generate_k2");
  return 0;
}

// ------------------------------------------------------------------------------------------------
// kernel maps
// ------------------------------------------------------------------------------------------------
template <int KS>
__global__ void k_kernel_map_probe(const int4* __restrict__ out_coords, int64_t n, const uint64_t* __restrict__ keys,
                                   const int32_t* __restrict__ vals, uint32_t mask, int sx, int sy, int sz,
                                   int32_t* __restrict__ nbr) {
  constexpr int R = KS / 2;
  for (int64_t o = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; o < n; o += (int64_t)gridDim.x * blockDim.x) {
    int4 c = __ldg(out_coords + o);
    int k = 0;
#pragma unroll
    for (int dz = -R; dz <= R; ++dz)
#pragma unroll
      for (int dy = -R; dy <= R; ++dy)
#pragma unroll
        for (int dx = -R; dx <= R; ++dx, ++k) {
          int v = table_find(keys, vals, mask, pack_key(c.x, c.y + dx * sx, c.z + dy * sy, c.w + dz * sz));
          nbr[(int64_t)k * n + o] = v;
        }
  }
}

extern "C" int pasco_kernel_map_probe(const int32_t* out_coords, int64_t n_out, const uint64_t* table_keys,
                                      const int32_t* table_vals, int64_t capacity, int32_t kernel_size, int32_t sx,
                                      int32_t sy, int32_t sz, int32_t* nbr, pasco_stream_t s) {
  PASCO_CHECK_ARG(kernel_size == 3 || kernel_size == 5 || kernel_size == 1,
                  "pasco_kernel_map_probe: odd kernel sizes 1/3/5 only (got %d)", kernel_size);
  PASCO_CHECK_ARG(is_pow2(capacity), "pasco_kernel_map_probe: capacity must be a power of two");
  if (n_out == 0) return 0;
  cudaStream_t st = (cudaStream_t)s;
  uint32_t mask = (uint32_t)(capacity - 1);
  int g = grid_for(n_out, 128);
  if (kernel_size == 3)
    k_kernel_map_probe<3><<<g, 128, 0, st>>>((const int4*)out_coords, n_out, table_keys, table_vals, mask, sx, sy, sz, nbr);
  else if (kernel_size == 5)
    k_kernel_map_probe<5><<<g, 128, 0, st>>>((const int4*)out_coords, n_out, table_keys, table_vals, mask, sx, sy, sz, nbr);
  else
    k_kernel_map_probe<1><<<g, 128, 0, st>>>((const int4*)out_coords, n_out, table_keys, table_vals, mask, sx, sy, sz, nbr);
  PASCO_CHECK_LAUNCH("pasco_kernel_map_probe");
  return 0;
}

// anisotropic odd box kernel (kx,ky,kz), offsets x fastest — dense bottleneck kernels (3,3,1) (5,5,3) (7,7,5)
__global__ void k_kernel_map_box(const int4* __restrict__ out_coords, int64_t n, const uint64_t* __restrict__ keys,
                                 const int32_t* __restrict__ vals, uint32_t mask, int kx, int ky, int kz, int sx, int sy,
                                 int sz, int32_t* __restrict__ nbr) {
  const int K = kx * ky * kz;
  const int64_t total = n * K;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int k = (int)(t / n);
    const int64_t o = t - (int64_t)k * n;
    const int dx = k % kx - kx / 2, dy = (k / kx) % ky - ky / 2, dz = k / (kx * ky) - kz / 2;
    int4 c = __ldg(out_coords + o);
    nbr[t] = table_find(keys, vals, mask, pack_key(c.x, c.y + dx * sx, c.z + dy * sy, c.w + dz * sz));
  }
}

extern "C" int pasco_kernel_map_box(const int32_t* out_coords, int64_t n_out, const uint64_t* table_keys,
                                    const int32_t* table_vals, int64_t capacity, int32_t kx, int32_t ky, int32_t kz,
                                    int32_t sx, int32_t sy, int32_t sz, int32_t* nbr, pasco_stream_t s) {
  PASCO_CHECK_ARG(kx % 2 == 1 && ky % 2 == 1 && kz % 2 == 1 && kx <= 15 && ky <= 15 && kz <= 15,
                  "pasco_kernel_map_box: kernel sizes must be odd and <= 15 (got %d,%d,%d)", kx, ky, kz);
  PASCO_CHECK_ARG(is_pow2(capacity), "pasco_kernel_map_box: capacity must be a power of two");
  if (n_out == 0) return 0;
  k_kernel_map_box<<<grid_for(n_out * kx * ky * kz, 256), 256, 0, (cudaStream_t)s>>>(
      (const int4*)out_coords, n_out, table_keys, table_vals, (uint32_t)(capacity - 1), kx, ky, kz, sx, sy, sz, nbr);
  PASCO_CHECK_LAUNCH("pasco_kernel_map_box");
  return 0;
}

__global__ void k_kernel_map_down(const int4* __restrict__ child, int64_t n, const uint64_t* __restrict__ keys,
                                  const int32_t* __restrict__ vals, uint32_t mask, int ks, int sx, int sy, int sz,
                                  int32_t* __restrict__ parent_of, int32_t* __restrict__ slot_of,
                                  int32_t* __restrict__ nbr, int64_t n_parent) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int4 c = __ldg(child + i);
    int px = floor_div(c.y, sx * ks) * sx * ks, py = floor_div(c.z, sy * ks) * sy * ks,
        pz = floor_div(c.w, sz * ks) * sz * ks;
    int p = table_find(keys, vals, mask, pack_key(c.x, px, py, pz));
    int k = (c.y - px) / sx + ks * ((c.z - py) / sy) + ks * ks * ((c.w - pz) / sz);
    if (parent_of) parent_of[i] = p;
    if (slot_of) slot_of[i] = k;
    if (nbr && p >= 0) nbr[(int64_t)k * n_parent + p] = (int)i;
  }
}

extern "C" int pasco_kernel_map_down(const int32_t* child_coords, int64_t n_child, const uint64_t* table_keys,
                                     const int32_t* table_vals, int64_t capacity, int32_t ks, int32_t child_sx,
                                     int32_t child_sy, int32_t child_sz, int32_t* parent_of, int32_t* slot_of,
                                     int32_t* nbr, int64_t n_parent, pasco_stream_t s) {
  PASCO_CHECK_ARG(ks >= 1 && ks <= 8, "pasco_kernel_map_down: kernel size out of range");
  PASCO_CHECK_ARG(is_pow2(capacity), "pasco_kernel_map_down: capacity must be a power of two");
  if (n_child == 0) return 0;
  k_kernel_map_down<<<grid_for(n_child, 256), 256, 0, (cudaStream_t)s>>>(
      (const int4*)child_coords, n_child, table_keys, table_vals, (uint32_t)(capacity - 1), ks, child_sx, child_sy,
      child_sz, parent_of, slot_of, nbr, n_parent);
  PASCO_CHECK_LAUNCH("pasco_kernel_map_down");
  return 0;
}

// ------------------------------------------------------------------------------------------------
// order-preserving compaction
// ------------------------------------------------------------------------------------------------
constexpr int kCompactBlock = 1024;

__global__ void k_mask_block_counts(const uint8_t* __restrict__ mask, int64_t n, int32_t* __restrict__ counts) {
  int64_t i = (int64_t)blockIdx.x * kCompactBlock + threadIdx.x;
  int keep = (i < n) && mask[i];
  int c = __syncthreads_count(keep);
  if (threadIdx.x == 0) counts[blockIdx.x] = c;
}

__global__ void k_mask_compact(const uint8_t* __restrict__ mask, int64_t n, const int32_t* __restrict__ offsets,
                               int32_t* __restrict__ new_row, int32_t* __restrict__ kept_rows) {
  __shared__ int warp_sum[32];
  int64_t i = (int64_t)blockIdx.x * kCompactBlock + threadIdx.x;
  int keep = (i < n) && mask[i];
  unsigned b = __ballot_sync(0xffffffffu, keep);
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int pre = __popc(b & ((1u << lane) - 1));
  if (lane == 0) warp_sum[w] = __popc(b);
  __syncthreads();
  if (w == 0) {
    int v = warp_sum[lane];
    int incl = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      int t = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += t;
    }
    warp_sum[lane] = incl - v;
  }
  __syncthreads();
  if (i < n) {
    int pos = offsets[blockIdx.x] + warp_sum[w] + pre;
    if (new_row) new_row[i] = keep ? pos : -1;
    if (keep && kept_rows) kept_rows[pos] = (int)i;
  }
}

extern "C" int pasco_mask_block_counts(const uint8_t* mask, int64_t n, int32_t* block_counts, pasco_stream_t s) {
  if (n == 0) return 0;
  int64_t nb = (n + kCompactBlock - 1) / kCompactBlock;
  k_mask_block_counts<<<(unsigned)nb, kCompactBlock, 0, (cudaStream_t)s>>>(mask, n, block_counts);
  PASCO_CHECK_LAUNCH("pasco_mask_block_counts");
  return 0;
}

extern "C" int pasco_mask_compact(const uint8_t* mask, int64_t n, const int32_t* block_offsets, int32_t* new_row,
                                  int32_t* kept_rows, pasco_stream_t s) {
  if (n == 0) return 0;
  int64_t nb = (n + kCompactBlock - 1) / kCompactBlock;
  k_mask_compact<<<(unsigned)nb, kCompactBlock, 0, (cudaStream_t)s>>>(mask, n, block_offsets, new_row, kept_rows);
  PASCO_CHECK_LAUNCH("pasco_mask_compact");
  return 0;
}

// ------------------------------------------------------------------------------------------------
// row gather / scatter
// ------------------------------------------------------------------------------------------------
template <typename V>
__global__ void k_gather_rows(const V* __restrict__ src, const int32_t* __restrict__ rows, int64_t n_rows, int cv,
                              V* __restrict__ out) {
  int64_t total = n_rows * cv;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = t / cv;
    int c = (int)(t - r * cv);
    int sr = __ldg(rows + r);
    V v;
    if (sr >= 0)
      v = __ldg(src + (int64_t)sr * cv + c);
    else
      memset(&v, 0, sizeof(V));
    out[t] = v;
  }
}

template <typename V, bool ACC>
__global__ void k_scatter_rows(const V* __restrict__ src, const int32_t* __restrict__ rows, int64_t n_rows, int cv,
                               V* __restrict__ dst) {
  int64_t total = n_rows * cv;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = t / cv;
    int c = (int)(t - r * cv);
    int dr = __ldg(rows + r);
    if (dr < 0) continue;
    V v = __ldg(src + t);
    V* p = dst + (int64_t)dr * cv + c;
    if constexpr (ACC) {
      V o = *p;
      if constexpr (sizeof(V) == 16) {
        o.x += v.x; o.y += v.y; o.z += v.z; o.w += v.w;
      } else {
        o += v;
      }
      *p = o;
    } else {
      *p = v;
    }
  }
}

extern "C" int pasco_gather_rows(const float* src, const int32_t* rows, int64_t n_rows, int32_t C, float* out,
                                 pasco_stream_t s) {
  if (n_rows == 0 || C == 0) return 0;
  cudaStream_t st = (cudaStream_t)s;
  bool vec = (C % 4 == 0) && (((uintptr_t)src | (uintptr_t)out) % 16 == 0);
  if (vec)
    k_gather_rows<float4><<<grid_for(n_rows * (C / 4), 256), 256, 0, st>>>((const float4*)src, rows, n_rows, C / 4,
                                                                           (float4*)out);
  else
    k_gather_rows<float><<<grid_for(n_rows * C, 256), 256, 0, st>>>(src, rows, n_rows, C, out);
  PASCO_CHECK_LAUNCH("pasco_gather_rows");
  return 0;
}

extern "C" int pasco_scatter_rows(const float* src, const int32_t* rows, int64_t n_rows, int32_t C, float* dst,
                                  int32_t accumulate, pasco_stream_t s) {
  if (n_rows == 0 || C == 0) return 0;
  cudaStream_t st = (cudaStream_t)s;
  bool vec = (C % 4 == 0) && (((uintptr_t)src | (uintptr_t)dst) % 16 == 0);
  if (vec) {
    int g = grid_for(n_rows * (C / 4), 256);
    if (accumulate)
      k_scatter_rows<float4, true><<<g, 256, 0, st>>>((const float4*)src, rows, n_rows, C / 4, (float4*)dst);
    else
      k_scatter_rows<float4, false><<<g, 256, 0, st>>>((const float4*)src, rows, n_rows, C / 4, (float4*)dst);
  } else {
    int g = grid_for(n_rows * C, 256);
    if (accumulate)
      k_scatter_rows<float, true><<<g, 256, 0, st>>>(src, rows, n_rows, C, dst);
    else
      k_scatter_rows<float, false><<<g, 256, 0, st>>>(src, rows, n_rows, C, dst);
  }
  PASCO_CHECK_LAUNCH("pasco_scatter_rows");
  return 0;
}

extern "C" int pasco_gather_coords(const int32_t* src, const int32_t* rows, int64_t n_rows, int32_t* out,
                                   pasco_stream_t s) {
  if (n_rows == 0) return 0;
  k_gather_rows<int4><<<grid_for(n_rows, 256), 256, 0, (cudaStream_t)s>>>((const int4*)src, rows, n_rows, 1, (int4*)out);
  PASCO_CHECK_LAUNCH("pasco_gather_coords");
  return 0;
}

// ------------------------------------------------------------------------------------------------
// dense <-> sparse
// ------------------------------------------------------------------------------------------------
struct DenseGeom {
  int min_c[3], stride[3];
  int B, X, Y, Z;
};

template <bool TO_DENSE>
__global__ void k_dense_xfer(float* __restrict__ feats, const int4* __restrict__ coords, int64_t n, int C,
                             DenseGeom g, float* __restrict__ dense, int* __restrict__ err) {
  int64_t total = n * C;
  int64_t cells = (int64_t)g.X * g.Y * g.Z;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    int64_t i = t / C;
    int c = (int)(t - i * C);
    int4 q = __ldg(coords + i);
    int x = floor_div(q.y - g.min_c[0], g.stride[0]), y = floor_div(q.z - g.min_c[1], g.stride[1]),
        z = floor_div(q.w - g.min_c[2], g.stride[2]);
    if (q.x < 0 || q.x >= g.B || x < 0 || x >= g.X || y < 0 || y >= g.Y || z < 0 || z >= g.Z) {
      if (err) *err = 1;
      if (!TO_DENSE) feats[t] = 0.f;      // a row outside the volume reads as zero (never uninitialised memory)
      continue;
    }
    int64_t d = ((int64_t)q.x * C + c) * cells + ((int64_t)x * g.Y + y) * g.Z + z;
    if (TO_DENSE)
      dense[d] = feats[t];
    else
      feats[t] = dense[d];
  }
}

static DenseGeom make_geom(const int32_t min_c[3], const int32_t stride[3], int B, int X, int Y, int Z) {
  DenseGeom g;
  for (int i = 0; i < 3; ++i) {
    g.min_c[i] = min_c[i];
    g.stride[i] = stride[i];
  }
  g.B = B; g.X = X; g.Y = Y; g.Z = Z;
  return g;
}

extern "C" int pasco_to_dense(const float* feats, const int32_t* coords, int64_t n, int32_t C, const int32_t min_c[3],
                              const int32_t stride[3], float* dense, int32_t B, int32_t X, int32_t Y, int32_t Z,
                              int32_t* err_flag, pasco_stream_t s) {
  PASCO_CHECK_ARG(stride[0] > 0 && stride[1] > 0 && stride[2] > 0, "pasco_to_dense: bad stride");
  if (n == 0 || C == 0) return 0;
  k_dense_xfer<true><<<grid_for(n * C, 256), 256, 0, (cudaStream_t)s>>>(
      const_cast<float*>(feats), (const int4*)coords, n, C, make_geom(min_c, stride, B, X, Y, Z), dense, err_flag);
  PASCO_CHECK_LAUNCH("pasco_to_dense");
  return 0;
}

extern "C" int pasco_from_dense(const float* dense, const int32_t* coords, int64_t n, int32_t C,
                                const int32_t min_c[3], const int32_t stride[3], float* feats, int32_t B, int32_t X,
                                int32_t Y, int32_t Z, int32_t* err_flag, pasco_stream_t s) {
  PASCO_CHECK_ARG(stride[0] > 0 && stride[1] > 0 && stride[2] > 0, "pasco_from_dense: bad stride");
  if (n == 0 || C == 0) return 0;
  k_dense_xfer<false><<<grid_for(n * C, 256), 256, 0, (cudaStream_t)s>>>(
      feats, (const int4*)coords, n, C, make_geom(min_c, stride, B, X, Y, Z), const_cast<float*>(dense), err_flag);
  PASCO_CHECK_LAUNCH("pasco_from_dense");
  return 0;
}

__global__ void k_dense_occupancy(const float* __restrict__ dense, int B, int C, int64_t cells,
                                  uint8_t* __restrict__ mask) {
  int64_t total = (int64_t)B * cells;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    int64_t b = t / cells, cell = t - b * cells;
    const float* p = dense + b * C * cells + cell;
    float acc = 0.f;
    for (int c = 0; c < C; ++c) acc += fabsf(__ldg(p + (int64_t)c * cells));
    mask[t] = acc != 0.f;
  }
}

extern "C" int pasco_dense_occupancy(const float* dense, int32_t B, int32_t C, int64_t cells, uint8_t* mask,
                                     pasco_stream_t s) {
  if ((int64_t)B * cells == 0) return 0;
  k_dense_occupancy<<<grid_for((int64_t)B * cells, 256), 256, 0, (cudaStream_t)s>>>(dense, B, C, cells, mask);
  PASCO_CHECK_LAUNCH("pasco_dense_occupancy");
  return 0;
}
