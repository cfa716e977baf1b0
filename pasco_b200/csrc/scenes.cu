// SemanticKITTI scene preparation on the device (sm_90a): what KittiDataset.get_individual (kitti_dataset.py:142-288,
// 329-490) and collate_fn compute from one scan's files, with the reference's fp32 / fp64 sequences restated so the
// results carry its bits.
//
//   pasco_scene_source      source cells: forward-transform bounds of the labelled cells (transform_scene step 1) and
//                           the classes / instance ids present in the untransformed volumes
//   pasco_scene_resample    every cell of the transformed box: inverse transform of its centre and a nearest sample of
//                           label + 1 (transform_scene steps 2-4, grid_sample(align_corners=True, mode="nearest"))
//   pasco_scene_crop        the training crop's bounds from the semantic rows' extent and the host's np.random.rand(3)
//   pasco_scene_crop_stats  extent, classes and instance ids of the rows the crop keeps
//   pasco_scene_points      the point path's extent filter, voxel coordinates, transform and crop flags
//   pasco_scene_point_rows  the kept points' feature rows and coordinates, and the extent-filtered pass-through fields
//   pasco_scene_box         the dense semantic / instance / completion volumes on the item's box
//   pasco_scene_scale       the scale-2 / scale-4 semantic and geometry labels, one pass per scale
//   pasco_scene_masks       prepare_mask_label's labels and bool masks after one zero fill
//
// Every reduction is an integer atomic (min, max, add) or a store of a constant flag, so no output depends on the order
// in which threads run.
#include <limits.h>
#include <math.h>

#include "common.cuh"

using namespace pasco;

namespace {

constexpr int kBlock = 256;

struct Mat4 {
  float m[16];          // row-major 4x4
};

// the fixed grid of transform_utils.transform: min_bound (fp32 tensor), resolution 0.2, resolution / 2
__device__ __constant__ float kMinBound[3] = {0.f, -25.6f, -2.f};

// T @ [p, 1] for row a in fp32: a chain of fused multiply-adds in k order, as a CPU sgemm kernel accumulates
__device__ __forceinline__ float mat_row(const Mat4& T, int a, float p0, float p1, float p2) {
  float acc = __fmul_rn(T.m[4 * a + 0], p0);
  acc = __fmaf_rn(T.m[4 * a + 1], p1, acc);
  acc = __fmaf_rn(T.m[4 * a + 2], p2, acc);
  return __fadd_rn(acc, T.m[4 * a + 3]);
}

// (new_points − min_bound − resolution / 2) / resolution, torch.round (half to even), .int()
__device__ __forceinline__ int to_cell(float h, int a) {
  return (int)rintf(__fdiv_rn(__fsub_rn(__fsub_rn(h, kMinBound[a]), 0.1f), 0.2f));
}

// transform(coords, T) of integer cells: coords * 0.2 + 0.1 + min_bound, all fp32
__device__ __forceinline__ void transform_cell(const Mat4& T, int x, int y, int z, int out[3]) {
  const float p0 = __fadd_rn(__fadd_rn(__fmul_rn((float)x, 0.2f), 0.1f), kMinBound[0]);
  const float p1 = __fadd_rn(__fadd_rn(__fmul_rn((float)y, 0.2f), 0.1f), kMinBound[1]);
  const float p2 = __fadd_rn(__fadd_rn(__fmul_rn((float)z, 0.2f), 0.1f), kMinBound[2]);
  out[0] = to_cell(mat_row(T, 0, p0, p1, p2), 0);
  out[1] = to_cell(mat_row(T, 1, p0, p1, p2), 1);
  out[2] = to_cell(mat_row(T, 2, p0, p1, p2), 2);
}

// sample_grid_features' normalisation ((c / (n − 1) − 0.5) · 2) and grid_sample's align-corners unnormalisation
// (((g + 1) / 2) · (n − 1)), fp32, then nearbyint: the nearest source index along an axis of n cells, −1 outside
__device__ __forceinline__ int grid_index(int c, int n) {
  const float nm1 = (float)(n - 1);
  const float g = __fmul_rn(__fsub_rn(__fdiv_rn((float)c, nm1), 0.5f), 2.f);
  const int i = (int)rintf(__fmul_rn(__fdiv_rn(__fadd_rn(g, 1.f), 2.f), nm1));
  return (i >= 0 && i < n) ? i : -1;
}

// numpy's floor_divide for doubles (npy_divmod): fmod, the sign correction, then the floor with its 0.5 guard
__device__ __forceinline__ double np_floor_divide(double a, double b) {
  double mod = fmod(a, b);
  double div = (a - mod) / b;
  if (mod != 0.0) {
    if ((b < 0) != (mod < 0)) div -= 1.0;
  }
  double fl;
  if (div != 0.0) {
    fl = floor(div);
    if (div - fl > 0.5) fl += 1.0;
  } else {
    fl = copysign(0.0, a / b);
  }
  return fl;
}

__device__ __constant__ double kVoxOrigin[3] = {0.0, -25.6, -2.0};

// the crop's half-open test on the first two axes, in fp64 as torch compares an integer tensor with a float64 one
__device__ __forceinline__ bool in_crop(const double* __restrict__ bnd, double x, double y) {
  return x >= bnd[0] && x < bnd[2] && y >= bnd[1] && y < bnd[3];
}

// per-thread extents → one atomic per warp
__device__ __forceinline__ void flush_extent(int32_t* __restrict__ lo_out, int32_t* __restrict__ hi_out, const int lo[3],
                                             const int hi[3]) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const int l = __reduce_min_sync(0xffffffffu, lo[a]);
    const int h = __reduce_max_sync(0xffffffffu, hi[a]);
    if (lane == 0) {
      if (l != INT_MAX) atomicMin(lo_out + a, l);
      if (h != INT_MIN) atomicMax(hi_out + a, h);
    }
  }
}

__device__ __forceinline__ void flush_count(int32_t* __restrict__ out, int v) {
  const int s = __reduce_add_sync(0xffffffffu, v);
  if ((threadIdx.x & 31) == 0 && s) atomicAdd(out, s);
}

__device__ __forceinline__ void flush_flags(const int* s_flags, int32_t* __restrict__ out) {
  __syncthreads();
  for (int i = threadIdx.x; i < 256; i += blockDim.x)
    if (s_flags[i]) out[i] = 1;
}

__global__ void k_scene_stats_init(int32_t* __restrict__ stats) {
  for (int i = threadIdx.x; i < PASCO_SCENE_STATS; i += blockDim.x) {
    int v = 0;
    if ((i >= PASCO_SCENE_BND && i < PASCO_SCENE_BND + 3) || (i >= PASCO_SCENE_SEM_EXT && i < PASCO_SCENE_SEM_EXT + 3) ||
        (i >= PASCO_SCENE_BOX && i < PASCO_SCENE_BOX + 3))
      v = INT_MAX;
    if ((i >= PASCO_SCENE_BND + 3 && i < PASCO_SCENE_BND + 6) ||
        (i >= PASCO_SCENE_SEM_EXT + 3 && i < PASCO_SCENE_SEM_EXT + 6) || (i >= PASCO_SCENE_BOX + 3 && i < PASCO_SCENE_BOX + 6))
      v = INT_MIN;
    stats[i] = v;
  }
}

// ------------------------------------------------------------------------------------------------
// source cells: transform(nonzero(semantic != 255), T)'s min / max, and the flags of the untransformed volumes
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBlock) k_scene_source(const uint8_t* __restrict__ sem, const uint8_t* __restrict__ inst,
                                                         int X, int Y, int Z, Mat4 T, int32_t* __restrict__ stats) {
  __shared__ int s_cls[256], s_inst[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) s_cls[i] = s_inst[i] = 0;
  __syncthreads();
  int lo[3] = {INT_MAX, INT_MAX, INT_MAX}, hi[3] = {INT_MIN, INT_MIN, INT_MIN};
  int n_lab = 0, n_inst = 0;
  const int64_t cells = (int64_t)X * Y * Z;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < cells; i += (int64_t)gridDim.x * blockDim.x) {
    const int s = __ldg(sem + i), n = __ldg(inst + i);
    s_cls[s] = 1;
    if (n != 0) {
      s_inst[n] = 1;
      ++n_inst;
    }
    if (s == 255) continue;
    ++n_lab;
    const int z = (int)(i % Z), y = (int)((i / Z) % Y), x = (int)(i / ((int64_t)Y * Z));
    int c[3];
    transform_cell(T, x, y, z, c);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      lo[a] = min(lo[a], c[a]);
      hi[a] = max(hi[a], c[a]);
    }
  }
  flush_extent(stats + PASCO_SCENE_BND, stats + PASCO_SCENE_BND + 3, lo, hi);
  flush_count(stats + PASCO_SCENE_N_LABELLED, n_lab);
  flush_count(stats + PASCO_SCENE_N_INSTANCE, n_inst);
  flush_flags(s_cls, stats + PASCO_SCENE_CLS_ORIGIN);
  flush_flags(s_inst, stats + PASCO_SCENE_INST_ORIGIN);
}

// ------------------------------------------------------------------------------------------------
// every cell of the box [lo, lo + G): label + 1 (uint8, so 255 wraps to 0 = no row) at the nearest source cell of its
// inverse-transformed centre, 0 outside the source; the extent and count of the semantic rows
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBlock) k_scene_resample(const uint8_t* __restrict__ sem, const uint8_t* __restrict__ inst,
                                                           int X, int Y, int Z, Mat4 Ti, int lx, int ly, int lz, int GX,
                                                           int GY, int GZ, int with_inst, uint8_t* __restrict__ gs,
                                                           uint8_t* __restrict__ gi, int32_t* __restrict__ stats) {
  int lo[3] = {INT_MAX, INT_MAX, INT_MAX}, hi[3] = {INT_MIN, INT_MIN, INT_MIN};
  int n_rows = 0;
  const int64_t cells = (int64_t)GX * GY * GZ;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i0 = blockIdx.x * (int64_t)blockDim.x; i0 < cells; i0 += stride) {
    const int64_t j = i0 + threadIdx.x;
    if (j >= cells) break;
    const int x = lx + (int)(j / ((int64_t)GY * GZ)), y = ly + (int)((j / GZ) % GY), z = lz + (int)(j % GZ);
    int p[3];
    transform_cell(Ti, x, y, z, p);
    const int sx = grid_index(p[0], X), sy = grid_index(p[1], Y), sz = grid_index(p[2], Z);
    uint8_t v = 0, w = 0;
    if (sx >= 0 && sy >= 0 && sz >= 0) {
      const int64_t src = ((int64_t)sx * Y + sy) * Z + sz;
      v = (uint8_t)(__ldg(sem + src) + 1);
      if (with_inst) w = (uint8_t)(__ldg(inst + src) + 1);
    }
    gs[j] = v;
    if (with_inst) gi[j] = w;
    if (v) {
      ++n_rows;
      lo[0] = min(lo[0], x), lo[1] = min(lo[1], y), lo[2] = min(lo[2], z);
      hi[0] = max(hi[0], x), hi[1] = max(hi[1], y), hi[2] = max(hi[2], z);
    }
  }
  __syncwarp();
  flush_extent(stats + PASCO_SCENE_SEM_EXT, stats + PASCO_SCENE_SEM_EXT + 3, lo, hi);
  flush_count(stats + PASCO_SCENE_N_SEM_ROWS, n_rows);
}

// crop (kitti_dataset.py:464-471): crop_size = (max − min) * 0.8 in fp32 (an int32 tensor times a Python float); the
// draw promotes (max − min − crop_size) to fp64; new_min = min + that, new_max = new_min + crop_size.  Without a crop
// the bounds are ±inf.  bnd = (new_min x, new_min y, new_max x, new_max y).
__global__ void k_scene_crop(const int32_t* __restrict__ stats, double r0, double r1, int train, double* __restrict__ bnd) {
  if (threadIdx.x != 0) return;
  if (!train) {
    bnd[0] = bnd[1] = -INFINITY;
    bnd[2] = bnd[3] = INFINITY;
    return;
  }
  const double r[2] = {r0, r1};
#pragma unroll
  for (int a = 0; a < 2; ++a) {
    const int mn = stats[PASCO_SCENE_SEM_EXT + a], mx = stats[PASCO_SCENE_SEM_EXT + 3 + a];
    const float size = __fmul_rn((float)(mx - mn), 0.8f);
    const float room = __fsub_rn((float)(mx - mn), size);
    const double nmin = __dadd_rn((double)mn, __dmul_rn((double)room, r[a]));
    bnd[a] = nmin;
    bnd[2 + a] = __dadd_rn(nmin, (double)size);
  }
}

// ------------------------------------------------------------------------------------------------
// the rows the crop keeps: their extent (semantic ∪ instance rows), the classes of the semantic rows, the ids of the
// instance rows, and the number of semantic rows
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBlock) k_scene_crop_stats(const uint8_t* __restrict__ gs, const uint8_t* __restrict__ gi,
                                                             int lx, int ly, int lz, int GX, int GY, int GZ, int with_inst,
                                                             const double* __restrict__ bnd, int32_t* __restrict__ stats) {
  __shared__ int s_cls[256], s_inst[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) s_cls[i] = s_inst[i] = 0;
  __syncthreads();
  const double b[4] = {bnd[0], bnd[1], bnd[2], bnd[3]};
  int lo[3] = {INT_MAX, INT_MAX, INT_MAX}, hi[3] = {INT_MIN, INT_MIN, INT_MIN};
  int n_sem = 0;
  const int64_t cells = (int64_t)GX * GY * GZ;
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < cells; j += (int64_t)gridDim.x * blockDim.x) {
    const int v = gs[j], w = with_inst ? gi[j] : 0;
    if (!v && !w) continue;
    const int x = lx + (int)(j / ((int64_t)GY * GZ)), y = ly + (int)((j / GZ) % GY), z = lz + (int)(j % GZ);
    if (!in_crop(b, (double)x, (double)y)) continue;
    if (v) {
      s_cls[v - 1] = 1;
      ++n_sem;
    }
    if (w) s_inst[w - 1] = 1;
    lo[0] = min(lo[0], x), lo[1] = min(lo[1], y), lo[2] = min(lo[2], z);
    hi[0] = max(hi[0], x), hi[1] = max(hi[1], y), hi[2] = max(hi[2], z);
  }
  flush_extent(stats + PASCO_SCENE_BOX, stats + PASCO_SCENE_BOX + 3, lo, hi);
  flush_count(stats + PASCO_SCENE_N_SEM_KEPT, n_sem);
  flush_flags(s_cls, stats + PASCO_SCENE_CLS);
  flush_flags(s_inst, stats + PASCO_SCENE_INST);
}

// ------------------------------------------------------------------------------------------------
// points (load_data_v3 lines 369-431, voxelize): extent filter, voxel coordinates xyz − vox_origin floor-divided by 0.2
// in fp64, transform(in_coords, T) — coords * 0.2 + 0.1 + min_bound in fp64, cast to fp32 by type_as(T) — and the crop
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool point_in_extent(float x, float y, float z) {
  // numpy compares the fp32 coordinates with np.float64 lower bounds in fp64 and with Python-float upper bounds in fp32;
  // no fp32 value lies between 51.2, 25.6 or 4.4 and its fp32 rounding, so fp64 compares give the same flags
  return (double)x < 51.2 && (double)x >= 0.0 && (double)y < 25.6 && (double)y >= -25.6 && (double)z < 4.4 &&
         (double)z >= -2.0;
}

__device__ __forceinline__ void point_cell(const Mat4& T, float x, float y, float z, double vc[3], int64_t out[3]) {
  const float xyz[3] = {x, y, z};
  float p[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    vc[a] = np_floor_divide((double)xyz[a] - kVoxOrigin[a], 0.2);
    p[a] = (float)__dadd_rn((double)kMinBound[a], __dadd_rn(__dmul_rn(vc[a], 0.2), 0.1));
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) out[a] = (int64_t)to_cell(mat_row(T, a, p[0], p[1], p[2]), a);
}

__global__ void __launch_bounds__(kBlock) k_scene_points(const float* __restrict__ pts, int64_t N, int pitch, Mat4 T,
                                                         const double* __restrict__ bnd, uint8_t* __restrict__ ext,
                                                         uint8_t* __restrict__ keep, int32_t* __restrict__ stats) {
  const double b[4] = {bnd[0], bnd[1], bnd[2], bnd[3]};
  int n_ext = 0, n_keep = 0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i0 = blockIdx.x * (int64_t)blockDim.x; i0 < N; i0 += stride) {
    const int64_t i = i0 + threadIdx.x;
    if (i >= N) break;
    const float x = __ldg(pts + i * pitch), y = __ldg(pts + i * pitch + 1), z = __ldg(pts + i * pitch + 2);
    const bool e = point_in_extent(x, y, z);
    bool k = false;
    if (e) {
      double vc[3];
      int64_t c[3];
      point_cell(T, x, y, z, vc, c);
      k = in_crop(b, (double)c[0], (double)c[1]);
    }
    ext[i] = e;
    keep[i] = k;
    n_ext += e;
    n_keep += k;
  }
  __syncwarp();
  flush_count(stats + PASCO_SCENE_N_POINTS, n_ext);
  flush_count(stats + PASCO_SCENE_N_POINTS_KEPT, n_keep);
}

// one thread per (kept row, column): [vote, intensity, radius, embedding, xyz − voxel centre, xyz] cast to fp32
__global__ void __launch_bounds__(kBlock) k_scene_point_rows(const float* __restrict__ pts, int pitch,
                                                             const float* __restrict__ vote, int V,
                                                             const float* __restrict__ emb, int E, int64_t N,
                                                             const int32_t* __restrict__ rows, int64_t n_rows, Mat4 T,
                                                             float* __restrict__ feats, int64_t* __restrict__ coords) {
  const int I = pitch - 3, Fw = V + I + 1 + E + 6;
  const int64_t total = n_rows * Fw;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / Fw;
    const int col = (int)(t % Fw);
    const int64_t i = __ldg(rows + r);
    const float* p = pts + i * pitch;
    float out;
    if (col < V) {
      out = __ldg(vote + i * V + col);
    } else if (col < V + I) {
      out = __ldg(p + 3 + (col - V));
    } else if (col == V + I) {                         // np.linalg.norm: sqrt of the sequential fp32 sum of squares
      const float x = __ldg(p), y = __ldg(p + 1), z = __ldg(p + 2);
      out = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
    } else if (col < V + I + 1 + E) {
      out = __ldg(emb + (int64_t)(col - V - I - 1) * N + i);   // embedding[idx] is [E, N]; the row is its .T
    } else {
      const int a = col - (V + I + 1 + E);
      const float x = __ldg(p + (a % 3));
      if (a < 3) {                                     // xyz − ((float32(coords) + 0.5) * 0.2 + vox_origin)
        const double c = np_floor_divide((double)x - kVoxOrigin[a], 0.2);
        const double centre = (double)__fmul_rn(__fadd_rn((float)c, 0.5f), 0.2f) + kVoxOrigin[a];
        out = (float)((double)x - centre);
      } else {
        out = x;
      }
      if (a == 0) {
        double vc[3];
        int64_t c[3];
        point_cell(T, __ldg(p), __ldg(p + 1), __ldg(p + 2), vc, c);
        coords[r * 3 + 0] = c[0], coords[r * 3 + 1] = c[1], coords[r * 3 + 2] = c[2];
      }
    }
    feats[t] = out;
  }
}

// the extent-filtered pass-through fields: xyz − vox_origin in fp64, and the .label words & 0xFFFF
__global__ void __launch_bounds__(kBlock) k_scene_point_pass(const float* __restrict__ pts, int pitch,
                                                             const int32_t* __restrict__ label,
                                                             const int32_t* __restrict__ rows, int64_t n_rows,
                                                             double* __restrict__ xyz, int32_t* __restrict__ label_out) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n_rows; r += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = __ldg(rows + r);
#pragma unroll
    for (int a = 0; a < 3; ++a) xyz[r * 3 + a] = (double)__ldg(pts + i * pitch + a) - kVoxOrigin[a];
    label_out[r] = __ldg(label + i) & 0xFFFF;
  }
}

// ------------------------------------------------------------------------------------------------
// the dense volumes on the item's box [b, b + S): semantic (fill 255), instance (fill 0) from the kept rows, and the
// completion label complete_voxel.type(uint8): 0 empty, 1 labelled, 255 unknown
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBlock) k_scene_box(const uint8_t* __restrict__ gs, const uint8_t* __restrict__ gi,
                                                      int lx, int ly, int lz, int GX, int GY, int GZ, int with_inst,
                                                      const double* __restrict__ bnd, int bx, int by, int bz, int SX,
                                                      int SY, int SZ, uint8_t* __restrict__ sem, uint8_t* __restrict__ inst,
                                                      uint8_t* __restrict__ geo) {
  const double b[4] = {bnd[0], bnd[1], bnd[2], bnd[3]};
  const int64_t cells = (int64_t)SX * SY * SZ;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < cells; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = bx + (int)(i / ((int64_t)SY * SZ)), y = by + (int)((i / SZ) % SY), z = bz + (int)(i % SZ);
    const int gx = x - lx, gy = y - ly, gz = z - lz;
    int s = 255, n = 0;
    if (gx >= 0 && gx < GX && gy >= 0 && gy < GY && gz >= 0 && gz < GZ && in_crop(b, (double)x, (double)y)) {
      const int64_t j = ((int64_t)gx * GY + gy) * GZ + gz;
      const int v = gs[j];
      if (v) s = v - 1;
      if (with_inst && gi[j]) n = gi[j] - 1;
    }
    sem[i] = (uint8_t)s;
    inst[i] = (uint8_t)n;
    geo[i] = (uint8_t)(s == 255 ? 255 : (s > 0 ? 1 : 0));
  }
}

// ------------------------------------------------------------------------------------------------
// one s³ block per thread (kitti_dataset.py:217-266): geometry = max of the occupied flags, 255 when all s³ cells are
// 255; semantics = the first class of 1-19 with the largest count (avg_pool of a one-hot is count / s³, exact), and
// when no cell has one of them, 0 if every cell is 255 and 255 otherwise.  Counts live in shared memory.
// ------------------------------------------------------------------------------------------------
template <int S>
__global__ void __launch_bounds__(kBlock) k_scene_scale(const uint8_t* __restrict__ sem, int X, int Y, int Z,
                                                        uint8_t* __restrict__ sem_out, uint8_t* __restrict__ geo_out) {
  __shared__ uint8_t s_cnt[20 * kBlock];
  uint8_t* cnt = s_cnt + threadIdx.x;
  const int OX = X / S, OY = Y / S, OZ = Z / S;
  const int64_t blocks = (int64_t)OX * OY * OZ;
  for (int64_t o = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; o < blocks; o += (int64_t)gridDim.x * blockDim.x) {
    for (int c = 1; c < 20; ++c) cnt[c * kBlock] = 0;
    const int ox = (int)(o / ((int64_t)OY * OZ)), oy = (int)((o / OZ) % OY), oz = (int)(o % OZ);
    int n255 = 0, occ = 0;
    for (int dx = 0; dx < S; ++dx)
      for (int dy = 0; dy < S; ++dy) {
        const uint8_t* row = sem + ((int64_t)(ox * S + dx) * Y + (oy * S + dy)) * Z + oz * S;
#pragma unroll
        for (int dz = 0; dz < S; ++dz) {
          const int v = __ldg(row + dz);
          if (v == 255) {
            ++n255;
          } else if (v != 0) {
            occ = 1;
            if (v < 20) cnt[v * kBlock] += 1;
          }
        }
      }
    int best = 0, best_n = 0;
    for (int c = 1; c < 20; ++c) {
      const int n = cnt[c * kBlock];
      if (n > best_n) best = c, best_n = n;
    }
    const bool all255 = n255 == S * S * S;
    geo_out[o] = all255 ? 255 : (uint8_t)occ;
    sem_out[o] = best ? (uint8_t)best : (all255 ? 0 : 255);
  }
}

// ------------------------------------------------------------------------------------------------
// prepare_mask_label (kitti_dataset.py:593-664): slot[c] (c = 0..255) is the mask of class c (stuff, ascending) and
// slot[256 + id] that of instance id (ascending after the stuff), −1 for none.  One pass writes both masks of a cell
// and takes each instance's first cell in C order (atomicMin of the linear index); a second gives the labels.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBlock) k_scene_masks(const uint8_t* __restrict__ sem, const uint8_t* __restrict__ inst,
                                                        int64_t cells, const int32_t* __restrict__ slot,
                                                        uint8_t* __restrict__ masks, int32_t* __restrict__ first) {
  __shared__ int s_slot[512];
  __shared__ int s_first[256];
  for (int i = threadIdx.x; i < 512; i += blockDim.x) s_slot[i] = slot[i];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) s_first[i] = INT_MAX;
  __syncthreads();
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < cells; i += (int64_t)gridDim.x * blockDim.x) {
    const int cs = s_slot[__ldg(sem + i)];
    if (cs >= 0) masks[(int64_t)cs * cells + i] = 1;
    const int id = __ldg(inst + i);
    const int is = s_slot[256 + id];
    if (is >= 0) {
      masks[(int64_t)is * cells + i] = 1;
      atomicMin(s_first + id, (int)min(i, (int64_t)INT_MAX - 1));
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 256; i += blockDim.x)
    if (s_first[i] != INT_MAX) atomicMin(first + i, s_first[i]);
}

__global__ void k_scene_mask_labels(const uint8_t* __restrict__ sem, const int32_t* __restrict__ slot,
                                    const int32_t* __restrict__ first, uint8_t* __restrict__ labels) {
  for (int i = threadIdx.x; i < 512; i += blockDim.x) {
    const int s = slot[i];
    if (s < 0) continue;
    labels[s] = i < 256 ? (uint8_t)i : __ldg(sem + first[i - 256]);
  }
}

__global__ void k_scene_fill_i32(int32_t* __restrict__ p, int n, int v) {
  for (int i = threadIdx.x; i < n; i += blockDim.x) p[i] = v;
}

Mat4 mat4(const float* T) {
  Mat4 m;
  for (int i = 0; i < 16; ++i) m.m[i] = T[i];
  return m;
}

}  // namespace

extern "C" int pasco_scene_source(const uint8_t* sem, const uint8_t* inst, int32_t X, int32_t Y, int32_t Z,
                                  const float T[16], int32_t* stats, pasco_stream_t s) {
  PASCO_CHECK_ARG(X >= 2 && Y >= 2 && Z >= 2, "pasco_scene_source: the volume needs at least 2 cells per axis");
  cudaStream_t st = (cudaStream_t)s;
  k_scene_stats_init<<<1, kBlock, 0, st>>>(stats);
  k_scene_source<<<grid_for((int64_t)X * Y * Z, kBlock), kBlock, 0, st>>>(sem, inst, X, Y, Z, mat4(T), stats);
  PASCO_CHECK_LAUNCH("pasco_scene_source");
  return 0;
}

extern "C" int pasco_scene_resample(const uint8_t* sem, const uint8_t* inst, int32_t X, int32_t Y, int32_t Z,
                                    const float Ti[16], const int32_t lo[3], const int32_t G[3], int32_t with_inst,
                                    uint8_t* gs, uint8_t* gi, int32_t* stats, pasco_stream_t s) {
  PASCO_CHECK_ARG(G[0] >= 1 && G[1] >= 1 && G[2] >= 1, "pasco_scene_resample: empty box");
  PASCO_CHECK_ARG(!with_inst || gi, "pasco_scene_resample: with_inst needs gi");
  const int64_t cells = (int64_t)G[0] * G[1] * G[2];
  k_scene_resample<<<grid_for(cells, kBlock), kBlock, 0, (cudaStream_t)s>>>(sem, inst, X, Y, Z, mat4(Ti), lo[0], lo[1],
                                                                            lo[2], G[0], G[1], G[2], with_inst, gs, gi,
                                                                            stats);
  PASCO_CHECK_LAUNCH("pasco_scene_resample");
  return 0;
}

extern "C" int pasco_scene_crop(const int32_t* stats, const double draw[3], int32_t train, double* bounds,
                                pasco_stream_t s) {
  k_scene_crop<<<1, 32, 0, (cudaStream_t)s>>>(stats, draw ? draw[0] : 0.0, draw ? draw[1] : 0.0, train, bounds);
  PASCO_CHECK_LAUNCH("pasco_scene_crop");
  return 0;
}

extern "C" int pasco_scene_crop_stats(const uint8_t* gs, const uint8_t* gi, const int32_t lo[3], const int32_t G[3],
                                      int32_t with_inst, const double* bounds, int32_t* stats, pasco_stream_t s) {
  const int64_t cells = (int64_t)G[0] * G[1] * G[2];
  k_scene_crop_stats<<<grid_for(cells, kBlock), kBlock, 0, (cudaStream_t)s>>>(gs, gi, lo[0], lo[1], lo[2], G[0], G[1],
                                                                              G[2], with_inst, bounds, stats);
  PASCO_CHECK_LAUNCH("pasco_scene_crop_stats");
  return 0;
}

extern "C" int pasco_scene_points(const float* pts, int64_t N, int32_t pitch, const float T[16], const double* bounds,
                                  uint8_t* ext, uint8_t* keep, int32_t* stats, pasco_stream_t s) {
  PASCO_CHECK_ARG(pitch >= 3, "pasco_scene_points: a point row needs x, y, z (pitch=%d)", pitch);
  if (N == 0) return 0;
  k_scene_points<<<grid_for(N, kBlock), kBlock, 0, (cudaStream_t)s>>>(pts, N, pitch, mat4(T), bounds, ext, keep, stats);
  PASCO_CHECK_LAUNCH("pasco_scene_points");
  return 0;
}

extern "C" int pasco_scene_point_rows(const float* pts, int32_t pitch, const float* vote, int32_t V, const float* emb,
                                      int32_t E, int64_t N, const int32_t* keep_rows, int64_t n_keep, const float T[16],
                                      float* feats, int64_t* coords, const int32_t* label, const int32_t* ext_rows,
                                      int64_t n_ext, double* xyz, int32_t* label_out, pasco_stream_t s) {
  PASCO_CHECK_ARG(pitch >= 3 && V >= 0 && E >= 0, "pasco_scene_point_rows: bad widths");
  cudaStream_t st = (cudaStream_t)s;
  const int64_t Fw = V + (pitch - 3) + 1 + E + 6;
  if (n_keep > 0)
    k_scene_point_rows<<<grid_for(n_keep * Fw, kBlock), kBlock, 0, st>>>(pts, pitch, vote, V, emb, E, N, keep_rows,
                                                                         n_keep, mat4(T), feats, coords);
  if (n_ext > 0)
    k_scene_point_pass<<<grid_for(n_ext, kBlock), kBlock, 0, st>>>(pts, pitch, label, ext_rows, n_ext, xyz, label_out);
  PASCO_CHECK_LAUNCH("pasco_scene_point_rows");
  return 0;
}

extern "C" int pasco_scene_box(const uint8_t* gs, const uint8_t* gi, const int32_t lo[3], const int32_t G[3],
                               int32_t with_inst, const double* bounds, const int32_t box_lo[3], const int32_t size[3],
                               uint8_t* sem, uint8_t* inst, uint8_t* geo, pasco_stream_t s) {
  const int64_t cells = (int64_t)size[0] * size[1] * size[2];
  PASCO_CHECK_ARG(cells > 0, "pasco_scene_box: empty box");
  k_scene_box<<<grid_for(cells, kBlock), kBlock, 0, (cudaStream_t)s>>>(gs, gi, lo[0], lo[1], lo[2], G[0], G[1], G[2],
                                                                       with_inst, bounds, box_lo[0], box_lo[1], box_lo[2],
                                                                       size[0], size[1], size[2], sem, inst, geo);
  PASCO_CHECK_LAUNCH("pasco_scene_box");
  return 0;
}

extern "C" int pasco_scene_scale(const uint8_t* sem, int32_t X, int32_t Y, int32_t Z, int32_t scale, uint8_t* sem_out,
                                 uint8_t* geo_out, pasco_stream_t s) {
  PASCO_CHECK_ARG(scale == 2 || scale == 4, "pasco_scene_scale: scale must be 2 or 4 (%d)", scale);
  PASCO_CHECK_ARG(X % scale == 0 && Y % scale == 0 && Z % scale == 0 && X > 0 && Y > 0 && Z > 0,
                  "pasco_scene_scale: the volume must be a non-empty multiple of the scale");
  const int64_t blocks = (int64_t)(X / scale) * (Y / scale) * (Z / scale);
  cudaStream_t st = (cudaStream_t)s;
  if (scale == 2)
    k_scene_scale<2><<<grid_for(blocks, kBlock), kBlock, 0, st>>>(sem, X, Y, Z, sem_out, geo_out);
  else
    k_scene_scale<4><<<grid_for(blocks, kBlock), kBlock, 0, st>>>(sem, X, Y, Z, sem_out, geo_out);
  PASCO_CHECK_LAUNCH("pasco_scene_scale");
  return 0;
}

extern "C" int pasco_scene_masks(const uint8_t* sem, const uint8_t* inst, int64_t cells, const int32_t* slot,
                                 int32_t n_masks, uint8_t* masks, uint8_t* labels, pasco_stream_t s) {
  PASCO_CHECK_ARG(cells > 0 && cells < INT_MAX && n_masks >= 0,
                  "pasco_scene_masks: need 0 < cells < 2^31 and n_masks >= 0");
  if (n_masks == 0) return 0;
  cudaStream_t st = (cudaStream_t)s;
  int32_t* first = nullptr;
  cudaError_t e = ws_alloc((void**)&first, 256 * sizeof(int32_t), st);
  if (e != cudaSuccess) {
    set_error("pasco_scene_masks: workspace: %s", cudaGetErrorString(e));
    return -1;
  }
  cudaMemsetAsync(masks, 0, (size_t)n_masks * cells, st);
  k_scene_fill_i32<<<1, kBlock, 0, st>>>(first, 256, INT_MAX);
  k_scene_masks<<<grid_for(cells, kBlock), kBlock, 0, st>>>(sem, inst, cells, slot, masks, first);
  k_scene_mask_labels<<<1, kBlock, 0, st>>>(sem, slot, first, labels);
  cudaFreeAsync(first, st);
  PASCO_CHECK_LAUNCH("pasco_scene_masks");
  return 0;
}
