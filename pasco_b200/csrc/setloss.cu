// The training criterion of the reference's SetCriterion (criterion_sparse.py, matcher_sparse.py, helper.py:7-37,
// lovasz.py:186-219) on the rows of one output level: target sampling into bit rows, the matcher's cost sums, the mask
// losses of the matched pairs, the voxel↔query semantic logits and the Lovász-softmax, forward and backward.
//
// Every float reduction runs in two steps: per-CTA partials over a fixed row chunk, then a column sum of the partials
// in CTA order (k_sl_reduce).  Integer counters use atomics.  Repeat calls therefore give identical bits.
#include "common.cuh"
#include <math.h>

namespace {

using namespace pasco;

constexpr int kBlock = 128;
constexpr int kMaxChunks = 264;
constexpr uint8_t kKnown = 1, kValid = 2;   // flags: not unknown; not unknown and at least one target bit

__device__ __forceinline__ float sigm(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ float softplus(float x) { return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x))); }

// losses.py:45-66 with alpha 0.25, gamma 2, for a 0/1 target
__device__ __forceinline__ float focal(float x, float p, bool t) {
  return t ? 0.25f * (1.f - p) * (1.f - p) * softplus(-x) : 0.75f * p * p * softplus(x);
}
__device__ __forceinline__ float focal_grad(float x, float p, bool t) {
  return t ? -0.25f * (1.f - p) * (1.f - p) * (2.f * p * softplus(-x) + (1.f - p))
           : 0.75f * p * p * (2.f * (1.f - p) * softplus(x) + p);
}

int chunks_for(int64_t n, int per) {
  int64_t g = (n + per - 1) / per;
  return (int)(g < 1 ? 1 : (g > kMaxChunks ? kMaxChunks : g));
}

// ---- target sampling ------------------------------------------------------------------------------------------------
// stats int32: [0, T) target bits over the valid rows, [T] valid rows (dwh), [T+1] rows outside the volume or with a
// label outside [0, K) other than 255, [T+2], [T+3] present-class bits (classes 0..31, 32..63), [T+4] known rows
struct SampleParams {
  const int32_t* xyz;
  int64_t n;
  const int32_t* min_c;
  const uint8_t* masks;
  int T, W;
  const uint8_t* unknown;
  const uint8_t* label;
  int X, Y, Z, K;
  uint32_t* bits;
  uint8_t* flags;
  int32_t* lab;
  int32_t* stats;
};

__global__ void __launch_bounds__(256) k_sl_sample(const __grid_constant__ SampleParams p) {
  extern __shared__ int s_cnt[];                    // [T + 5]
  for (int i = threadIdx.x; i < p.T + 5; i += blockDim.x) s_cnt[i] = 0;
  __syncthreads();
  const int64_t cells = (int64_t)p.X * p.Y * p.Z;
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < p.n; r += (int64_t)gridDim.x * blockDim.x) {
    const int32_t* c = p.xyz + r * 4;
    const int x = c[1] - p.min_c[0], y = c[2] - p.min_c[1], z = c[3] - p.min_c[2];
    uint32_t* row = p.bits + r * p.W;
    const bool other = c[0] != 0;                   // a row of another batch item: left out, not counted
    if (other || x < 0 || y < 0 || z < 0 || x >= p.X || y >= p.Y || z >= p.Z) {
      for (int w = 0; w < p.W; ++w) row[w] = 0u;
      p.flags[r] = 0;
      if (p.lab) p.lab[r] = -1;
      if (!other) atomicAdd(s_cnt + p.T + 1, 1);
      continue;
    }
    const int64_t cell = ((int64_t)x * p.Y + y) * p.Z + z;
    const bool known = __ldg(p.unknown + cell) == 0;
    bool any = false;
    for (int w = 0; w < p.W; ++w) {
      uint32_t b = 0u;
      for (int j = 0; j < 32 && w * 32 + j < p.T; ++j)
        if (__ldg(p.masks + (int64_t)(w * 32 + j) * cells + cell)) b |= 1u << j;
      row[w] = b;
      any |= b != 0u;
    }
    const bool valid = known && any;
    p.flags[r] = (known ? kKnown : 0) | (valid ? kValid : 0);
    if (known) atomicAdd(s_cnt + p.T + 4, 1);
    if (valid) {
      atomicAdd(s_cnt + p.T, 1);
      for (int w = 0; w < p.W; ++w)
        for (uint32_t b = row[w]; b; b &= b - 1) atomicAdd(s_cnt + w * 32 + __ffs(b) - 1, 1);
    }
    if (p.lab) {
      const int l = __ldg(p.label + cell);
      p.lab[r] = l == 255 ? -1 : l;
      if (l != 255) {
        if (l >= p.K) atomicAdd(s_cnt + p.T + 1, 1);
        else atomicOr((unsigned*)s_cnt + p.T + 2 + (l >> 5), 1u << (l & 31));
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < p.T + 5; i += blockDim.x) {
    const int v = s_cnt[i];
    if (!v) continue;
    if (i == p.T + 2 || i == p.T + 3) atomicOr((unsigned*)p.stats + i, (unsigned)v);
    else atomicAdd(p.stats + i, v);
  }
}

// ---- fixed-order column sums of per-CTA partials --------------------------------------------------------------------
__global__ void k_sl_reduce(const float* __restrict__ part, int G, int64_t L, float* __restrict__ out) {
  for (int64_t l = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; l < L; l += (int64_t)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int g = 0; g < G; ++g) s += part[(int64_t)g * L + l];
    out[l] = s;
  }
}

// ---- matching cost (matcher_sparse.py:96-157) -----------------------------------------------------------------------
// partial layout per CTA row chunk, L = Q·(3·W·32 + 2): Σσ·t, Σfocal_pos·t, Σfocal_neg·t as [Q][W·32] each, then Σσ
// and Σfocal_neg per query
struct CostParams {
  const float* F;
  int64_t n;
  int Q, W;
  const uint32_t* bits;
  const uint8_t* flags;
  int64_t chunk, L;
  float* part;
};

__global__ void __launch_bounds__(kBlock) k_sl_cost(const __grid_constant__ CostParams p) {
  const int q = blockIdx.y * kBlock + threadIdx.x, w = blockIdx.z, T32 = p.W * 32;
  const bool on = q < p.Q;
  float as[32], ap[32], an[32], ssum = 0.f, nsum = 0.f;
#pragma unroll
  for (int j = 0; j < 32; ++j) as[j] = ap[j] = an[j] = 0.f;
  const int64_t r0 = blockIdx.x * p.chunk, r1 = min(p.n, r0 + p.chunk);
  for (int64_t r = r0; r < r1; ++r) {
    if (!(__ldg(p.flags + r) & kValid)) continue;
    const uint32_t b = __ldg(p.bits + r * p.W + w);
    const float x = on ? __ldg(p.F + r * p.Q + q) : 0.f;
    const float s = sigm(x);
    const float fp = 0.25f * (1.f - s) * (1.f - s) * softplus(-x), fn = 0.75f * s * s * softplus(x);
    ssum += s;
    nsum += fn;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const float t = (float)((b >> j) & 1u);
      as[j] = fmaf(s, t, as[j]);
      ap[j] = fmaf(fp, t, ap[j]);
      an[j] = fmaf(fn, t, an[j]);
    }
  }
  if (!on) return;
  float* out = p.part + blockIdx.x * p.L;
  const int64_t plane = (int64_t)p.Q * T32;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int64_t i = (int64_t)q * T32 + w * 32 + j;
    out[i] = as[j];
    out[plane + i] = ap[j];
    out[2 * plane + i] = an[j];
  }
  if (w == 0) {
    out[3 * plane + q] = ssum;
    out[3 * plane + p.Q + q] = nsum;
  }
}

struct FinishParams {
  const float* sums;
  const int32_t* stats;
  const float* logits;   // [Q][K1]
  int K1;
  const int32_t* ids;    // [T]
  const float* cw;       // [K1]
  int Q, T, W;
  float cost_mask, cost_class, cost_dice;
  float* C;              // [Q][T]
};

__global__ void k_sl_cost_finish(const __grid_constant__ FinishParams p) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.Q * p.T) return;
  const int q = i / p.T, t = i % p.T, T32 = p.W * 32;
  const int64_t plane = (int64_t)p.Q * T32, at = (int64_t)q * T32 + t;
  const float* lg = p.logits + (int64_t)q * p.K1;
  float m = lg[0];
  for (int k = 1; k < p.K1; ++k) m = fmaxf(m, lg[k]);
  float z = 0.f;
  for (int k = 0; k < p.K1; ++k) z += expf(lg[k] - m);
  const int id = p.ids[t];
  const float prob = expf(lg[id] - m) / z;
  const int dwh = p.stats[p.T];
  const float tsum = (float)p.stats[t];
  const float dice = 1.f - (2.f * p.sums[at] + 1.f) / (p.sums[3 * plane + q] + tsum + 1.f);
  const float foc = dwh > 0 ? (p.sums[plane + at] + (p.sums[3 * plane + p.Q + q] - p.sums[2 * plane + at])) / (float)dwh
                            : 0.f;
  p.C[i] = (p.cost_mask * foc + p.cost_class * -prob + p.cost_dice * dice) * p.cw[id];
}

// ---- mask losses of the matched pairs (criterion_sparse.py:83-112), over the known rows -----------------------------
struct PairParams {
  const float* F;
  int64_t n;
  int Q, W;
  const uint32_t* bits;
  const uint8_t* flags;
  const int32_t* qi;
  const int32_t* tj;
  int P;
  int64_t chunk;
  float* part;           // [G][P][4]: Σfocal, Σσ·t, Σσ, Σt
  const float* g;        // backward: dL/d(the four sums) [P][4]
  float* gF;             // backward: [N][Q]
};

__global__ void __launch_bounds__(kBlock) k_sl_pair_sums(const __grid_constant__ PairParams p) {
  const int k = blockIdx.y * kBlock + threadIdx.x;
  if (k >= p.P) return;
  const int q = p.qi[k], t = p.tj[k];
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  const int64_t r0 = blockIdx.x * p.chunk, r1 = min(p.n, r0 + p.chunk);
  for (int64_t r = r0; r < r1; ++r) {
    if (!(__ldg(p.flags + r) & kKnown)) continue;
    const bool tb = (__ldg(p.bits + r * p.W + (t >> 5)) >> (t & 31)) & 1u;
    const float x = __ldg(p.F + r * p.Q + q), s = sigm(x);
    a0 += focal(x, s, tb);
    a1 += tb ? s : 0.f;
    a2 += s;
    a3 += tb ? 1.f : 0.f;
  }
  float* out = p.part + ((int64_t)blockIdx.x * p.P + k) * 4;
  out[0] = a0;
  out[1] = a1;
  out[2] = a2;
  out[3] = a3;
}

__global__ void __launch_bounds__(kBlock) k_sl_pair_backward(const __grid_constant__ PairParams p) {
  const int64_t total = p.n * p.P;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / p.P;
    const int k = (int)(i % p.P);
    if (!(__ldg(p.flags + r) & kKnown)) continue;
    const int q = p.qi[k], t = p.tj[k];
    const bool tb = (__ldg(p.bits + r * p.W + (t >> 5)) >> (t & 31)) & 1u;
    const float x = __ldg(p.F + r * p.Q + q), s = sigm(x);
    const float* g = p.g + k * 4;
    p.gF[r * p.Q + q] = g[0] * focal_grad(x, s, tb) + (g[1] * (tb ? 1.f : 0.f) + g[2]) * s * (1.f - s);
  }
}

// ---- semantic consistency (helper.py:7-37): out[n] = Σ_j a_nj · L[j], a_nj = (σ(F[n, keep_j]) + 1e-8) / Σ_j (…) --
constexpr int kMaxKeep = 128, kMaxClasses = 64, kRowsPerTile = 16;

struct SscParams {
  const float* F;
  int64_t n;
  int Q;
  const int32_t* keep;
  int kq;
  const float* L;        // [kq][K]
  int K;
  float* out;            // [N][K]
  const float* g;        // backward: dL/dout [N][K]
  float* gF;             // backward: [N][Q], kept columns written
  int64_t chunk;
  float* part;           // backward: [G][kq·K] partials of dL/dL
};

// one warp per row; a_n staged per warp in shared memory
__global__ void __launch_bounds__(kBlock) k_sl_ssc_forward(const __grid_constant__ SscParams p) {
  __shared__ float s_L[kMaxKeep * kMaxClasses];
  __shared__ float s_a[kBlock / 32][kMaxKeep];
  for (int i = threadIdx.x; i < p.kq * p.K; i += blockDim.x) s_L[i] = p.L[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  for (int64_t r = blockIdx.x * (int64_t)(kBlock / 32) + wp; r < p.n; r += (int64_t)gridDim.x * (kBlock / 32)) {
    float z = 0.f;
    for (int j = lane; j < p.kq; j += 32) {
      const float a = sigm(__ldg(p.F + r * p.Q + p.keep[j])) + 1e-8f;
      s_a[wp][j] = a;
      z += a;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) z += __shfl_xor_sync(0xffffffffu, z, o);
    __syncwarp();
    for (int c = lane; c < p.K; c += 32) {
      float acc = 0.f;
      for (int j = 0; j < p.kq; ++j) acc = fmaf(s_a[wp][j] / z, s_L[j * p.K + c], acc);
      p.out[r * p.K + c] = acc;
    }
    __syncwarp();
  }
}

// per CTA a fixed chunk of rows in tiles of kRowsPerTile: each warp writes dF for its rows and stages a_n and g_n; then
// every thread adds the tile into its own entries of dL/dL (entry e = threadIdx.x + kBlock·i, i < kMaxKeep·K / kBlock)
__global__ void __launch_bounds__(kBlock) k_sl_ssc_backward(const __grid_constant__ SscParams p) {
  __shared__ float s_L[kMaxKeep * (kMaxClasses + 1)];
  __shared__ float s_a[kRowsPerTile][kMaxKeep];
  __shared__ float s_g[kRowsPerTile][kMaxClasses];
  const int KP = p.K + 1, E = p.kq * p.K;
  for (int i = threadIdx.x; i < E; i += blockDim.x) s_L[(i / p.K) * KP + i % p.K] = p.L[i];
  constexpr int kEntries = kMaxKeep * kMaxClasses / kBlock;
  float acc[kEntries];
#pragma unroll
  for (int i = 0; i < kEntries; ++i) acc[i] = 0.f;
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  const int64_t r0 = blockIdx.x * p.chunk, r1 = min(p.n, r0 + p.chunk);
  for (int64_t t0 = r0; t0 < r1; t0 += kRowsPerTile) {
    __syncthreads();
    for (int rr = wp; rr < kRowsPerTile; rr += kBlock / 32) {
      const int64_t r = t0 + rr;
      if (r >= r1) {
        for (int j = lane; j < p.kq; j += 32) s_a[rr][j] = 0.f;
        continue;
      }
      float z = 0.f, go = 0.f;
      for (int j = lane; j < p.kq; j += 32) {
        const float a = sigm(__ldg(p.F + r * p.Q + p.keep[j])) + 1e-8f;
        s_a[rr][j] = a;
        z += a;
      }
      for (int c = lane; c < p.K; c += 32) {
        const float g = __ldg(p.g + r * p.K + c);
        s_g[rr][c] = g;
        go += g * __ldg(p.out + r * p.K + c);
      }
#pragma unroll
      for (int o = 16; o; o >>= 1) {
        z += __shfl_xor_sync(0xffffffffu, z, o);
        go += __shfl_xor_sync(0xffffffffu, go, o);
      }
      __syncwarp();
      for (int j = lane; j < p.kq; j += 32) {
        float dot = 0.f;
        for (int c = 0; c < p.K; ++c) dot = fmaf(s_g[rr][c], s_L[j * KP + c], dot);
        const float s = s_a[rr][j] - 1e-8f;
        p.gF[r * p.Q + p.keep[j]] = s * (1.f - s) * (dot - go) / z;
        s_a[rr][j] = s_a[rr][j] / z;
      }
    }
    __syncthreads();
    const int rows = (int)min((int64_t)kRowsPerTile, r1 - t0);
#pragma unroll
    for (int i = 0; i < kEntries; ++i) {
      const int e = threadIdx.x + kBlock * i;
      if (e < E) {
        const int j = e / p.K, c = e % p.K;
        float a = acc[i];
        for (int rr = 0; rr < rows; ++rr) a = fmaf(s_a[rr][j], s_g[rr][c], a);
        acc[i] = a;
      }
    }
  }
#pragma unroll
  for (int i = 0; i < kEntries; ++i) {
    const int e = threadIdx.x + kBlock * i;
    if (e < E) p.part[(int64_t)blockIdx.x * E + e] = acc[i];
  }
}

// ---- Lovász-softmax (lovasz.py:186-219) -----------------------------------------------------------------------------
// labels: -1 = row left out (sorted last through error −1), a class in [0, C), or >= C = background of every class
constexpr int kTile = 1024, kItems = kTile / 256;

__global__ void __launch_bounds__(256) k_lov_errors(const float* __restrict__ logits, int64_t P, int C,
                                                    const int32_t* __restrict__ labels, float* __restrict__ probs,
                                                    float* __restrict__ err) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < P; r += (int64_t)gridDim.x * blockDim.x) {
    const float* x = logits + r * C;
    float m = x[0];
    for (int c = 1; c < C; ++c) m = fmaxf(m, x[c]);
    float z = 0.f;
    for (int c = 0; c < C; ++c) z += expf(x[c] - m);
    const int l = labels[r];
    for (int c = 0; c < C; ++c) {
      const float pr = expf(x[c] - m) / z;
      probs[r * C + c] = pr;
      err[(int64_t)c * P + r] = l < 0 ? -1.f : fabsf((l == c ? 1.f : 0.f) - pr);
    }
  }
}

__device__ __forceinline__ int fg_at(const int32_t* labels, const int64_t* perm, int64_t P, int c, int64_t i) {
  return i < P && __ldg(labels + __ldg(perm + (int64_t)c * P + i)) == c;
}

// per (tile, class): foreground count of the tile in sorted order
__global__ void __launch_bounds__(256) k_lov_tile_counts(const int32_t* __restrict__ labels,
                                                         const int64_t* __restrict__ perm, int64_t P, int tiles,
                                                         int32_t* __restrict__ cnt) {
  const int c = blockIdx.y;
  __shared__ int s;
  if (threadIdx.x == 0) s = 0;
  __syncthreads();
  int v = 0;
  for (int k = 0; k < kItems; ++k) v += fg_at(labels, perm, P, c, (int64_t)blockIdx.x * kTile + k * 256 + threadIdx.x);
  atomicAdd(&s, v);
  __syncthreads();
  if (threadIdx.x == 0) cnt[(int64_t)c * tiles + blockIdx.x] = s;
}

// per class: exclusive tile offsets in place, and the class's foreground total after them
__global__ void k_lov_tile_scan(int32_t* cnt, int tiles, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  int32_t* t = cnt + (int64_t)c * (tiles + 1);
  int acc = 0;
  for (int i = 0; i < tiles; ++i) {
    const int v = t[i];
    t[i] = acc;
    acc += v;
  }
  t[tiles] = acc;
}

// lovasz_grad at every sorted position: jaccard_i = 1 − (gts − cumfg_i) / (gts + cumbg_i), grad_i = jaccard_i −
// jaccard_{i−1}; writes grad and the tile's partial of Σ err_i · grad_i
__global__ void __launch_bounds__(256) k_lov_grad(const float* __restrict__ err_sorted, const int64_t* __restrict__ perm,
                                                  const int32_t* __restrict__ labels, int64_t P, int tiles,
                                                  const int32_t* __restrict__ off, float* __restrict__ grad,
                                                  float* __restrict__ part) {
  const int c = blockIdx.y;
  const int64_t base = (int64_t)blockIdx.x * kTile + threadIdx.x * kItems;
  const int32_t* o = off + (int64_t)c * (tiles + 1);
  const int gts = o[tiles];
  int fg[kItems], run = 0;
#pragma unroll
  for (int k = 0; k < kItems; ++k) {
    fg[k] = fg_at(labels, perm, P, c, base + k);
    run += fg[k];
  }
  // exclusive scan of the per-thread counts over the block
  __shared__ int s_scan[256];
  __shared__ float s_red[256];
  s_scan[threadIdx.x] = run;
  __syncthreads();
  for (int d = 1; d < 256; d <<= 1) {
    const int v = threadIdx.x >= d ? s_scan[threadIdx.x - d] : 0;
    __syncthreads();
    s_scan[threadIdx.x] += v;
    __syncthreads();
  }
  int cum = o[blockIdx.x] + s_scan[threadIdx.x] - run;       // foreground before this thread's first item
  float dot = 0.f;
#pragma unroll
  for (int k = 0; k < kItems; ++k) {
    const int64_t i = base + k;
    if (i >= P) break;
    const float e = __ldg(err_sorted + (int64_t)c * P + i);
    const int before = cum;
    cum += fg[k];
    const float jac = 1.f - (float)(gts - cum) / (float)(gts + (int)(i + 1 - cum));
    float g = jac;
    if (i > 0) {
      const int bg_prev = (int)(i - before);
      g -= 1.f - (float)(gts - before) / (float)(gts + bg_prev);
    }
    if (e < 0.f) g = 0.f;                                     // a row left out: after every kept row
    grad[(int64_t)c * P + i] = g;
    dot += e < 0.f ? 0.f : e * g;
  }
  s_red[threadIdx.x] = dot;
  __syncthreads();
  for (int s = 128; s; s >>= 1) {
    if (threadIdx.x < s) s_red[threadIdx.x] += s_red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) part[(int64_t)c * tiles + blockIdx.x] = s_red[0];
}

__global__ void k_lov_class_sum(const float* __restrict__ part, int tiles, int C, float* __restrict__ loss) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float s = 0.f;
  for (int i = 0; i < tiles; ++i) s += part[(int64_t)c * tiles + i];
  loss[c] = s;
}

// dL/dp at the unsorted positions: g_c · grad_i · sign(p − fg)
__global__ void __launch_bounds__(256) k_lov_scatter(const float* __restrict__ probs, const int32_t* __restrict__ labels,
                                                     const int64_t* __restrict__ perm, const float* __restrict__ grad,
                                                     const float* __restrict__ g, int64_t P, int C,
                                                     float* __restrict__ dp) {
  const int64_t total = P * C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i / P);
    const int64_t r = __ldg(perm + i);
    const int l = __ldg(labels + r);
    if (l < 0) continue;
    const float d = __ldg(probs + r * C + c) - (l == c ? 1.f : 0.f);
    const float sg = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);
    dp[r * C + c] = __ldg(g + c) * __ldg(grad + i) * sg;
  }
}

__global__ void __launch_bounds__(256) k_lov_softmax_backward(const float* __restrict__ probs,
                                                              const float* __restrict__ dp, int64_t P, int C,
                                                              float* __restrict__ dx) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < P; r += (int64_t)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int c = 0; c < C; ++c) s += dp[r * C + c] * probs[r * C + c];
    for (int c = 0; c < C; ++c) dx[r * C + c] = probs[r * C + c] * (dp[r * C + c] - s);
  }
}

int reduce_to(const char* name, const float* part, int G, int64_t L, float* out, cudaStream_t st) {
  k_sl_reduce<<<grid_for(L, 256, 4), 256, 0, st>>>(part, G, L, out);
  PASCO_CHECK_LAUNCH(name);
  return 0;
}

}  // namespace

extern "C" int pasco_setloss_sample(const int32_t* xyz, int64_t n, const int32_t* min_c, const uint8_t* masks,
                                    int32_t T, const uint8_t* unknown, const uint8_t* label, int32_t X, int32_t Y,
                                    int32_t Z, int32_t K, uint32_t* bits, uint8_t* flags, int32_t* lab, int32_t* stats,
                                    pasco_stream_t s) {
  PASCO_CHECK_ARG(n >= 0 && T >= 0 && X > 0 && Y > 0 && Z > 0 && K >= 1 && K <= 64,
                  "pasco_setloss_sample: bad sizes (rows %lld, targets %d, classes %d)", (long long)n, T, K);
  if (n == 0) return 0;
  SampleParams p = {xyz, n, min_c, masks, T, T > 0 ? (T + 31) / 32 : 1, unknown, label, X, Y, Z, K, bits, flags, lab,
                    stats};
  k_sl_sample<<<grid_for(n, 256, 4), 256, sizeof(int) * (T + 5), (cudaStream_t)s>>>(p);
  PASCO_CHECK_LAUNCH("pasco_setloss_sample");
  return 0;
}

extern "C" int pasco_setloss_match_cost(const float* F, int64_t n, int32_t Q, const uint32_t* bits, int32_t T,
                                        const uint8_t* flags, const int32_t* stats, const float* query_logits,
                                        int32_t K1, const int32_t* ids, const float* class_weight, float cost_mask,
                                        float cost_class, float cost_dice, float* C, pasco_stream_t s) {
  PASCO_CHECK_ARG(n >= 0 && Q >= 1 && T >= 0 && K1 >= 2, "pasco_setloss_match_cost: bad sizes");
  if (T == 0) return 0;
  const cudaStream_t st = (cudaStream_t)s;
  CostParams p = {};
  p.F = F;
  p.n = n;
  p.Q = Q;
  p.W = (T + 31) / 32;
  p.bits = bits;
  p.flags = flags;
  const int yt = (Q + kBlock - 1) / kBlock;
  const int G = chunks_for(n, 512);
  p.chunk = n > 0 ? (n + G - 1) / G : 1;
  p.L = (int64_t)Q * (3 * p.W * 32 + 2);
  float* ws = nullptr;
  cudaError_t e = ws_alloc((void**)&ws, sizeof(float) * (size_t)p.L * (G + 1), st);
  PASCO_CHECK_ARG(e == cudaSuccess, "pasco_setloss_match_cost: workspace: %s", cudaGetErrorString(e));
  p.part = ws + p.L;
  k_sl_cost<<<dim3(G, yt, p.W), kBlock, 0, st>>>(p);
  PASCO_CHECK_LAUNCH("pasco_setloss_match_cost");
  if (reduce_to("pasco_setloss_match_cost", p.part, G, p.L, ws, st)) return -1;
  FinishParams f = {ws, stats, query_logits, K1, ids, class_weight, Q, T, p.W, cost_mask, cost_class, cost_dice, C};
  k_sl_cost_finish<<<(Q * T + 127) / 128, 128, 0, st>>>(f);
  PASCO_CHECK_LAUNCH("pasco_setloss_match_cost");
  cudaFreeAsync(ws, st);
  return 0;
}

extern "C" int pasco_setloss_pair_sums(const float* F, int64_t n, int32_t Q, const uint32_t* bits, int32_t T,
                                       const uint8_t* flags, const int32_t* qi, const int32_t* tj, int32_t P,
                                       float* sums, pasco_stream_t s) {
  PASCO_CHECK_ARG(n >= 0 && Q >= 1 && T >= 1 && P >= 0, "pasco_setloss_pair_sums: bad sizes");
  if (P == 0) return 0;
  const cudaStream_t st = (cudaStream_t)s;
  const int G = chunks_for(n, 512);
  PairParams p = {};
  p.F = F;
  p.n = n;
  p.Q = Q;
  p.W = (T + 31) / 32;
  p.bits = bits;
  p.flags = flags;
  p.qi = qi;
  p.tj = tj;
  p.P = P;
  p.chunk = n > 0 ? (n + G - 1) / G : 1;
  cudaError_t e = ws_alloc((void**)&p.part, sizeof(float) * (size_t)G * P * 4, st);
  PASCO_CHECK_ARG(e == cudaSuccess, "pasco_setloss_pair_sums: workspace: %s", cudaGetErrorString(e));
  k_sl_pair_sums<<<dim3(G, (P + kBlock - 1) / kBlock), kBlock, 0, st>>>(p);
  PASCO_CHECK_LAUNCH("pasco_setloss_pair_sums");
  if (reduce_to("pasco_setloss_pair_sums", p.part, G, (int64_t)P * 4, sums, st)) return -1;
  cudaFreeAsync(p.part, st);
  return 0;
}

extern "C" int pasco_setloss_pair_backward(const float* F, int64_t n, int32_t Q, const uint32_t* bits, int32_t T,
                                           const uint8_t* flags, const int32_t* qi, const int32_t* tj, int32_t P,
                                           const float* g, float* gF, pasco_stream_t s) {
  PASCO_CHECK_ARG(n >= 0 && Q >= 1 && T >= 1 && P >= 0, "pasco_setloss_pair_backward: bad sizes");
  if (P == 0 || n == 0) return 0;
  PairParams p = {};
  p.F = F;
  p.n = n;
  p.Q = Q;
  p.W = (T + 31) / 32;
  p.bits = bits;
  p.flags = flags;
  p.qi = qi;
  p.tj = tj;
  p.P = P;
  p.g = g;
  p.gF = gF;
  k_sl_pair_backward<<<grid_for(n * P, kBlock, 8), kBlock, 0, (cudaStream_t)s>>>(p);
  PASCO_CHECK_LAUNCH("pasco_setloss_pair_backward");
  return 0;
}

extern "C" int pasco_setloss_ssc_forward(const float* F, int64_t n, int32_t Q, const int32_t* keep, int32_t kq,
                                         const float* L, int32_t K, float* out, pasco_stream_t s) {
  PASCO_CHECK_ARG(kq >= 1 && kq <= kMaxKeep && K >= 1 && K <= kMaxClasses && kq <= Q,
                  "pasco_setloss_ssc_forward: 1 <= kept queries <= %d, 1 <= classes <= %d", kMaxKeep, kMaxClasses);
  if (n == 0) return 0;
  SscParams p = {};
  p.F = F;
  p.n = n;
  p.Q = Q;
  p.keep = keep;
  p.kq = kq;
  p.L = L;
  p.K = K;
  p.out = out;
  k_sl_ssc_forward<<<grid_for(n, kBlock / 32, 8), kBlock, 0, (cudaStream_t)s>>>(p);
  PASCO_CHECK_LAUNCH("pasco_setloss_ssc_forward");
  return 0;
}

extern "C" int pasco_setloss_ssc_backward(const float* F, int64_t n, int32_t Q, const int32_t* keep, int32_t kq,
                                          const float* L, int32_t K, const float* out, const float* g, float* gF,
                                          float* gL, pasco_stream_t s) {
  PASCO_CHECK_ARG(kq >= 1 && kq <= kMaxKeep && K >= 1 && K <= kMaxClasses && kq <= Q,
                  "pasco_setloss_ssc_backward: 1 <= kept queries <= %d, 1 <= classes <= %d", kMaxKeep, kMaxClasses);
  const cudaStream_t st = (cudaStream_t)s;
  const int G = chunks_for(n, 512);
  const int64_t E = (int64_t)kq * K;
  SscParams p = {};
  p.F = F;
  p.n = n;
  p.Q = Q;
  p.keep = keep;
  p.kq = kq;
  p.L = L;
  p.K = K;
  p.out = const_cast<float*>(out);
  p.g = g;
  p.gF = gF;
  p.chunk = n > 0 ? (n + G - 1) / G : 1;
  cudaError_t e = ws_alloc((void**)&p.part, sizeof(float) * (size_t)G * E, st);
  PASCO_CHECK_ARG(e == cudaSuccess, "pasco_setloss_ssc_backward: workspace: %s", cudaGetErrorString(e));
  k_sl_ssc_backward<<<G, kBlock, 0, st>>>(p);
  PASCO_CHECK_LAUNCH("pasco_setloss_ssc_backward");
  if (reduce_to("pasco_setloss_ssc_backward", p.part, G, E, gL, st)) return -1;
  cudaFreeAsync(p.part, st);
  return 0;
}

extern "C" int pasco_lovasz_errors(const float* logits, int64_t P, int32_t C, const int32_t* labels, float* probs,
                                   float* err, pasco_stream_t s) {
  PASCO_CHECK_ARG(P >= 0 && C >= 1 && C <= 64, "pasco_lovasz_errors: 1 <= classes <= 64 (got %d)", C);
  if (P == 0) return 0;
  k_lov_errors<<<grid_for(P, 256, 4), 256, 0, (cudaStream_t)s>>>(logits, P, C, labels, probs, err);
  PASCO_CHECK_LAUNCH("pasco_lovasz_errors");
  return 0;
}

extern "C" int pasco_lovasz_grad(const float* err_sorted, const int64_t* perm, const int32_t* labels, int64_t P,
                                 int32_t C, float* grad, float* loss, pasco_stream_t s) {
  PASCO_CHECK_ARG(P >= 1 && C >= 1 && C <= 64, "pasco_lovasz_grad: bad sizes");
  const cudaStream_t st = (cudaStream_t)s;
  const int64_t tiles64 = (P + kTile - 1) / kTile;
  PASCO_CHECK_ARG(tiles64 < (1 << 30), "pasco_lovasz_grad: too many rows");
  const int tiles = (int)tiles64;
  int32_t* off = nullptr;
  cudaError_t e = ws_alloc((void**)&off, sizeof(int32_t) * (size_t)C * (tiles + 1) + sizeof(float) * (size_t)C * tiles,
                           st);
  PASCO_CHECK_ARG(e == cudaSuccess, "pasco_lovasz_grad: workspace: %s", cudaGetErrorString(e));
  float* part = (float*)(off + (size_t)C * (tiles + 1));
  // counts written with a stride of tiles + 1 so the scan can append each class's total in place
  int32_t* cnt = off;
  k_lov_tile_counts<<<dim3(tiles, C), 256, 0, st>>>(labels, perm, P, tiles + 1, cnt);
  PASCO_CHECK_LAUNCH("pasco_lovasz_grad");
  k_lov_tile_scan<<<1, 64, 0, st>>>(cnt, tiles, C);
  PASCO_CHECK_LAUNCH("pasco_lovasz_grad");
  k_lov_grad<<<dim3(tiles, C), 256, 0, st>>>(err_sorted, perm, labels, P, tiles, off, grad, part);
  PASCO_CHECK_LAUNCH("pasco_lovasz_grad");
  k_lov_class_sum<<<1, 64, 0, st>>>(part, tiles, C, loss);
  PASCO_CHECK_LAUNCH("pasco_lovasz_grad");
  cudaFreeAsync(off, st);
  return 0;
}

extern "C" int pasco_lovasz_backward(const float* probs, const int32_t* labels, const int64_t* perm, const float* grad,
                                     const float* g, int64_t P, int32_t C, float* dx, pasco_stream_t s) {
  PASCO_CHECK_ARG(P >= 0 && C >= 1 && C <= 64, "pasco_lovasz_backward: bad sizes");
  if (P == 0) return 0;
  const cudaStream_t st = (cudaStream_t)s;
  float* dp = nullptr;
  cudaError_t e = ws_alloc((void**)&dp, sizeof(float) * (size_t)P * C, st);
  PASCO_CHECK_ARG(e == cudaSuccess, "pasco_lovasz_backward: workspace: %s", cudaGetErrorString(e));
  cudaMemsetAsync(dp, 0, sizeof(float) * (size_t)P * C, st);
  k_lov_scatter<<<grid_for(P * C, 256, 8), 256, 0, st>>>(probs, labels, perm, grad, g, P, C, dp);
  PASCO_CHECK_LAUNCH("pasco_lovasz_backward");
  k_lov_softmax_backward<<<grid_for(P, 256, 4), 256, 0, st>>>(probs, dp, P, C, dx);
  PASCO_CHECK_LAUNCH("pasco_lovasz_backward");
  cudaFreeAsync(dp, st);
  return 0;
}
