// The training criterion of the reference's SetCriterion (criterion_sparse.py, matcher_sparse.py, helper.py:7-37,
// lovasz.py:186-219) on the rows of one output level: target sampling into bit rows, the matcher's cost sums, the mask
// losses of the matched pairs, the voxel↔query semantic logits and the Lovász-softmax, forward and backward.
//
// Every float reduction runs in two steps: per-CTA partials over a fixed row chunk, then a column sum of the partials
// in CTA order (k_sl_reduce).  Integer counters use atomics.  Repeat calls therefore give identical bits.
#include "common.cuh"
#include <math.h>
#include <vector>

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

// ---- level tables ---------------------------------------------------------------------------------------------------
// A grouped launch carries up to kMaxLevels parameter sets by value.  Level l owns the blocks [start[l], start[l+1]) of
// blockIdx.x and sees them renumbered from 0, so each level runs exactly the launch a one-level call would make.
constexpr int kMaxLevels = 24;   // keeps every table under 4 KB of kernel parameters

template <class P>
struct Group {
  P lv[kMaxLevels];
  int start[kMaxLevels + 1];
  int count;
};

struct Slot {
  int l;
  int64_t b, nb;   // the block's index within its level, and the level's block count
};

template <class P>
__device__ __forceinline__ Slot slot_of(const Group<P>& g) {
  int l = 0;
  while (l + 1 < g.count && (int)blockIdx.x >= g.start[l + 1]) ++l;
  return {l, (int64_t)blockIdx.x - g.start[l], (int64_t)(g.start[l + 1] - g.start[l])};
}

// Launches `launch(group, grid)` for every run of up to kMaxLevels levels; make(l, params) fills level l's parameters
// and returns its block count (0: the level has nothing to do in this pass).
template <class P, class Make, class Launch>
int for_groups(const char* name, int count, Make make, Launch launch) {
  for (int l0 = 0; l0 < count; l0 += kMaxLevels) {
    Group<P> g;
    g.count = 0;
    int grid = 0;
    for (int l = l0; l < count && l < l0 + kMaxLevels; ++l) {
      const int nb = make(l, g.lv[g.count]);
      if (nb <= 0) continue;
      g.start[g.count++] = grid;
      grid += nb;
    }
    if (g.count == 0) continue;
    g.start[g.count] = grid;
    launch(g, grid);
    PASCO_CHECK_LAUNCH(name);
  }
  return 0;
}

// ---- fixed-order column sums of per-CTA partials --------------------------------------------------------------------
struct ReduceParams {
  const float* part;
  int G;
  int64_t L;
  float* out;
};

__global__ void k_sl_reduce(const __grid_constant__ Group<ReduceParams> gr) {
  const Slot sl = slot_of(gr);
  const ReduceParams& p = gr.lv[sl.l];
  for (int64_t l = sl.b * blockDim.x + threadIdx.x; l < p.L; l += sl.nb * blockDim.x) {
    float s = 0.f;
    for (int g = 0; g < p.G; ++g) s += p.part[(int64_t)g * p.L + l];
    p.out[l] = s;
  }
}

// ---- kept queries (helper.py:20-23): arg-max of the class logits is not the no-object class, in ascending order -----
struct KeepParams {
  const float* logits;   // [Q][K1]
  int Q, K1;
  int32_t* keep;
  int32_t* kept;
};

// one CTA per level; a block-wide ballot scan keeps the query order
__global__ void __launch_bounds__(kBlock) k_sl_keep(const __grid_constant__ Group<KeepParams> gr) {
  const Slot sl = slot_of(gr);
  const KeepParams& p = gr.lv[sl.l];
  __shared__ int s_warp[kBlock / 32];
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  int base = 0;
  for (int q0 = 0; q0 < p.Q; q0 += kBlock) {
    const int q = q0 + threadIdx.x;
    bool on = false;
    if (q < p.Q) {
      const float* lg = p.logits + (int64_t)q * p.K1;
      int arg = 0;
      float m = lg[0];
      for (int k = 1; k < p.K1; ++k)
        if (lg[k] > m) m = lg[k], arg = k;
      on = arg != p.K1 - 1;
    }
    const unsigned bal = __ballot_sync(0xffffffffu, on);
    if (lane == 0) s_warp[wp] = __popc(bal);
    __syncthreads();
    int before = base;
    for (int w = 0; w < wp; ++w) before += s_warp[w];
    if (on) p.keep[before + __popc(bal & ((1u << lane) - 1u))] = q;
    for (int w = 0; w < kBlock / 32; ++w) base += s_warp[w];
    __syncthreads();
  }
  if (threadIdx.x == 0) *p.kept = base;
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

__global__ void __launch_bounds__(kBlock) k_sl_cost(const __grid_constant__ Group<CostParams> gr) {
  const Slot sl = slot_of(gr);
  const CostParams& p = gr.lv[sl.l];
  if ((int)blockIdx.z >= p.W || (int)blockIdx.y * kBlock >= p.Q) return;
  const int q = blockIdx.y * kBlock + threadIdx.x, w = blockIdx.z, T32 = p.W * 32;
  const bool on = q < p.Q;
  float as[32], ap[32], an[32], ssum = 0.f, nsum = 0.f;
#pragma unroll
  for (int j = 0; j < 32; ++j) as[j] = ap[j] = an[j] = 0.f;
  const int64_t r0 = sl.b * p.chunk, r1 = min(p.n, r0 + p.chunk);
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
  float* out = p.part + sl.b * p.L;
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

__global__ void k_sl_cost_finish(const __grid_constant__ Group<FinishParams> gr) {
  const Slot sl = slot_of(gr);
  const FinishParams& p = gr.lv[sl.l];
  const int i = (int)sl.b * blockDim.x + threadIdx.x;
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

__global__ void __launch_bounds__(kBlock) k_sl_pair_sums(const __grid_constant__ Group<PairParams> gr) {
  const Slot sl = slot_of(gr);
  const PairParams& p = gr.lv[sl.l];
  const int k = blockIdx.y * kBlock + threadIdx.x;
  if (k >= p.P) return;
  const int q = p.qi[k], t = p.tj[k];
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  const int64_t r0 = sl.b * p.chunk, r1 = min(p.n, r0 + p.chunk);
  for (int64_t r = r0; r < r1; ++r) {
    if (!(__ldg(p.flags + r) & kKnown)) continue;
    const bool tb = (__ldg(p.bits + r * p.W + (t >> 5)) >> (t & 31)) & 1u;
    const float x = __ldg(p.F + r * p.Q + q), s = sigm(x);
    a0 += focal(x, s, tb);
    a1 += tb ? s : 0.f;
    a2 += s;
    a3 += tb ? 1.f : 0.f;
  }
  float* out = p.part + (sl.b * p.P + k) * 4;
  out[0] = a0;
  out[1] = a1;
  out[2] = a2;
  out[3] = a3;
}

__global__ void __launch_bounds__(kBlock) k_sl_pair_backward(const __grid_constant__ Group<PairParams> gr) {
  const Slot sl = slot_of(gr);
  const PairParams& p = gr.lv[sl.l];
  const int64_t total = p.n * p.P;
  for (int64_t i = sl.b * blockDim.x + threadIdx.x; i < total; i += sl.nb * blockDim.x) {
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
  const float* L;        // row j at L + (Lrows ? Lrows[j] : j)·ldL, K columns
  const int32_t* Lrows;
  int ldL, K;
  float* out;            // [N][K]
  const float* g;        // backward: dL/dout [N][K]
  float* gF;             // backward: [N][Q], kept columns written
  int64_t chunk;
  float* part;           // backward: [G][kq·K] partials of dL/dL
};

__device__ __forceinline__ float ssc_L(const SscParams& p, int j, int c) {
  return p.L[(int64_t)(p.Lrows ? p.Lrows[j] : j) * p.ldL + c];
}

// one warp per row; a_n staged per warp in shared memory
__global__ void __launch_bounds__(kBlock) k_sl_ssc_forward(const __grid_constant__ Group<SscParams> gr) {
  const Slot sl = slot_of(gr);
  const SscParams& p = gr.lv[sl.l];
  __shared__ float s_L[kMaxKeep * kMaxClasses];
  __shared__ float s_a[kBlock / 32][kMaxKeep];
  for (int i = threadIdx.x; i < p.kq * p.K; i += blockDim.x) s_L[i] = ssc_L(p, i / p.K, i % p.K);
  __syncthreads();
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  for (int64_t r = sl.b * (kBlock / 32) + wp; r < p.n; r += sl.nb * (kBlock / 32)) {
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
__global__ void __launch_bounds__(kBlock) k_sl_ssc_backward(const __grid_constant__ Group<SscParams> gr) {
  const Slot sl = slot_of(gr);
  const SscParams& p = gr.lv[sl.l];
  __shared__ float s_L[kMaxKeep * (kMaxClasses + 1)];
  __shared__ float s_a[kRowsPerTile][kMaxKeep];
  __shared__ float s_g[kRowsPerTile][kMaxClasses];
  const int KP = p.K + 1, E = p.kq * p.K;
  for (int i = threadIdx.x; i < E; i += blockDim.x) s_L[(i / p.K) * KP + i % p.K] = ssc_L(p, i / p.K, i % p.K);
  constexpr int kEntries = kMaxKeep * kMaxClasses / kBlock;
  float acc[kEntries];
#pragma unroll
  for (int i = 0; i < kEntries; ++i) acc[i] = 0.f;
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  const int64_t r0 = sl.b * p.chunk, r1 = min(p.n, r0 + p.chunk);
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
    if (e < E) p.part[sl.b * E + e] = acc[i];
  }
}

// ---- Lovász-softmax (lovasz.py:186-219) -----------------------------------------------------------------------------
// labels: -1 = row left out (sorted last through error −1), a class in [0, C), or >= C = background of every class
constexpr int kTile = 1024, kItems = kTile / 256;

struct LovParams {
  const float* logits;
  int64_t P;
  int C, tiles;
  const int32_t* labels;
  float* probs;
  float* err;
  const float* err_sorted;
  const int64_t* perm;
  int32_t* off;          // [C][tiles + 1]: per-tile foreground counts, then their exclusive scan and the total
  float* part;           // [C][tiles]
  float* grad;
  float* loss;
  const float* g;
  float* dp;             // [P][C]
  float* dx;
};

__global__ void __launch_bounds__(256) k_lov_errors(const __grid_constant__ Group<LovParams> gr) {
  const Slot sl = slot_of(gr);
  const LovParams& p = gr.lv[sl.l];
  const int C = p.C;
  for (int64_t r = sl.b * blockDim.x + threadIdx.x; r < p.P; r += sl.nb * blockDim.x) {
    const float* x = p.logits + r * C;
    float m = x[0];
    for (int c = 1; c < C; ++c) m = fmaxf(m, x[c]);
    float z = 0.f;
    for (int c = 0; c < C; ++c) z += expf(x[c] - m);
    const int l = p.labels[r];
    for (int c = 0; c < C; ++c) {
      const float pr = expf(x[c] - m) / z;
      p.probs[r * C + c] = pr;
      p.err[(int64_t)c * p.P + r] = l < 0 ? -1.f : fabsf((l == c ? 1.f : 0.f) - pr);
    }
  }
}

__device__ __forceinline__ int fg_at(const int32_t* labels, const int64_t* perm, int64_t P, int c, int64_t i) {
  return i < P && __ldg(labels + __ldg(perm + (int64_t)c * P + i)) == c;
}

// per (tile, class): foreground count of the tile in sorted order
__global__ void __launch_bounds__(256) k_lov_tile_counts(const __grid_constant__ Group<LovParams> gr) {
  const Slot sl = slot_of(gr);
  const LovParams& p = gr.lv[sl.l];
  const int c = blockIdx.y;
  if (c >= p.C) return;
  __shared__ int s;
  if (threadIdx.x == 0) s = 0;
  __syncthreads();
  int v = 0;
  for (int k = 0; k < kItems; ++k) v += fg_at(p.labels, p.perm, p.P, c, sl.b * kTile + k * 256 + threadIdx.x);
  atomicAdd(&s, v);
  __syncthreads();
  if (threadIdx.x == 0) p.off[(int64_t)c * (p.tiles + 1) + sl.b] = s;
}

// per class: exclusive tile offsets in place, and the class's foreground total after them
__global__ void k_lov_tile_scan(const __grid_constant__ Group<LovParams> gr) {
  const Slot sl = slot_of(gr);
  const LovParams& p = gr.lv[sl.l];
  const int c = threadIdx.x;
  if (c >= p.C) return;
  int32_t* t = p.off + (int64_t)c * (p.tiles + 1);
  int acc = 0;
  for (int i = 0; i < p.tiles; ++i) {
    const int v = t[i];
    t[i] = acc;
    acc += v;
  }
  t[p.tiles] = acc;
}

// lovasz_grad at every sorted position: jaccard_i = 1 − (gts − cumfg_i) / (gts + cumbg_i), grad_i = jaccard_i −
// jaccard_{i−1}; writes grad and the tile's partial of Σ err_i · grad_i
__global__ void __launch_bounds__(256) k_lov_grad(const __grid_constant__ Group<LovParams> gr) {
  const Slot sl = slot_of(gr);
  const LovParams& p = gr.lv[sl.l];
  const int c = blockIdx.y;
  if (c >= p.C) return;
  const int64_t P = p.P, base = sl.b * kTile + threadIdx.x * kItems;
  const int32_t* o = p.off + (int64_t)c * (p.tiles + 1);
  const int gts = o[p.tiles];
  int fg[kItems], run = 0;
#pragma unroll
  for (int k = 0; k < kItems; ++k) {
    fg[k] = fg_at(p.labels, p.perm, P, c, base + k);
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
  int cum = o[sl.b] + s_scan[threadIdx.x] - run;             // foreground before this thread's first item
  float dot = 0.f;
#pragma unroll
  for (int k = 0; k < kItems; ++k) {
    const int64_t i = base + k;
    if (i >= P) break;
    const float e = __ldg(p.err_sorted + (int64_t)c * P + i);
    const int before = cum;
    cum += fg[k];
    const float jac = 1.f - (float)(gts - cum) / (float)(gts + (int)(i + 1 - cum));
    float g = jac;
    if (i > 0) {
      const int bg_prev = (int)(i - before);
      g -= 1.f - (float)(gts - before) / (float)(gts + bg_prev);
    }
    if (e < 0.f) g = 0.f;                                     // a row left out: after every kept row
    p.grad[(int64_t)c * P + i] = g;
    dot += e < 0.f ? 0.f : e * g;
  }
  s_red[threadIdx.x] = dot;
  __syncthreads();
  for (int s = 128; s; s >>= 1) {
    if (threadIdx.x < s) s_red[threadIdx.x] += s_red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) p.part[(int64_t)c * p.tiles + sl.b] = s_red[0];
}

__global__ void k_lov_class_sum(const __grid_constant__ Group<LovParams> gr) {
  const Slot sl = slot_of(gr);
  const LovParams& p = gr.lv[sl.l];
  const int c = threadIdx.x;
  if (c >= p.C) return;
  float s = 0.f;
  for (int i = 0; i < p.tiles; ++i) s += p.part[(int64_t)c * p.tiles + i];
  p.loss[c] = s;
}

// dL/dp at the unsorted positions: g_c · grad_i · sign(p − fg)
__global__ void __launch_bounds__(256) k_lov_scatter(const __grid_constant__ Group<LovParams> gr) {
  const Slot sl = slot_of(gr);
  const LovParams& p = gr.lv[sl.l];
  const int C = p.C;
  const int64_t total = p.P * C;
  for (int64_t i = sl.b * blockDim.x + threadIdx.x; i < total; i += sl.nb * blockDim.x) {
    const int c = (int)(i / p.P);
    const int64_t r = __ldg(p.perm + i);
    const int l = __ldg(p.labels + r);
    if (l < 0) continue;
    const float d = __ldg(p.probs + r * C + c) - (l == c ? 1.f : 0.f);
    const float sg = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);
    p.dp[r * C + c] = __ldg(p.g + c) * __ldg(p.grad + i) * sg;
  }
}

__global__ void __launch_bounds__(256) k_lov_softmax_backward(const __grid_constant__ Group<LovParams> gr) {
  const Slot sl = slot_of(gr);
  const LovParams& p = gr.lv[sl.l];
  const int C = p.C;
  for (int64_t r = sl.b * blockDim.x + threadIdx.x; r < p.P; r += sl.nb * blockDim.x) {
    float s = 0.f;
    for (int c = 0; c < C; ++c) s += p.dp[r * C + c] * p.probs[r * C + c];
    for (int c = 0; c < C; ++c) p.dx[r * C + c] = p.probs[r * C + c] * (p.dp[r * C + c] - s);
  }
}

// ---- drivers over a level table -------------------------------------------------------------------------------------
// Each takes `count` levels, checks every level as its one-level entry point does, takes one workspace for the whole
// table and launches each pass once per run of kMaxLevels levels.
using Level = pasco_setloss_level;
using Term = pasco_lovasz_term;

int reduce_group(const char* name, int count, const ReduceParams* r, cudaStream_t st) {
  return for_groups<ReduceParams>(
      name, count, [&](int l, ReduceParams& p) { p = r[l]; return p.L > 0 ? grid_for(p.L, 256, 4) : 0; },
      [&](const Group<ReduceParams>& g, int grid) { k_sl_reduce<<<grid, 256, 0, st>>>(g); });
}

int keep_levels(const char* name, const Level* lv, int count, cudaStream_t st) {
  for (int l = 0; l < count; ++l)
    PASCO_CHECK_ARG(lv[l].Q >= 1 && lv[l].Q <= 4096 && lv[l].K1 >= 2 && lv[l].K1 <= kMaxClasses + 1,
                    "%s: level %d: 1 <= queries <= 4096, 2 <= classes + 1 <= %d", name, l, kMaxClasses + 1);
  return for_groups<KeepParams>(
      name, count,
      [&](int l, KeepParams& p) {
        p = {lv[l].query_logits, lv[l].Q, lv[l].K1, lv[l].keep, lv[l].kept};
        return 1;
      },
      [&](const Group<KeepParams>& g, int grid) { k_sl_keep<<<grid, kBlock, 0, st>>>(g); });
}

int cost_levels(const char* name, const Level* lv, int count, float cost_mask, float cost_class, float cost_dice,
                cudaStream_t st) {
  std::vector<CostParams> cp(count);
  std::vector<int> G(count, 0);
  size_t total = 0;
  int yt = 1, wz = 1;
  for (int l = 0; l < count; ++l) {
    const Level& v = lv[l];
    PASCO_CHECK_ARG(v.n >= 0 && v.Q >= 1 && v.T >= 0 && v.K1 >= 2, "%s: level %d: bad sizes", name, l);
    if (v.T == 0) continue;
    CostParams& p = cp[l];
    p = {};
    p.F = v.F;
    p.n = v.n;
    p.Q = v.Q;
    p.W = (v.T + 31) / 32;
    p.bits = v.bits;
    p.flags = v.flags;
    G[l] = chunks_for(v.n, 512);
    p.chunk = v.n > 0 ? (v.n + G[l] - 1) / G[l] : 1;
    p.L = (int64_t)v.Q * (3 * p.W * 32 + 2);
    total += (size_t)p.L * (G[l] + 1);
    yt = max(yt, (v.Q + kBlock - 1) / kBlock);
    wz = max(wz, p.W);
  }
  if (total == 0) return 0;
  float* ws = nullptr;
  cudaError_t e = ws_alloc((void**)&ws, sizeof(float) * total, st);
  PASCO_CHECK_ARG(e == cudaSuccess, "%s: workspace: %s", name, cudaGetErrorString(e));
  // per level: the reduced sums [L], then the partials [G][L]
  std::vector<ReduceParams> rp(count, ReduceParams{nullptr, 0, 0, nullptr});
  size_t at = 0;
  for (int l = 0; l < count; ++l) {
    if (!G[l]) continue;
    rp[l] = {ws + at + cp[l].L, G[l], cp[l].L, ws + at};
    cp[l].part = ws + at + cp[l].L;
    at += (size_t)cp[l].L * (G[l] + 1);
  }
  if (for_groups<CostParams>(
          name, count, [&](int l, CostParams& p) { p = cp[l]; return G[l]; },
          [&](const Group<CostParams>& g, int grid) { k_sl_cost<<<dim3(grid, yt, wz), kBlock, 0, st>>>(g); }))
    return -1;
  if (reduce_group(name, count, rp.data(), st)) return -1;
  if (for_groups<FinishParams>(
          name, count,
          [&](int l, FinishParams& f) {
            const Level& v = lv[l];
            f = {rp[l].out, v.stats, v.query_logits, v.K1, v.ids, v.class_weight, v.Q, v.T, cp[l].W, cost_mask,
                 cost_class, cost_dice, v.C};
            return G[l] ? (v.Q * v.T + 127) / 128 : 0;
          },
          [&](const Group<FinishParams>& g, int grid) { k_sl_cost_finish<<<grid, 128, 0, st>>>(g); }))
    return -1;
  cudaFreeAsync(ws, st);
  return 0;
}

PairParams pair_params(const Level& v) {
  PairParams p = {};
  p.F = v.F;
  p.n = v.n;
  p.Q = v.Q;
  p.W = (v.T + 31) / 32;
  p.bits = v.bits;
  p.flags = v.flags;
  p.qi = v.qi;
  p.tj = v.tj;
  p.P = v.P;
  p.g = v.g_sums;
  p.gF = v.gF_pairs;
  return p;
}

int pair_sums_levels(const char* name, const Level* lv, int count, cudaStream_t st) {
  std::vector<PairParams> pp(count);
  std::vector<ReduceParams> rp(count, ReduceParams{nullptr, 0, 0, nullptr});
  std::vector<int> G(count, 0);
  size_t total = 0;
  int yt = 1;
  for (int l = 0; l < count; ++l) {
    const Level& v = lv[l];
    PASCO_CHECK_ARG(v.n >= 0 && v.Q >= 1 && v.T >= 1 && v.P >= 0, "%s: level %d: bad sizes", name, l);
    if (v.P == 0) continue;
    pp[l] = pair_params(v);
    G[l] = chunks_for(v.n, 512);
    pp[l].chunk = v.n > 0 ? (v.n + G[l] - 1) / G[l] : 1;
    total += (size_t)G[l] * v.P * 4;
    yt = max(yt, (v.P + kBlock - 1) / kBlock);
  }
  if (total == 0) return 0;
  float* ws = nullptr;
  cudaError_t e = ws_alloc((void**)&ws, sizeof(float) * total, st);
  PASCO_CHECK_ARG(e == cudaSuccess, "%s: workspace: %s", name, cudaGetErrorString(e));
  size_t at = 0;
  for (int l = 0; l < count; ++l) {
    if (!G[l]) continue;
    pp[l].part = ws + at;
    rp[l] = {ws + at, G[l], (int64_t)lv[l].P * 4, lv[l].sums};
    at += (size_t)G[l] * lv[l].P * 4;
  }
  if (for_groups<PairParams>(
          name, count, [&](int l, PairParams& p) { p = pp[l]; return G[l]; },
          [&](const Group<PairParams>& g, int grid) { k_sl_pair_sums<<<dim3(grid, yt), kBlock, 0, st>>>(g); }))
    return -1;
  if (reduce_group(name, count, rp.data(), st)) return -1;
  cudaFreeAsync(ws, st);
  return 0;
}

int pair_backward_levels(const char* name, const Level* lv, int count, cudaStream_t st) {
  for (int l = 0; l < count; ++l)
    PASCO_CHECK_ARG(lv[l].n >= 0 && lv[l].Q >= 1 && lv[l].T >= 1 && lv[l].P >= 0, "%s: level %d: bad sizes", name, l);
  return for_groups<PairParams>(
      name, count,
      [&](int l, PairParams& p) {
        p = pair_params(lv[l]);
        return (p.P == 0 || p.n == 0) ? 0 : grid_for(p.n * p.P, kBlock, 8);
      },
      [&](const Group<PairParams>& g, int grid) { k_sl_pair_backward<<<grid, kBlock, 0, st>>>(g); });
}

int ssc_check(const char* name, const Level* lv, int count) {
  for (int l = 0; l < count; ++l) {
    const Level& v = lv[l];
    PASCO_CHECK_ARG(v.kq >= 0, "%s: level %d: kept queries < 0", name, l);
    if (v.kq == 0) continue;                                  // no ssc term: the level's other fields are not read
    PASCO_CHECK_ARG(v.kq <= kMaxKeep && v.K >= 1 && v.K <= kMaxClasses && v.kq <= v.Q && v.n >= 0,
                    "%s: level %d: 1 <= kept queries <= %d, 1 <= classes <= %d", name, l, kMaxKeep, kMaxClasses);
  }
  return 0;
}

SscParams ssc_params(const Level& v) {
  SscParams p = {};
  p.F = v.F;
  p.n = v.n;
  p.Q = v.Q;
  p.keep = v.keep;
  p.kq = v.kq;
  p.L = v.L;
  p.Lrows = v.L_rows;
  p.ldL = v.ldL;
  p.K = v.K;
  p.out = v.ssc;
  p.g = v.g_ssc;
  p.gF = v.gF_ssc;
  return p;
}

int ssc_forward_levels(const char* name, const Level* lv, int count, cudaStream_t st) {
  if (ssc_check(name, lv, count)) return -2;
  return for_groups<SscParams>(
      name, count,
      [&](int l, SscParams& p) {
        p = ssc_params(lv[l]);
        return (p.kq == 0 || p.n == 0) ? 0 : grid_for(p.n, kBlock / 32, 8);
      },
      [&](const Group<SscParams>& g, int grid) { k_sl_ssc_forward<<<grid, kBlock, 0, st>>>(g); });
}

int ssc_backward_levels(const char* name, const Level* lv, int count, cudaStream_t st) {
  if (ssc_check(name, lv, count)) return -2;
  std::vector<SscParams> sp(count);
  std::vector<ReduceParams> rp(count, ReduceParams{nullptr, 0, 0, nullptr});
  std::vector<int> G(count, 0);
  size_t total = 0;
  for (int l = 0; l < count; ++l) {
    if (lv[l].kq == 0) continue;
    sp[l] = ssc_params(lv[l]);
    G[l] = chunks_for(lv[l].n, 512);
    sp[l].chunk = lv[l].n > 0 ? (lv[l].n + G[l] - 1) / G[l] : 1;
    total += (size_t)G[l] * lv[l].kq * lv[l].K;
  }
  if (total == 0) return 0;
  float* ws = nullptr;
  cudaError_t e = ws_alloc((void**)&ws, sizeof(float) * total, st);
  PASCO_CHECK_ARG(e == cudaSuccess, "%s: workspace: %s", name, cudaGetErrorString(e));
  size_t at = 0;
  for (int l = 0; l < count; ++l) {
    if (!G[l]) continue;
    const int64_t E = (int64_t)lv[l].kq * lv[l].K;
    sp[l].part = ws + at;
    rp[l] = {ws + at, G[l], E, lv[l].gL};
    at += (size_t)G[l] * E;
  }
  if (for_groups<SscParams>(
          name, count, [&](int l, SscParams& p) { p = sp[l]; return G[l]; },
          [&](const Group<SscParams>& g, int grid) { k_sl_ssc_backward<<<grid, kBlock, 0, st>>>(g); }))
    return -1;
  if (reduce_group(name, count, rp.data(), st)) return -1;
  cudaFreeAsync(ws, st);
  return 0;
}

LovParams lov_params(const Term& t) {
  LovParams p = {};
  p.logits = t.logits;
  p.P = t.P;
  p.C = t.C;
  p.labels = t.labels;
  p.probs = t.probs;
  p.err = t.err;
  p.err_sorted = t.err_sorted;
  p.perm = t.perm;
  p.grad = t.grad;
  p.loss = t.loss;
  p.g = t.g;
  p.dx = t.dx;
  return p;
}

int lov_errors_terms(const char* name, const Term* t, int count, cudaStream_t st) {
  for (int l = 0; l < count; ++l)
    PASCO_CHECK_ARG(t[l].P >= 0 && t[l].C >= 1 && t[l].C <= 64, "%s: term %d: 1 <= classes <= 64 (got %d)", name, l,
                    t[l].C);
  return for_groups<LovParams>(
      name, count,
      [&](int l, LovParams& p) {
        p = lov_params(t[l]);
        return p.P == 0 ? 0 : grid_for(p.P, 256, 4);
      },
      [&](const Group<LovParams>& g, int grid) { k_lov_errors<<<grid, 256, 0, st>>>(g); });
}

int lov_grad_terms(const char* name, const Term* t, int count, cudaStream_t st) {
  std::vector<LovParams> lp(count);
  size_t total = 0;
  for (int l = 0; l < count; ++l) {
    PASCO_CHECK_ARG(t[l].P >= 1 && t[l].C >= 1 && t[l].C <= 64, "%s: term %d: bad sizes", name, l);
    const int64_t tiles64 = (t[l].P + kTile - 1) / kTile;
    PASCO_CHECK_ARG(tiles64 < (1 << 30), "%s: term %d: too many rows", name, l);
    lp[l] = lov_params(t[l]);
    lp[l].tiles = (int)tiles64;
    total += sizeof(int32_t) * (size_t)t[l].C * (lp[l].tiles + 1) + sizeof(float) * (size_t)t[l].C * lp[l].tiles;
  }
  if (count == 0) return 0;
  char* ws = nullptr;
  cudaError_t e = ws_alloc((void**)&ws, total, st);
  PASCO_CHECK_ARG(e == cudaSuccess, "%s: workspace: %s", name, cudaGetErrorString(e));
  size_t at = 0;
  for (int l = 0; l < count; ++l) {
    // counts written with a stride of tiles + 1 so the scan can append each class's total in place
    lp[l].off = (int32_t*)(ws + at);
    at += sizeof(int32_t) * (size_t)lp[l].C * (lp[l].tiles + 1);
    lp[l].part = (float*)(ws + at);
    at += sizeof(float) * (size_t)lp[l].C * lp[l].tiles;
  }
  int cmax = 1;
  for (int l = 0; l < count; ++l) cmax = max(cmax, lp[l].C);
  auto tiled = [&](int l, LovParams& p) { p = lp[l]; return p.tiles; };
  auto single = [&](int l, LovParams& p) { p = lp[l]; return 1; };
  if (for_groups<LovParams>(name, count, tiled, [&](const Group<LovParams>& g, int grid) {
        k_lov_tile_counts<<<dim3(grid, cmax), 256, 0, st>>>(g);
      }))
    return -1;
  if (for_groups<LovParams>(name, count, single,
                            [&](const Group<LovParams>& g, int grid) { k_lov_tile_scan<<<grid, 64, 0, st>>>(g); }))
    return -1;
  if (for_groups<LovParams>(name, count, tiled, [&](const Group<LovParams>& g, int grid) {
        k_lov_grad<<<dim3(grid, cmax), 256, 0, st>>>(g);
      }))
    return -1;
  if (for_groups<LovParams>(name, count, single,
                            [&](const Group<LovParams>& g, int grid) { k_lov_class_sum<<<grid, 64, 0, st>>>(g); }))
    return -1;
  cudaFreeAsync(ws, st);
  return 0;
}

int lov_backward_terms(const char* name, const Term* t, int count, cudaStream_t st) {
  std::vector<LovParams> lp(count);
  size_t total = 0;
  for (int l = 0; l < count; ++l) {
    PASCO_CHECK_ARG(t[l].P >= 0 && t[l].C >= 1 && t[l].C <= 64, "%s: term %d: bad sizes", name, l);
    lp[l] = lov_params(t[l]);
    total += (size_t)t[l].P * t[l].C;
  }
  if (total == 0) return 0;
  float* dp = nullptr;
  cudaError_t e = ws_alloc((void**)&dp, sizeof(float) * total, st);
  PASCO_CHECK_ARG(e == cudaSuccess, "%s: workspace: %s", name, cudaGetErrorString(e));
  cudaMemsetAsync(dp, 0, sizeof(float) * total, st);
  size_t at = 0;
  for (int l = 0; l < count; ++l) {
    lp[l].dp = dp + at;
    at += (size_t)t[l].P * t[l].C;
  }
  if (for_groups<LovParams>(
          name, count,
          [&](int l, LovParams& p) {
            p = lp[l];
            return p.P == 0 ? 0 : grid_for(p.P * p.C, 256, 8);
          },
          [&](const Group<LovParams>& g, int grid) { k_lov_scatter<<<grid, 256, 0, st>>>(g); }))
    return -1;
  if (for_groups<LovParams>(
          name, count,
          [&](int l, LovParams& p) {
            p = lp[l];
            return p.P == 0 ? 0 : grid_for(p.P, 256, 4);
          },
          [&](const Group<LovParams>& g, int grid) { k_lov_softmax_backward<<<grid, 256, 0, st>>>(g); }))
    return -1;
  cudaFreeAsync(dp, st);
  return 0;
}

Level one_level(const float* F, int64_t n, int32_t Q, const uint32_t* bits, int32_t T, const uint8_t* flags) {
  Level v = {};
  v.F = F;
  v.n = n;
  v.Q = Q;
  v.T = T;
  v.bits = bits;
  v.flags = flags;
  return v;
}

Level ssc_level(const float* F, int64_t n, int32_t Q, const int32_t* keep, int32_t kq, const float* L, int32_t K) {
  Level v = one_level(F, n, Q, nullptr, 0, nullptr);
  v.keep = const_cast<int32_t*>(keep);
  v.kq = kq;
  v.L = L;
  v.ldL = K;
  v.K = K;
  return v;
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
  Level v = one_level(F, n, Q, bits, T, flags);
  v.stats = stats;
  v.query_logits = query_logits;
  v.K1 = K1;
  v.ids = ids;
  v.class_weight = class_weight;
  v.C = C;
  return cost_levels("pasco_setloss_match_cost", &v, 1, cost_mask, cost_class, cost_dice, (cudaStream_t)s);
}

extern "C" int pasco_setloss_pair_sums(const float* F, int64_t n, int32_t Q, const uint32_t* bits, int32_t T,
                                       const uint8_t* flags, const int32_t* qi, const int32_t* tj, int32_t P,
                                       float* sums, pasco_stream_t s) {
  Level v = one_level(F, n, Q, bits, T, flags);
  v.qi = qi;
  v.tj = tj;
  v.P = P;
  v.sums = sums;
  return pair_sums_levels("pasco_setloss_pair_sums", &v, 1, (cudaStream_t)s);
}

extern "C" int pasco_setloss_pair_backward(const float* F, int64_t n, int32_t Q, const uint32_t* bits, int32_t T,
                                           const uint8_t* flags, const int32_t* qi, const int32_t* tj, int32_t P,
                                           const float* g, float* gF, pasco_stream_t s) {
  Level v = one_level(F, n, Q, bits, T, flags);
  v.qi = qi;
  v.tj = tj;
  v.P = P;
  v.g_sums = g;
  v.gF_pairs = gF;
  return pair_backward_levels("pasco_setloss_pair_backward", &v, 1, (cudaStream_t)s);
}

extern "C" int pasco_setloss_ssc_forward(const float* F, int64_t n, int32_t Q, const int32_t* keep, int32_t kq,
                                         const float* L, int32_t K, float* out, pasco_stream_t s) {
  PASCO_CHECK_ARG(kq >= 1, "pasco_setloss_ssc_forward: 1 <= kept queries <= %d, 1 <= classes <= %d", kMaxKeep,
                  kMaxClasses);
  Level v = ssc_level(F, n, Q, keep, kq, L, K);
  v.ssc = out;
  return ssc_forward_levels("pasco_setloss_ssc_forward", &v, 1, (cudaStream_t)s);
}

extern "C" int pasco_setloss_ssc_backward(const float* F, int64_t n, int32_t Q, const int32_t* keep, int32_t kq,
                                          const float* L, int32_t K, const float* out, const float* g, float* gF,
                                          float* gL, pasco_stream_t s) {
  PASCO_CHECK_ARG(kq >= 1, "pasco_setloss_ssc_backward: 1 <= kept queries <= %d, 1 <= classes <= %d", kMaxKeep,
                  kMaxClasses);
  Level v = ssc_level(F, n, Q, keep, kq, L, K);
  v.ssc = const_cast<float*>(out);
  v.g_ssc = g;
  v.gF_ssc = gF;
  v.gL = gL;
  return ssc_backward_levels("pasco_setloss_ssc_backward", &v, 1, (cudaStream_t)s);
}

extern "C" int pasco_lovasz_errors(const float* logits, int64_t P, int32_t C, const int32_t* labels, float* probs,
                                   float* err, pasco_stream_t s) {
  Term t = {};
  t.logits = logits;
  t.P = P;
  t.C = C;
  t.labels = labels;
  t.probs = probs;
  t.err = err;
  return lov_errors_terms("pasco_lovasz_errors", &t, 1, (cudaStream_t)s);
}

extern "C" int pasco_lovasz_grad(const float* err_sorted, const int64_t* perm, const int32_t* labels, int64_t P,
                                 int32_t C, float* grad, float* loss, pasco_stream_t s) {
  Term t = {};
  t.err_sorted = err_sorted;
  t.perm = perm;
  t.labels = labels;
  t.P = P;
  t.C = C;
  t.grad = grad;
  t.loss = loss;
  return lov_grad_terms("pasco_lovasz_grad", &t, 1, (cudaStream_t)s);
}

extern "C" int pasco_lovasz_backward(const float* probs, const int32_t* labels, const int64_t* perm, const float* grad,
                                     const float* g, int64_t P, int32_t C, float* dx, pasco_stream_t s) {
  Term t = {};
  t.probs = const_cast<float*>(probs);
  t.labels = labels;
  t.perm = perm;
  t.grad = const_cast<float*>(grad);
  t.g = g;
  t.P = P;
  t.C = C;
  t.dx = dx;
  return lov_backward_terms("pasco_lovasz_backward", &t, 1, (cudaStream_t)s);
}

extern "C" int pasco_setloss_keep_group(const pasco_setloss_level* lv, int32_t count, pasco_stream_t s) {
  PASCO_CHECK_ARG(count >= 0 && (count == 0 || lv), "pasco_setloss_keep_group: bad table");
  return keep_levels("pasco_setloss_keep_group", lv, count, (cudaStream_t)s);
}

extern "C" int pasco_setloss_match_cost_group(const pasco_setloss_level* lv, int32_t count, float cost_mask,
                                              float cost_class, float cost_dice, pasco_stream_t s) {
  PASCO_CHECK_ARG(count >= 0 && (count == 0 || lv), "pasco_setloss_match_cost_group: bad table");
  return cost_levels("pasco_setloss_match_cost_group", lv, count, cost_mask, cost_class, cost_dice, (cudaStream_t)s);
}

extern "C" int pasco_setloss_pair_sums_group(const pasco_setloss_level* lv, int32_t count, pasco_stream_t s) {
  PASCO_CHECK_ARG(count >= 0 && (count == 0 || lv), "pasco_setloss_pair_sums_group: bad table");
  return pair_sums_levels("pasco_setloss_pair_sums_group", lv, count, (cudaStream_t)s);
}

extern "C" int pasco_setloss_pair_backward_group(const pasco_setloss_level* lv, int32_t count, pasco_stream_t s) {
  PASCO_CHECK_ARG(count >= 0 && (count == 0 || lv), "pasco_setloss_pair_backward_group: bad table");
  return pair_backward_levels("pasco_setloss_pair_backward_group", lv, count, (cudaStream_t)s);
}

extern "C" int pasco_setloss_ssc_forward_group(const pasco_setloss_level* lv, int32_t count, pasco_stream_t s) {
  PASCO_CHECK_ARG(count >= 0 && (count == 0 || lv), "pasco_setloss_ssc_forward_group: bad table");
  return ssc_forward_levels("pasco_setloss_ssc_forward_group", lv, count, (cudaStream_t)s);
}

extern "C" int pasco_setloss_ssc_backward_group(const pasco_setloss_level* lv, int32_t count, pasco_stream_t s) {
  PASCO_CHECK_ARG(count >= 0 && (count == 0 || lv), "pasco_setloss_ssc_backward_group: bad table");
  return ssc_backward_levels("pasco_setloss_ssc_backward_group", lv, count, (cudaStream_t)s);
}

extern "C" int pasco_lovasz_errors_group(const pasco_lovasz_term* t, int32_t count, pasco_stream_t s) {
  PASCO_CHECK_ARG(count >= 0 && (count == 0 || t), "pasco_lovasz_errors_group: bad table");
  return lov_errors_terms("pasco_lovasz_errors_group", t, count, (cudaStream_t)s);
}

extern "C" int pasco_lovasz_grad_group(const pasco_lovasz_term* t, int32_t count, pasco_stream_t s) {
  PASCO_CHECK_ARG(count >= 0 && (count == 0 || t), "pasco_lovasz_grad_group: bad table");
  return lov_grad_terms("pasco_lovasz_grad_group", t, count, (cudaStream_t)s);
}

extern "C" int pasco_lovasz_backward_group(const pasco_lovasz_term* t, int32_t count, pasco_stream_t s) {
  PASCO_CHECK_ARG(count >= 0 && (count == 0 || t), "pasco_lovasz_backward_group: bad table");
  return lov_backward_terms("pasco_lovasz_backward_group", t, count, (cudaStream_t)s);
}
