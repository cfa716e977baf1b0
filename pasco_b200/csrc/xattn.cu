// Masked cross-attention of a few hundred queries over ALL voxels of a scale, sm_90a (wgmma).
//
//   O[q, h, :] = Σ_v softmax_v( Q[q,h,:]·K[v,h,:]·scale + mask[q,v] ) · V[v,h,:]
//
// (pasco/models/transformer/blocks.py:73-92 with the attention mask of transformer_predictor_v2.py:220-289: 100 queries,
// 8 heads of width 48, P = 25 k … 400 k keys.)  Q is tiny and P huge, so the kernel streams K and V once per pass
// through shared memory and keeps the query operand resident; FLOPs are negligible, the roofline is HBM:
// 2 passes x P x H x D x 4 B (K twice, V once).
//
// Two passes share one kernel template (no online-softmax rescaling of the accumulator is needed):
//   PASS 0  S = Q_h·K_hᵀ per 64-key tile (wgmma, 2 x M=64 queries, N=64 keys, K=64 padded head dim) → per (chunk, h, q)
//           running max m and Σ exp(s − m); `k_xattn_lse` merges the chunks into lse[h, q].
//   PASS 1  S again, p = exp(s − lse) (already normalised), P → bf16 (hi+lo) K-major smem tile, O_h += P·V_h (wgmma,
//           V tile as MN-major B operand), accumulated in registers over all tiles of the CTA; `k_xattn_osum` adds
//           the chunks' shares in chunk order (deterministic: the attention mask of the next layer thresholds O-derived
//           logits, so run-to-run rounding differences could flip mask bits).
// A CTA = (query block of 128 rows, head, key chunk); Q <= 128 is one query block, and each further block of 128 queries
// streams K and V once more.  Warps 0-3 (one warpgroup): issue the MMAs, pass each result through a [64 col][128 row]
// fp32 scratch so that thread t then holds query row t (mask, exp, row statistics); warps 4-7: K/V tile gather (16
// lanes per 256-byte padded row segment, fp32 → bf16 hi/lo split, 128-byte swizzle).  Operands are split bf16x3 like
// the convolution ("fp32" mode).  The backward (below) shares the CTAs, the warp roles, the K/V producer, the operand
// staging and the mask bits with the forward; only the consumer bodies differ.
#include <initializer_list>
#include <math_constants.h>
#include "common.cuh"
#include "gmma.cuh"

using namespace pasco;
using namespace gmma;

namespace {

constexpr int BK = 64;                      // keys per tile
constexpr int QM = 128;                     // query rows of a query block (padded) = 2 x wgmma M
constexpr int DP = 64;                      // padded head dim = one 128-byte swizzle row of bf16
constexpr int TILE_Q = QM * 128;            // 16 KB: [128 rows][64] bf16
constexpr int TILE_K = BK * 128;            // 8 KB : [64 keys][64] bf16
constexpr int NTHREADS = 8 * 32;
constexpr int SCRATCH = 64 * QM * 4;        // 32 KB: one [64 col][128 row] fp32 accumulator, row-contiguous per column

// arguments of both forward passes and of the backward; the fields a kernel does not use are null
struct XParams {
  const float* q;       // [Q, H*D]
  const float* k;       // [P, H*D]
  const float* v;       // [P, H*D]
  const uint32_t* mask; // bit rows [Q, 2*ceil(P/64)]: bit j of word 2t + j/32 = key 64t + j masked; nullptr = none
  const float* lse;     // [H, Q]            (forward pass 1, backward)
  const float* out;     // [Q, H*D]          (backward: the forward's output)
  const float* dout;    // [Q, H*D]          (backward)
  float* dk;            // [P, H*D]          (backward)
  float* dv;            // [P, H*D]          (backward)
  float* ws;            // [chunks, H, Q, 2] (forward pass 0: row statistics of each chunk)
  float* part;          // [chunks, Q, H*D]  (this chunk's share of O in forward pass 1, of dQ in the backward)
  float* dkv;           // [nqb-1, 2, P, H*D] (backward, Q > 128: dK then dV of query blocks 1..; block 0 writes dk, dv)
  int Q, H, D;
  int64_t P;
  int chunks;
  float scale;
};

// smem layout (bytes from a 1024-aligned base)
//   Q_hi | Q_lo                                 2 x 16 KB
//   stage s (x2): K_hi | K_lo | V_hi | V_lo     4 x 8 KB
//   P_hi | P_lo                                 2 x 16 KB   (pass 1)
//   scratch                                     32 KB
constexpr int OFF_Q = 0;
constexpr int OFF_KV = 2 * TILE_Q;
constexpr int KV_STAGE = 4 * TILE_K;
constexpr int OFF_P = OFF_KV + 2 * KV_STAGE;
constexpr int OFF_SCR = OFF_P + 2 * TILE_Q;
constexpr int OFF_BAR = OFF_SCR + SCRATCH;
constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;

// D[128 rows][64] (+)= A[128 rows][16 k-steps of K-major smem, 64 K] · B[64 K][64 N], bf16x3; A K-major, B K-major (TB = 0)
// with 16-element k-steps of 32 bytes, or MN-major (TB = 1) with 16-row k-steps of 2048 bytes
template <int TB>
__device__ __forceinline__ void mma_rows128(float (&d)[2][32], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo) {
  const uint32_t b_step = TB ? 128u : 2u, b_lbo = TB ? TILE_K : 16;
#pragma unroll
  for (int hm = 0; hm < 2; ++hm) {
    const uint64_t ah = make_desc_sw128(a_hi + hm * 8192, 16, 1024), al = make_desc_sw128(a_lo + hm * 8192, 16, 1024);
    const uint64_t bh = make_desc_sw128(b_hi, b_lbo, 1024), bl = make_desc_sw128(b_lo, b_lbo, 1024);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      wgmma_n64<0, TB>(d[hm], ah + 2 * j, bh + b_step * j);
      wgmma_n64<0, TB>(d[hm], al + 2 * j, bh + b_step * j);
      wgmma_n64<0, TB>(d[hm], ah + 2 * j, bl + b_step * j);
    }
  }
}
__device__ __forceinline__ void zero_acc(float (&d)[2][32]) {
#pragma unroll
  for (int hm = 0; hm < 2; ++hm)
#pragma unroll
    for (int i = 0; i < 32; ++i) d[hm][i] = 0.f;
}
// accumulator fragments of the row warpgroup (thread t = warp w, lane l) → scratch[col][row] → v[j] = D[t][j]
__device__ __forceinline__ void acc_to_rows(const float (&d)[2][32], float* scr, float (&v)[64], int warp, int lane) {
  named_sync(1, 128);                  // the previous readers of the scratch are done
#pragma unroll
  for (int hm = 0; hm < 2; ++hm)
#pragma unroll
    for (int i = 0; i < 32; ++i) scr[frag_col(i, lane) * QM + hm * 64 + frag_row(i, warp, lane)] = d[hm][i];
  named_sync(1, 128);
  const int row = warp * 32 + lane;
#pragma unroll
  for (int j = 0; j < 64; ++j) v[j] = scr[j * QM + row];
}

// this CTA's query block (rows [q0, q0 + 128) of Q), head, key chunk, and its key tiles [t0, t0 + my_tiles) out of the
// n_tiles that cover P
struct CtaTiles {
  int qb, q0, h, chunk;
  int64_t n_tiles, t0, my_tiles;
};
__device__ __forceinline__ CtaTiles cta_tiles(const XParams& p) {
  CtaTiles c;
  c.qb = blockIdx.y;
  c.q0 = c.qb * QM;
  c.h = blockIdx.x % p.H;
  c.chunk = blockIdx.x / p.H;
  c.n_tiles = (p.P + BK - 1) / BK;
  const int64_t tiles_per_chunk = (c.n_tiles + p.chunks - 1) / p.chunks;
  c.t0 = (int64_t)c.chunk * tiles_per_chunk;
  const int64_t t1 = c.t0 + tiles_per_chunk < c.n_tiles ? c.t0 + tiles_per_chunk : c.n_tiles;
  c.my_tiles = t1 > c.t0 ? t1 - c.t0 : 0;
  return c;
}

// the two-stage K/V ring: full[s] takes one arrival per gather warp, empty[s] one per MMA warp
__device__ __forceinline__ void init_kv_ring(uint64_t* kv_full, uint64_t* kv_empty) {
  if (threadIdx.x == 0) {
    for (int i = 0; i < 2; ++i) {
      mbar_init(smem_u32(kv_full + i), 4);
      mbar_init(smem_u32(kv_empty + i), 4);
    }
    fence_barrier_init();
  }
}

// f[0..7] → bf16 hi / lo of 16-byte chunk c of row `row` in a [128 rows][64] tile pair (hi at `tile`, lo TILE_Q on)
__device__ __forceinline__ void store_split8(uint8_t* tile, uint32_t row, uint32_t c, const float* f) {
  uint2 h0, l0, h1, l1;
  split4(make_float4(f[0], f[1], f[2], f[3]), h0, l0);
  split4(make_float4(f[4], f[5], f[6], f[7]), h1, l1);
  const uint32_t off = sw128_off(row, c);
  *reinterpret_cast<uint4*>(tile + off) = make_uint4(h0.x, h0.y, h1.x, h1.y);
  *reinterpret_cast<uint4*>(tile + TILE_Q + off) = make_uint4(l0.x, l0.y, l1.x, l1.y);
}

// resident operand, all threads: head h's columns of rows [q0, q0 + 128) of the [Q, H*D] matrix `src` times `factor`
// → bf16 hi / lo [128 rows][64] at `tile`; rows >= Q and columns >= D are zero
__device__ __forceinline__ void stage_rows(uint8_t* tile, const float* src, float factor, const XParams& p, int q0, int h) {
  const int HD = p.H * p.D;
  for (int t = threadIdx.x; t < QM * 8; t += NTHREADS) {       // one 16-byte output chunk (8 bf16) per iteration
    const int row = t >> 3, c = t & 7;
    float f[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int d = c * 8 + j;
      f[j] = (q0 + row < p.Q && d < p.D) ? __ldg(src + (int64_t)(q0 + row) * HD + h * p.D + d) * factor : 0.f;
    }
    store_split8(tile, row, c, f);
  }
}

// warps 4-7 (16 keys per warp): the CTA's K tiles, and V tiles when WITH_V, into the two-stage ring at `ring`
template <bool WITH_V>
__device__ __forceinline__ void produce_kv(const XParams& p, const CtaTiles& ct, uint8_t* ring, uint64_t* kv_full,
                                           uint64_t* kv_empty, int warp, int lane) {
  const int HD = p.H * p.D;
  const int gw = warp - 4;
  const int chunk4 = lane & 15, rsub = lane >> 4;
  uint32_t phase = 0;
  for (int64_t it = 0; it < ct.my_tiles; ++it) {
    const int st = (int)(it & 1);
    const int64_t key0 = (ct.t0 + it) * BK;
    // loads first (before the stage is free)
    float4 kv[2][8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int r = gw * 16 + i * 2 + rsub;
      const int64_t key = key0 + r;
      const bool ok = key < p.P && chunk4 * 4 < p.D;
      kv[0][i] = ok ? __ldg(reinterpret_cast<const float4*>(p.k + key * HD + ct.h * p.D + chunk4 * 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
      if (WITH_V)
        kv[1][i] = ok ? __ldg(reinterpret_cast<const float4*>(p.v + key * HD + ct.h * p.D + chunk4 * 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    mbar_wait(smem_u32(kv_empty + st), phase ^ 1);
    uint8_t* base = ring + st * KV_STAGE;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const uint32_t off = sw128_half_off((uint32_t)(gw * 16 + i * 2 + rsub), (uint32_t)chunk4);
      uint2 hi, lo;
      split4(kv[0][i], hi, lo);
      *reinterpret_cast<uint2*>(base + off) = hi;
      *reinterpret_cast<uint2*>(base + TILE_K + off) = lo;
      if (WITH_V) {
        split4(kv[1][i], hi, lo);
        *reinterpret_cast<uint2*>(base + 2 * TILE_K + off) = hi;
        *reinterpret_cast<uint2*>(base + 3 * TILE_K + off) = lo;
      }
    }
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) mbar_arrive(smem_u32(kv_full + st));
    if (st == 1) phase ^= 1;
  }
}

// mask bits of (global) query row `qrow` for the 64 keys of `tile` (bit set = masked); keys >= P and rows >= Q are masked
__device__ __forceinline__ void tile_mask_bits(uint32_t (&mbits)[2], const XParams& p, int qrow, int64_t n_tiles,
                                               int64_t tile) {
  mbits[0] = mbits[1] = 0xffffffffu;
  if (qrow >= p.Q) return;
  if (p.mask) {
    const uint2 w = __ldg(reinterpret_cast<const uint2*>(p.mask + ((int64_t)qrow * n_tiles + tile) * 2));
    mbits[0] = w.x;
    mbits[1] = w.y;
  } else {
    mbits[0] = mbits[1] = 0u;
  }
  const int64_t left = p.P - tile * BK;
  if (left < 64) {
    if (left <= 32) {
      mbits[1] = 0xffffffffu;
      if (left < 32) mbits[0] |= ~0u << left;
    } else {
      mbits[1] |= ~0u << (left - 32);
    }
  }
}

template <int PASS>
__global__ void __launch_bounds__(NTHREADS, 1) k_xattn_fwd(const __grid_constant__ XParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
  uint64_t* kv_full = bars;        // [2]
  uint64_t* kv_empty = bars + 2;   // [2]
  float* scr = reinterpret_cast<float*>(smem + OFF_SCR);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const CtaTiles ct = cta_tiles(p);
  const int h = ct.h;
  const int HD = p.H * p.D;

  init_kv_ring(kv_full, kv_empty);
  stage_rows(smem + OFF_Q, p.q, p.scale, p, ct.q0, h);   // resident query operand Q_h * scale
  fence_proxy_async_smem();
  __syncthreads();

  if (warp >= 4) {
    produce_kv<PASS == 1>(p, ct, smem + OFF_KV, kv_full, kv_empty, warp, lane);
  } else {
    // ===================================== MMA + softmax rows (warps 0-3) =====================================
    const int row = warp * 32 + lane, qrow = ct.q0 + row;    // tile row, query row
    const bool qok = qrow < p.Q;
    const uint32_t q_hi = smem_u32(smem + OFF_Q), q_lo = q_hi + TILE_Q;
    const uint32_t p_hi = smem_u32(smem + OFF_P), p_lo = p_hi + TILE_Q;
    float m_run = -CUDART_INF_F, l_run = 0.f;
    const float my_lse = (PASS == 1 && qok) ? __ldg(p.lse + (int64_t)h * p.Q + qrow) : 0.f;
    float oacc[2][32];
    zero_acc(oacc);
    for (int64_t it = 0; it < ct.my_tiles; ++it) {
      const int st = (int)(it & 1);
      uint32_t mbits[2];
      tile_mask_bits(mbits, p, qrow, ct.n_tiles, ct.t0 + it);
      mbar_wait(smem_u32(kv_full + st), (uint32_t)((it >> 1) & 1));
      const uint32_t k_hi = smem_u32(smem + OFF_KV + st * KV_STAGE), k_lo = k_hi + TILE_K;
      float s[BK];
      {
        float sacc[2][32];
        zero_acc(sacc);
        wg_fence();
        mma_rows128<0>(sacc, q_hi, q_lo, k_hi, k_lo);   // S[128 q][64 keys] = Q (K-major) · K (K-major)
        wg_commit();
        wg_wait<0>();
        acc_to_rows(sacc, scr, s, warp, lane);
      }
      if (PASS == 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(kv_empty + st));
        float mx = m_run;
#pragma unroll
        for (int j = 0; j < BK; ++j)
          if (!((mbits[j >> 5] >> (j & 31)) & 1u)) mx = fmaxf(mx, s[j]);
        if (mx > -CUDART_INF_F) {
          float acc = l_run * __expf(m_run - mx);
#pragma unroll
          for (int j = 0; j < BK; ++j)
            if (!((mbits[j >> 5] >> (j & 31)) & 1u)) acc += __expf(s[j] - mx);
          l_run = acc;
          m_run = mx;
        }
      } else {
#pragma unroll
        for (int c = 0; c < 8; ++c) {       // 8 probabilities per 16-byte chunk
          float f[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int col = c * 8 + j;
            f[j] = ((mbits[col >> 5] >> (col & 31)) & 1u) ? 0.f : __expf(s[col] - my_lse);
          }
          store_split8(smem + OFF_P, (uint32_t)row, (uint32_t)c, f);
        }
        fence_proxy_async_smem();
        named_sync(1, 128);                 // the whole P tile is written
        const uint32_t v_hi = k_hi + 2 * TILE_K, v_lo = v_hi + TILE_K;
        wg_fence();
        mma_rows128<1>(oacc, p_hi, p_lo, v_hi, v_lo);   // O[128 q][64 d] += P (K-major) · V (MN-major)
        wg_commit();
        wg_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(kv_empty + st));
      }
    }
    if (PASS == 0) {
      if (qok) {
        float* w = p.ws + (((int64_t)ct.chunk * p.H + h) * p.Q + qrow) * 2;
        w[0] = m_run;
        w[1] = l_run;
      }
    } else {                                 // a chunk without tiles stores zeros
      float o[DP];
      acc_to_rows(oacc, scr, o, warp, lane);
      if (qok) {
        float* orow = p.part + ((int64_t)ct.chunk * p.Q + qrow) * HD + h * p.D;
#pragma unroll
        for (int d = 0; d < DP; ++d)
          if (d < p.D) orow[d] = o[d];
      }
    }
  }
}

__global__ void k_xattn_lse(const float* __restrict__ ws, int chunks, int HQ, float* __restrict__ lse) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= HQ) return;
  float M = -CUDART_INF_F;
  for (int c = 0; c < chunks; ++c) M = fmaxf(M, ws[((int64_t)c * HQ + i) * 2]);
  float L = 0.f;
  for (int c = 0; c < chunks; ++c) {
    const float m = ws[((int64_t)c * HQ + i) * 2], l = ws[((int64_t)c * HQ + i) * 2 + 1];
    if (m > -CUDART_INF_F) L += l * __expf(m - M);
  }
  lse[i] = M + logf(L);
}

// out[i] = Σ_c opart[c, i] in chunk order
__global__ void k_xattn_osum(const float* __restrict__ opart, int chunks, int64_t n, float* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float acc = 0.f;
    for (int c = 0; c < chunks; ++c) acc += __ldg(opart + c * n + i);
    out[i] = acc;
  }
}

// dk[i] (i < n) / dv[i - n] (i >= n) += dkv[b, i] for the query blocks b = 1.. in block order; n is a multiple of 4
__global__ void k_xattn_dkv_sum(const float4* __restrict__ dkv, int parts, int64_t n, float4* __restrict__ dk,
                                float4* __restrict__ dv) {
  const int64_t n4 = n / 4;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < 2 * n4; i += (int64_t)gridDim.x * blockDim.x) {
    float4* dst = i < n4 ? dk + i : dv + (i - n4);
    float4 acc = *dst;
    for (int b = 0; b < parts; ++b) {
      const float4 w = __ldg(dkv + b * 2 * n4 + i);
      acc.x += w.x; acc.y += w.y; acc.z += w.z; acc.w += w.w;
    }
    *dst = acc;
  }
}

// key chunks per (query block, head): ~one CTA per SM over the nqb x H x chunks grid
int pick_chunks(int64_t P, int H, int nqb) {
  int64_t tiles = (P + BK - 1) / BK;
  int c = (num_sms() + H * nqb - 1) / (H * nqb);
  if (c > tiles) c = (int)tiles;
  return c < 1 ? 1 : c;
}

// What both entry points do before their launches: check the shape, fill in the shape fields and the chunk count of
// `p`, opt the kernels in to `smem` bytes of shared memory, and take the chunks' shares `part` [chunks, Q, H*D] from the
// library's stream-ordered pool.  Behind them lie the forward's row statistics `ws` [chunks, H, Q, 2], or for the
// backward at Q > 128 the dK / dV partials `dkv` [nqb-1, 2, P, H*D].  Returns the number of query blocks nqb (< 0 on
// error); the caller frees p.part on the same stream after its launches.
int xattn_setup(const char* fn, XParams& p, int32_t Q, int64_t P, int32_t H, int32_t D, float scale, int smem,
                std::initializer_list<const void*> kernels, bool forward, cudaStream_t st) {
  PASCO_CHECK_ARG(Q >= 1 && Q <= 65535 * QM, "%s: Q (%d) must be in [1,%d]", fn, Q, 65535 * QM);
  PASCO_CHECK_ARG(D >= 4 && D <= DP && D % 4 == 0, "%s: head dim (%d) must be a multiple of 4, <= 64", fn, D);
  PASCO_CHECK_ARG(H >= 1 && P >= 1, "%s: bad shape (H = %d, P = %lld)", fn, H, (long long)P);
  p.Q = Q; p.H = H; p.D = D; p.P = P; p.scale = scale;
  const int nqb = (Q + QM - 1) / QM;
  p.chunks = pick_chunks(P, H, nqb);
  for (const void* k : kernels) {
    const cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) {
      set_error("%s: cudaFuncSetAttribute(%d) failed: %s", fn, smem, cudaGetErrorString(e));
      return -1;
    }
  }
  const int64_t n = (int64_t)p.chunks * Q * H * D;
  const int64_t extra = forward ? (int64_t)p.chunks * H * Q * 2 : (int64_t)(nqb - 1) * 2 * P * H * D;
  const cudaError_t e = ws_alloc((void**)&p.part, (size_t)(n + extra) * sizeof(float), st);
  if (e != cudaSuccess) {
    set_error("%s: workspace of %lld bytes: %s", fn, (long long)(n + extra) * 4, cudaGetErrorString(e));
    return -1;
  }
  p.ws = forward ? p.part + n : nullptr;
  p.dkv = !forward && nqb > 1 ? p.part + n : nullptr;
  return nqb;
}

}  // namespace

extern "C" int pasco_xattn_forward(const float* q, const float* k, const float* v, const uint32_t* mask, int32_t Q,
                                   int64_t P, int32_t H, int32_t D, float scale, float* out, float* lse,
                                   pasco_stream_t s) {
  PASCO_CHECK_ARG((((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)out) & 15) == 0, "pasco_xattn_forward: pointers must be 16-byte aligned");
  XParams p = {};
  p.q = q; p.k = k; p.v = v; p.mask = mask; p.lse = lse;
  cudaStream_t st = (cudaStream_t)s;
  const int nqb = xattn_setup("pasco_xattn_forward", p, Q, P, H, D, scale, SMEM_BYTES,
                              {(const void*)k_xattn_fwd<0>, (const void*)k_xattn_fwd<1>}, true, st);
  if (nqb < 0) return nqb;
  const dim3 grid(p.chunks * H, nqb);
  const int64_t n = (int64_t)Q * H * D;
  k_xattn_fwd<0><<<grid, NTHREADS, SMEM_BYTES, st>>>(p);
  k_xattn_lse<<<(H * Q + 127) / 128, 128, 0, st>>>(p.ws, p.chunks, H * Q, lse);
  k_xattn_fwd<1><<<grid, NTHREADS, SMEM_BYTES, st>>>(p);
  k_xattn_osum<<<grid_for(n, 256), 256, 0, st>>>(p.part, p.chunks, n, out);
  cudaFreeAsync(p.part, st);
  PASCO_CHECK_LAUNCH("pasco_xattn_forward");
  return 0;
}

// ==================================================================================================================
// backward:  given dO, recompute S and P from the saved log-sum-exp and produce dQ, dK, dV
//
//   P = exp(S − lse) (masked → 0),  dP = dO·Vᵀ,  dS = P ∘ (dP − rowsum(dO ∘ O)),
//   dV = Pᵀ·dO,  dK = dSᵀ·Qs,  dQ = scale · dS·K                       (Qs = scale·Q)
//
// Same CTA = (query block, head, key chunk) decomposition, warp roles and 64-key tiles as the forward.  Five wgmma GEMMs
// per tile:
//   S  [128q x 64k] = Qs(K-major) · K(K-major)            dP [128q x 64k] = dO(K-major) · V(K-major)
//   dVᵀ[ 64d x 64k] = dOᵀ(MN-major) · P(MN-major)          dKᵀ[ 64d x 64k] = Qsᵀ(MN-major) · dS(MN-major)
//   dQ [128q x 64d] += dS(K-major) · K(MN-major)              (accumulates in registers over the CTA's tiles)
// every dK/dV row is written exactly once per query block (no atomics): block 0 into dk / dv, blocks 1.. into a workspace
// that k_xattn_dkv_sum adds to dk / dv in block order.  Each (block, chunk) stores its share of dQ, k_xattn_osum adds
// the chunks' shares in order.
// ==================================================================================================================
namespace {

constexpr int B_OFF_Q = 0;                          // Qs hi | lo           2 x 16 KB
constexpr int B_OFF_DO = 2 * TILE_Q;                // dO hi | lo           2 x 16 KB
constexpr int B_OFF_KV = 4 * TILE_Q;                // 2 stages x (K hi|lo, V hi|lo) = 2 x 32 KB
constexpr int B_OFF_P = B_OFF_KV + 2 * KV_STAGE;    // P hi | lo            2 x 16 KB
constexpr int B_OFF_DS = B_OFF_P + 2 * TILE_Q;      // dS hi | lo           2 x 16 KB
constexpr int B_OFF_SCR = B_OFF_DS + 2 * TILE_Q;    // scratch              32 KB
constexpr int B_OFF_BAR = B_OFF_SCR + SCRATCH;
constexpr int B_SMEM_BYTES = B_OFF_BAR + 256 + 1024;

// D[64 d][64 keys] = Aᵀ·B over the 128 query rows: A, B tiles of [128 q rows][128 B], both MN-major
__device__ __forceinline__ void mma_t64(float (&d)[32], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo) {
  const uint64_t ah = make_desc_sw128(a_hi, TILE_Q, 1024), al = make_desc_sw128(a_lo, TILE_Q, 1024);
  const uint64_t bh = make_desc_sw128(b_hi, TILE_Q, 1024), bl = make_desc_sw128(b_lo, TILE_Q, 1024);
#pragma unroll
  for (int j = 0; j < QM / 16; ++j) {                  // 16 rows = 2048 bytes = 128 address units per k-step
    wgmma_n64<1, 1>(d, ah + 128 * j, bh + 128 * j);
    wgmma_n64<1, 1>(d, al + 128 * j, bh + 128 * j);
    wgmma_n64<1, 1>(d, ah + 128 * j, bl + 128 * j);
  }
}

__global__ void __launch_bounds__(NTHREADS, 1) k_xattn_bwd(const __grid_constant__ XParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + B_OFF_BAR);
  uint64_t* kv_full = bars;         // [2]
  uint64_t* kv_empty = bars + 2;    // [2]
  float* scr = reinterpret_cast<float*>(smem + B_OFF_SCR);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const CtaTiles ct = cta_tiles(p);
  const int h = ct.h;
  const int HD = p.H * p.D;

  init_kv_ring(kv_full, kv_empty);
  stage_rows(smem + B_OFF_Q, p.q, p.scale, p, ct.q0, h);    // resident operands: Qs = scale*Q_h and dO_h
  stage_rows(smem + B_OFF_DO, p.dout, 1.f, p, ct.q0, h);
  fence_proxy_async_smem();
  __syncthreads();

  if (warp >= 4) {
    produce_kv<true>(p, ct, smem + B_OFF_KV, kv_full, kv_empty, warp, lane);
  } else {
    // ===================================== MMA + query rows (warps 0-3) =====================================
    const int row = warp * 32 + lane, qrow = ct.q0 + row;    // tile row, query row
    const bool qok = qrow < p.Q;
    const uint32_t q_hi = smem_u32(smem + B_OFF_Q), q_lo = q_hi + TILE_Q;
    const uint32_t o_hi = smem_u32(smem + B_OFF_DO), o_lo = o_hi + TILE_Q;
    const uint32_t p_hi = smem_u32(smem + B_OFF_P), p_lo = p_hi + TILE_Q;
    const uint32_t s_hi = smem_u32(smem + B_OFF_DS), s_lo = s_hi + TILE_Q;
    float my_lse = 0.f, my_delta = 0.f;
    if (qok) {
      my_lse = __ldg(p.lse + (int64_t)h * p.Q + qrow);
      for (int d = 0; d < p.D; ++d)
        my_delta += __ldg(p.dout + (int64_t)qrow * HD + h * p.D + d) * __ldg(p.out + (int64_t)qrow * HD + h * p.D + d);
    }
    // query block 0 writes its dK / dV straight into dk / dv, blocks 1.. their partials into p.dkv
    float* dk = ct.qb == 0 ? p.dk : p.dkv + (int64_t)(ct.qb - 1) * 2 * p.P * HD;
    float* dv = ct.qb == 0 ? p.dv : dk + p.P * HD;
    float dq[2][32];
    zero_acc(dq);
    for (int64_t it = 0; it < ct.my_tiles; ++it) {
      const int st = (int)(it & 1);
      const int64_t key0 = (ct.t0 + it) * BK;
      uint32_t mbits[2];
      tile_mask_bits(mbits, p, qrow, ct.n_tiles, ct.t0 + it);
      mbar_wait(smem_u32(kv_full + st), (uint32_t)((it >> 1) & 1));
      const uint32_t k_hi = smem_u32(smem + B_OFF_KV + st * KV_STAGE), k_lo = k_hi + TILE_K;
      const uint32_t v_hi = k_hi + 2 * TILE_K, v_lo = v_hi + TILE_K;
      float pr[BK], ds[BK];
      {
        float acc[2][32], a[BK];
        zero_acc(acc);
        wg_fence();
        mma_rows128<0>(acc, q_hi, q_lo, k_hi, k_lo);    // S
        wg_commit();
        wg_wait<0>();
        acc_to_rows(acc, scr, a, warp, lane);
#pragma unroll
        for (int j = 0; j < BK; ++j) pr[j] = ((mbits[j >> 5] >> (j & 31)) & 1u) ? 0.f : __expf(a[j] - my_lse);
        zero_acc(acc);
        wg_fence();
        mma_rows128<0>(acc, o_hi, o_lo, v_hi, v_lo);    // dP
        wg_commit();
        wg_wait<0>();
        acc_to_rows(acc, scr, a, warp, lane);
#pragma unroll
        for (int j = 0; j < BK; ++j) ds[j] = pr[j] * (a[j] - my_delta);
      }
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        store_split8(smem + B_OFF_P, (uint32_t)row, (uint32_t)c, pr + c * 8);
        store_split8(smem + B_OFF_DS, (uint32_t)row, (uint32_t)c, ds + c * 8);
      }
      fence_proxy_async_smem();
      named_sync(1, 128);                               // the whole P / dS tiles are written
      {
        float dvt[32], dkt[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) dvt[i] = dkt[i] = 0.f;
        wg_fence();
        mma_t64(dvt, o_hi, o_lo, p_hi, p_lo);           // dVᵀ = dOᵀ · P
        mma_t64(dkt, q_hi, q_lo, s_hi, s_lo);           // dKᵀ = Qsᵀ · dS
        mma_rows128<1>(dq, s_hi, s_lo, k_hi, k_lo);     // dQ += dS · K   (K tile as MN-major B: 16 keys = 2 KB)
        wg_commit();
        wg_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(kv_empty + st));
#pragma unroll
        for (int i = 0; i < 32; ++i) {                  // row = head-dim index, column = key of the tile
          const int d = frag_row(i, warp, lane);
          const int64_t key = key0 + frag_col(i, lane);
          if (d < p.D && key < p.P) {
            dv[key * HD + h * p.D + d] = dvt[i];
            dk[key * HD + h * p.D + d] = dkt[i];
          }
        }
      }
    }
    {                                        // a chunk without tiles stores zeros
      float a[DP];
      acc_to_rows(dq, scr, a, warp, lane);
      if (qok) {
        float* row = p.part + ((int64_t)ct.chunk * p.Q + qrow) * HD + h * p.D;
#pragma unroll
        for (int d = 0; d < DP; ++d)
          if (d < p.D) row[d] = a[d] * p.scale;
      }
    }
  }
}

}  // namespace

extern "C" int pasco_xattn_backward(const float* q, const float* k, const float* v, const uint32_t* mask, const float* lse,
                                    const float* out, const float* dout, int32_t Q, int64_t P, int32_t H, int32_t D,
                                    float scale, float* dq, float* dk, float* dv, pasco_stream_t s) {
  PASCO_CHECK_ARG((((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)dq | (uintptr_t)dk | (uintptr_t)dv) & 15) == 0,
                  "pasco_xattn_backward: pointers must be 16-byte aligned");
  XParams p = {};
  p.q = q; p.k = k; p.v = v; p.mask = mask; p.lse = lse; p.out = out; p.dout = dout; p.dk = dk; p.dv = dv;
  cudaStream_t st = (cudaStream_t)s;
  const int nqb = xattn_setup("pasco_xattn_backward", p, Q, P, H, D, scale, B_SMEM_BYTES, {(const void*)k_xattn_bwd},
                              false, st);
  if (nqb < 0) return nqb;
  const int64_t n = (int64_t)Q * H * D;
  k_xattn_bwd<<<dim3(p.chunks * H, nqb), NTHREADS, B_SMEM_BYTES, st>>>(p);
  k_xattn_osum<<<grid_for(n, 256), 256, 0, st>>>(p.part, p.chunks, n, dq);
  if (nqb > 1) {
    const int64_t nkv = P * H * D;
    k_xattn_dkv_sum<<<grid_for(2 * nkv / 4, 256), 256, 0, st>>>((const float4*)p.dkv, nqb - 1, nkv, (float4*)dk,
                                                                 (float4*)dv);
  }
  cudaFreeAsync(p.part, st);
  PASCO_CHECK_LAUNCH("pasco_xattn_backward");
  return 0;
}
