// Sparse convolution on the Hopper tensor cores (wgmma), sm_90a.
//
//   out[o, :] = Σ_k  in[nbr[k, o], :] @ W[k]           (output-stationary implicit GEMM)
//
// One persistent CTA per SM walks work items of 128-row output tiles.  A work item is a GROUP of T consecutive tiles
// (T x the item's columns <= 128 accumulator columns) and walks offset k → 64-channel block → tile, so every weight
// slice W[k] is fetched from L2 once per group instead of once per tile.  Outputs wider than 128 channels are cut into
// column ranges, one work item each.  Warp roles:
//   warps 0-7   gather: load the neighbour rows of a tile (coalesced 16-byte loads, 16 lanes per 256-byte row
//               segment; neighbour indices arrive through a cp.async ring one offset ahead), optionally apply
//               the fused BatchNorm affine + activation of the producing layer, split fp32 → bf16 hi (+ lo), and
//               store the 128x64 tile into shared memory in the 128-byte-swizzled K-major layout.  Loads of
//               slot s+1 are in flight in registers while slot s is converted and stored.
//   warps 8-15  two consumer warpgroups: warpgroup g issues wgmma (M=64 rows [64 g, 64 g + 64), N=128, 64 or 16, K=16)
//               into register accumulators, then adds the bias and stores its fp32 rows.
//   warp  16    streams the pre-swizzled weight slices with bulk async copies into their own ring (warps 17-19 only
//               complete its warpgroup, whose registers go to the gather and consumer warpgroups).
// No atomics: every output row is written exactly once, results are run-to-run deterministic.
//
// precision 3 (the "fp32" mode): operands split as x = hi + lo (bf16 each) and three MMAs
// hi·hi + lo·hi + hi·lo accumulate in fp32 — ~2^-16 relative error, well inside the 1e-3 parity bound.
#include "common.cuh"
#include "gmma.cuh"
#include <cstdlib>

using namespace pasco;
using namespace gmma;

namespace {

constexpr int BLOCK_M = 128;
constexpr int KBLK = 64;                    // channels per K-block (= one 128-byte swizzle row of bf16)
constexpr int A_TILE_BYTES = BLOCK_M * 128; // 16 KB
constexpr int NUM_GATHER_WARPS = 8;                             // 16 tile rows each
constexpr int NUM_CONS_WARPS = 8;                               // two consumer warpgroups
constexpr int CONS_WARP0 = NUM_GATHER_WARPS;                    // warpgroup-aligned (a multiple of 4)
constexpr int LOAD_WARP = CONS_WARP0 + NUM_CONS_WARPS;          // first warp of the last warpgroup; its 3 others idle
constexpr int NUM_THREADS = (LOAD_WARP + 4) * 32;              // 640 = 5 warpgroups (96 registers each at launch)
// setmaxnreg budgets (640 x 96 at launch): the loader warpgroup keeps 24 and the registers it releases go to the gather
// and consumer warpgroups, 2 x 128 x (gather - 96) + 2 x 128 x (consumer - 96) <= 128 x (96 - 24).  The register-gather
// producers (k_conv_tc) hold two slots of loads and spill at 112, so they get 120 and the consumers 104; the plane-gather
// producers (k_conv_pl) only issue copies, so there the consumers get 120.  With these budgets ptxas reports no spills.
constexpr int LOAD_REGS = 24;
constexpr int TC_GATHER_REGS = 120, TC_CONS_REGS = 104;
constexpr int PL_GATHER_REGS = 104, PL_CONS_REGS = 120;
static_assert(2 * 128 * (TC_GATHER_REGS - 96) + 2 * 128 * (TC_CONS_REGS - 96) <= 128 * (96 - LOAD_REGS), "setmaxnreg budget");
static_assert(2 * 128 * (PL_GATHER_REGS - 96) + 2 * 128 * (PL_CONS_REGS - 96) <= 128 * (96 - LOAD_REGS), "setmaxnreg budget");
constexpr int ROWS_PER_WARP = BLOCK_M / NUM_GATHER_WARPS;       // 16
constexpr int LOADS_PER_SLOT = ROWS_PER_WARP / 2;               // float4 per lane per slot
constexpr int TILES_PER_IDX_STEP = 32 / ROWS_PER_WARP;          // tiles whose indices one warp-wide cp.async covers
constexpr int MAX_STAGES = 8;
constexpr int ACC_COLS = 128;               // accumulator columns per consumer warpgroup (64 fp32 registers per thread)

struct ConvParams {
  const float* in;
  const int32_t* nbr;  // [K, n_out] or nullptr (identity)
  const uint8_t* wpk;  // packed weights
  const float* bias;
  const float* in_scale;
  const float* in_shift;
  float* out;
  double* stats;       // optional [2*Cout]: column sums / sums of squares of `out` accumulate here (fused BN statistics)
  int64_t n_out;
  int64_t out_pitch;   // row stride of out (floats)
  int64_t in_pitch;    // row stride of in (floats)
  int K, Cin, Cout, in_act;
  int sa, sb, tiles_per_group;
  int nsplit, ncols;          // output columns in ranges of ncols (the last one may be narrower), one work item each
  int koff_base, koff_step;   // weight slice of table row k = koff_base + koff_step * k
  int ksplit, kchunk;         // split-K: offset range ks covers [ks*kchunk, (ks+1)*kchunk); partial results go to
                              // out + ks * n_out * out_pitch (summed by k_splitk_reduce)
  // k_conv_pl only: the input as pre-split bf16 planes x = hi + lo, [n_in, Cin] each with row pitch pl_pitch (elements)
  const uint16_t* pl_hi;
  const uint16_t* pl_lo;
  int64_t pl_pitch;
};

// ------------------------------------------------------------------------------------------------------------
// weight packing: fp32 [K, Cin, Cout] → per (k, kb): [hi image | lo image], image = N rows x 128 B, swizzled
// ------------------------------------------------------------------------------------------------------------
__global__ void k_pack_weights(const float* __restrict__ W, int K, int Cin, int Cout, int transpose,
                               uint8_t* __restrict__ packed) {
  const int N = transpose ? Cin : Cout;   // B rows
  const int Kc = transpose ? Cout : Cin;  // contraction length
  const int KB = Kc / KBLK;
  int64_t total = (int64_t)K * KB * N * 8;  // one thread per 16-byte chunk (8 bf16)
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    int c = (int)(t & 7);
    int64_t r = t >> 3;
    int n = (int)(r % N);
    r /= N;
    int kb = (int)(r % KB);
    int k = (int)(r / KB);
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      int kc = kb * KBLK + c * 8 + j;
      v[j] = transpose ? __ldg(W + ((int64_t)k * Cin + n) * Cout + kc) : __ldg(W + ((int64_t)k * Cin + kc) * Cout + n);
    }
    uint4 hi, lo;
    uint2 h0, l0, h1, l1;
    split4(make_float4(v[0], v[1], v[2], v[3]), h0, l0);
    split4(make_float4(v[4], v[5], v[6], v[7]), h1, l1);
    hi = make_uint4(h0.x, h0.y, h1.x, h1.y);
    lo = make_uint4(l0.x, l0.y, l1.x, l1.y);
    int64_t tile = ((int64_t)k * KB + kb) * (int64_t)N * 256;  // hi image then lo image
    int64_t off = (int64_t)n * 128 + ((c ^ (n & 7)) << 4);
    *reinterpret_cast<uint4*>(packed + tile + off) = hi;
    *reinterpret_cast<uint4*>(packed + tile + (int64_t)N * 128 + off) = lo;
  }
}

// ------------------------------------------------------------------------------------------------------------
// forward / dgrad kernel
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float act_apply(float z, int act) {
  if (act == 1) return fmaxf(z, 0.f);
  if (act == 2) return z > 0.f ? z : 0.01f * z;
  return z;
}

// ------------------------------------------------------------------------------------------------------------
// cp.async helpers for the neighbour-index ring
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void cp_async4(uint32_t dst_smem, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst_smem), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

constexpr int IDX_RING = 6;  // neighbour-index ring depth (entries of T*128 ints, one per (tile group, offset))

// position of a gather warp inside the flat slot sequence  group → k → kb → t
struct SlotIt {
  int64_t v;       // work item handled by this CTA
  int64_t group;   // = item_group(v)
  int gk;          // running (work item, k) counter → index ring slot
  int k, k1, kb, t;  // k walks [k0(v), k1(v))
  int t_eff;       // tiles in this group
  bool valid;
};

// ------------------------------------------------------------------------------------------------------------
// consumer-side roles shared by the register-gather kernel (k_conv_tc) and the plane-gather kernel (k_conv_pl)
// ------------------------------------------------------------------------------------------------------------
struct Pipe {
  uint8_t* a_smem;          // [sa][A_hi | A_lo]
  uint8_t* b_smem;          // [sb][B_hi | B_lo]
  uint64_t *afull, *aempty, *bfull, *bempty;
  double* stat_acc;         // [2*Cout] per-CTA accumulators in shared memory (nullptr: no fused statistics)
  int a_stage_bytes, b_tile;
  int KB, T;
  int64_t num_tiles, num_groups, num_items;
};

// work item v = (tile group, offset range, column range): columns vary fastest, then offset ranges
__device__ __forceinline__ int64_t item_group(const ConvParams& p, int64_t v) { return v / ((int64_t)p.ksplit * p.nsplit); }
__device__ __forceinline__ int item_ks(const ConvParams& p, int64_t v) { return (int)((v / p.nsplit) % p.ksplit); }
__device__ __forceinline__ int item_n0(const ConvParams& p, int64_t v) { return (int)(v % p.nsplit) * p.ncols; }
__device__ __forceinline__ int item_ncols(const ConvParams& p, int64_t v) {
  const int n0 = item_n0(p, v);
  return p.Cout - n0 < p.ncols ? p.Cout - n0 : p.ncols;
}

// one thread: streams the pre-swizzled weight slices (the item's column range of the hi [and lo] image) with bulk async
// copies into the B ring
__device__ __forceinline__ void role_weight_loader(const ConvParams& p, const Pipe& pl, int n_op) {
  int stage = 0;
  uint32_t phase = 0;
  for (int64_t v = blockIdx.x; v < pl.num_items; v += gridDim.x) {
    const int k0 = item_ks(p, v) * p.kchunk, k1 = k0 + p.kchunk < p.K ? k0 + p.kchunk : p.K;
    const int n0 = item_n0(p, v);
    const uint32_t bytes = (uint32_t)item_ncols(p, v) * 128u;
    for (int k = k0; k < k1; ++k) {
      for (int kb = 0; kb < pl.KB; ++kb) {
        mbar_wait(smem_u32(pl.bempty + stage), phase ^ 1);
        mbar_arrive_expect_tx(smem_u32(pl.bfull + stage), bytes * n_op);
        const uint8_t* src = p.wpk + ((int64_t)(p.koff_base + p.koff_step * k) * pl.KB + kb) * (int64_t)p.Cout * 256 + n0 * 128;
        const uint32_t dst = smem_u32(pl.b_smem + (size_t)stage * n_op * pl.b_tile);
        bulk_g2s(dst, src, bytes, smem_u32(pl.bfull + stage));
        if (n_op == 2) bulk_g2s(dst + pl.b_tile, src + (int64_t)p.Cout * 128, bytes, smem_u32(pl.bfull + stage));
        if (++stage == p.sb) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
  }
}

// Consumer warpgroup g (0 or 1) owns rows [64 g, 64 g + 64) of every tile of a group: it issues wgmma
// (M = 64, N = CH per instruction, K = 16) over the A and B rings into register accumulators, then stores the finished
// rows itself.  acc[c] holds accumulator columns [c CH, c CH + CH); the group's T tiles sit side by side, tile t in
// columns [t ncols, (t + 1) ncols).  Every consumer warp arrives on the ring "empty" barriers (expected count 8), so a
// stage is refilled only after both warpgroups' MMAs on it have completed.
// Retire: one wgmma group stays in flight.  After committing slot n the warpgroup waits for all but the newest group
// (wait_group 1), i.e. for slot n - 1, and only then releases slot n - 1's A stage (and its B stage after the B stage's
// last tile), so the MMAs of consecutive slots overlap.  The ring needs sa >= 3 for a slot to be filled ahead of the
// one being multiplied and the one held back.  The item's last slot is drained (wait_group 0) before the epilogue.
// The epilogue adds the bias, stores fp32 rows and optionally accumulates the per-channel sum and sum of squares of
// what was stored (the BatchNorm statistics of the next layer): per warp over its rows with shuffles, then in fp64 in
// shared memory, one global fp64 atomic per channel and CTA.
template <int NSPLIT, bool CPASYNC_A, int CH>
__device__ __forceinline__ void role_consumer(const ConvParams& p, const Pipe& pl, int g, int wq, int lane) {
  constexpr int NCH = ACC_COLS / CH;
  float acc[NCH][CH / 2];
  const bool want_stats = pl.stat_acc != nullptr;
  int sa = 0, sb = 0;
  uint32_t pa = 0, pb = 0;
  int held_a = -1, held_b = -1;     // stages of the slot whose MMAs may still be in flight (-1: none)
  auto release_held = [&]() {
    __syncwarp();
    if (lane == 0) {
      if (held_a >= 0) mbar_arrive(smem_u32(pl.aempty + held_a));
      if (held_b >= 0) mbar_arrive(smem_u32(pl.bempty + held_b));
    }
    held_a = held_b = -1;
  };
  for (int64_t v = blockIdx.x; v < pl.num_items; v += gridDim.x) {
    const int64_t group = item_group(p, v);
    const int k0 = item_ks(p, v) * p.kchunk, k1 = k0 + p.kchunk < p.K ? k0 + p.kchunk : p.K;
    const int ncols = item_ncols(p, v);
#pragma unroll
    for (int c = 0; c < NCH; ++c)
#pragma unroll
      for (int i = 0; i < CH / 2; ++i) acc[c][i] = 0.f;
    for (int k = k0; k < k1; ++k) {
      for (int kb = 0; kb < pl.KB; ++kb) {
        mbar_wait(smem_u32(pl.bfull + sb), pb);
        const uint32_t b_hi = smem_u32(pl.b_smem + (size_t)sb * (NSPLIT == 3 ? 2 : 1) * pl.b_tile), b_lo = b_hi + pl.b_tile;
        for (int t = 0; t < pl.T; ++t) {     // the last group is padded to T tiles (rows >= n_out: never gathered, never stored)
          mbar_wait(smem_u32(pl.afull + sa), pa);
          if (CPASYNC_A) fence_proxy_async_smem();   // the A stage was written by cp.async copies (generic proxy)
          const uint32_t a_hi = smem_u32(pl.a_smem + (size_t)sa * pl.a_stage_bytes) + (uint32_t)g * (64 * 128), a_lo = a_hi + A_TILE_BYTES;
          const uint64_t da_hi = make_desc_sw128(a_hi, 16, 1024), da_lo = make_desc_sw128(a_lo, 16, 1024);
          // one chunk's k-steps (3 products each in bf16x3 mode) into acc[c], B columns from `col` of the weight slice
          auto mma_chunk = [&](float (&a)[CH / 2], int col) {
            const uint64_t db_hi = make_desc_sw128(b_hi + (uint32_t)col * 128u, 16, 1024);
            const uint64_t db_lo = make_desc_sw128(b_lo + (uint32_t)col * 128u, 16, 1024);
#pragma unroll
            for (int j = 0; j < KBLK / 16; ++j) {   // the start-address field (16-byte units) advances by 2 per 32 bytes
              if constexpr (CH == 128) {
                wgmma_n128<0, 0>(a, da_hi + 2 * j, db_hi + 2 * j);
                if (NSPLIT == 3) {
                  wgmma_n128<0, 0>(a, da_lo + 2 * j, db_hi + 2 * j);
                  wgmma_n128<0, 0>(a, da_hi + 2 * j, db_lo + 2 * j);
                }
              } else if constexpr (CH == 64) {
                wgmma_n64<0, 0>(a, da_hi + 2 * j, db_hi + 2 * j);
                if (NSPLIT == 3) {
                  wgmma_n64<0, 0>(a, da_lo + 2 * j, db_hi + 2 * j);
                  wgmma_n64<0, 0>(a, da_hi + 2 * j, db_lo + 2 * j);
                }
              } else {
                wgmma_n16(a, da_hi + 2 * j, db_hi + 2 * j);
                if (NSPLIT == 3) {
                  wgmma_n16(a, da_lo + 2 * j, db_hi + 2 * j);
                  wgmma_n16(a, da_hi + 2 * j, db_lo + 2 * j);
                }
              }
            }
          };
          wg_fence();
          if constexpr (CH == 128) {
            // column ranges of exactly 128 (C_out % 128 == 0): T = 1 and the tile fills chunk 0, so the slot's MMAs and
            // its commit are one basic block
            mma_chunk(acc[0], 0);
            wg_commit();
          } else {
            // the tile's chunks: each chain is committed inside its own branch
#pragma unroll
            for (int c = 0; c < NCH; ++c) {
              const int col = c * CH - t * p.ncols;     // chunk column inside tile t
              if (col >= 0 && col < ncols) {
                mma_chunk(acc[c], col);
                wg_commit();
              }
            }
          }
          wg_wait<1>();                        // the previous slot's MMAs are complete
          release_held();
          held_a = sa;
          held_b = t == pl.T - 1 ? sb : -1;    // the B stage is free after its last tile's MMAs
          if (++sa == p.sa) {
            sa = 0;
            pa ^= 1;
          }
        }
        if (++sb == p.sb) {
          sb = 0;
          pb ^= 1;
        }
      }
    }
    wg_wait<0>();
    release_held();
    // ---- epilogue ----
    float* out_part = p.out + item_ks(p, v) * p.n_out * p.out_pitch;    // this split's partial output
    const int n0 = item_n0(p, v);
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const int t = (c * CH) / p.ncols, col0 = c * CH - t * p.ncols;
      if (t >= pl.T || col0 >= ncols) continue;
      const int64_t rbase = (group * pl.T + t) * BLOCK_M + g * 64;
#pragma unroll
      for (int i4 = 0; i4 < CH / 8; ++i4) {
        const int col = n0 + col0 + frag_col(i4 * 4, lane);
        float2 b = make_float2(0.f, 0.f);
        if (p.bias) b = __ldg(reinterpret_cast<const float2*>(p.bias + col));
        float s1[2] = {0.f, 0.f}, s2[2] = {0.f, 0.f};
#pragma unroll
        for (int h = 0; h < 2; ++h) {              // rows r and r + 8
          const int64_t row = rbase + frag_row(i4 * 4 + 2 * h, wq, lane);
          const float v0 = acc[c][i4 * 4 + 2 * h] + b.x, v1 = acc[c][i4 * 4 + 2 * h + 1] + b.y;
          if (row < p.n_out) {
            *reinterpret_cast<float2*>(out_part + row * p.out_pitch + col) = make_float2(v0, v1);
            s1[0] += v0; s1[1] += v1;
            s2[0] += v0 * v0; s2[1] += v1 * v1;
          }
        }
        if (want_stats) {
#pragma unroll
          for (int w = 4; w < 32; w <<= 1) {        // lanes with the same (lane & 3) hold the same columns
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              s1[e] += __shfl_xor_sync(0xffffffffu, s1[e], w);
              s2[e] += __shfl_xor_sync(0xffffffffu, s2[e], w);
            }
          }
          if (lane < 4) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              atomicAdd(pl.stat_acc + col + e, (double)s1[e]);
              atomicAdd(pl.stat_acc + p.Cout + col + e, (double)s2[e]);
            }
          }
        }
      }
    }
  }
  if (want_stats) {
    named_sync(1, NUM_CONS_WARPS * 32);   // the consumer warps
    const int ct = g * 128 + wq * 32 + lane;
    for (int i = ct; i < 2 * p.Cout; i += NUM_CONS_WARPS * 32) atomicAdd(p.stats + i, pl.stat_acc[i]);
  }
}

// the consumer role of warp `warp` (CONS_WARP0 <= warp < LOAD_WARP), dispatched on the chunk width
template <int NSPLIT, bool CPASYNC_A>
__device__ __forceinline__ void run_consumer(const ConvParams& p, const Pipe& pl, int warp, int lane) {
  const int g = (warp - CONS_WARP0) >> 2, wq = (warp - CONS_WARP0) & 3;
  if (p.Cout % 128 == 0) role_consumer<NSPLIT, CPASYNC_A, 128>(p, pl, g, wq, lane);   // column ranges of exactly 128
  else if (p.Cout % 64 == 0) role_consumer<NSPLIT, CPASYNC_A, 64>(p, pl, g, wq, lane);
  else role_consumer<NSPLIT, CPASYNC_A, 16>(p, pl, g, wq, lane);
}

template <int NSPLIT, bool PROLOGUE>
__global__ void __launch_bounds__(NUM_THREADS, 1) k_conv_tc(const __grid_constant__ ConvParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  constexpr int n_op = (NSPLIT == 3) ? 2 : 1;
  const int b_tile = p.ncols * 128;
  const int a_stage_bytes = n_op * A_TILE_BYTES;
  const int b_stage_bytes = n_op * b_tile;
  const int T = p.tiles_per_group;
  uint8_t* a_smem = smem;                                           // [sa][A_hi | A_lo]
  uint8_t* b_smem = smem + (size_t)p.sa * a_stage_bytes;            // [sb][B_hi | B_lo]
  int* idx_ring = reinterpret_cast<int*>(b_smem + (size_t)p.sb * b_stage_bytes);   // [IDX_RING][T*128]
  uint64_t* bars = reinterpret_cast<uint64_t*>(idx_ring + IDX_RING * T * BLOCK_M);
  uint64_t* afull = bars;                         // [MAX_STAGES]
  uint64_t* aempty = bars + MAX_STAGES;           // [MAX_STAGES]
  uint64_t* bfull = bars + 2 * MAX_STAGES;        // [MAX_STAGES]
  uint64_t* bempty = bars + 3 * MAX_STAGES;       // [MAX_STAGES]
  double* stat_acc = p.stats ? reinterpret_cast<double*>(bars + 4 * MAX_STAGES) : nullptr;   // [2*Cout]

  const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x, 0) >> 5, lane = threadIdx.x & 31;   // provably warp-uniform, else ptxas serializes the wgmma
  const int KB = p.Cin / KBLK;
  const int64_t num_tiles = (p.n_out + BLOCK_M - 1) / BLOCK_M;
  const int64_t num_groups = (num_tiles + T - 1) / T;

  if (stat_acc)
    for (int i = threadIdx.x; i < 2 * p.Cout; i += NUM_THREADS) stat_acc[i] = 0.0;
  if (threadIdx.x == 0) {
    for (int s = 0; s < MAX_STAGES; ++s) {
      mbar_init(smem_u32(afull + s), NUM_GATHER_WARPS);
      mbar_init(smem_u32(aempty + s), NUM_CONS_WARPS);
      mbar_init(smem_u32(bfull + s), 1);
      mbar_init(smem_u32(bempty + s), NUM_CONS_WARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();
  Pipe pl;
  pl.a_smem = a_smem; pl.b_smem = b_smem;
  pl.afull = afull; pl.aempty = aempty; pl.bfull = bfull; pl.bempty = bempty;
  pl.stat_acc = stat_acc;
  pl.a_stage_bytes = a_stage_bytes; pl.b_tile = b_tile;
  pl.KB = KB; pl.T = T; pl.num_tiles = num_tiles; pl.num_groups = num_groups;
  pl.num_items = num_groups * p.ksplit * p.nsplit;

  if (warp < NUM_GATHER_WARPS) {
    reg_alloc<TC_GATHER_REGS>();
    // ===================================== gather producers =====================================
    const int chunk = lane & 15;  // 16-byte fp32 chunk inside the 64-channel block
    const int rsub = lane >> 4;   // which of the 2 rows this half-warp handles per step
    const bool affine = PROLOGUE && p.in_scale != nullptr;

    // async prefetch of the neighbour indices of (group, k) into ring slot gk % IDX_RING: this warp's 32 rows of
    // each of the group's tiles
    auto prefetch_idx = [&](int64_t group, int k, int gk, int t_eff) {
      int* dst = idx_ring + (gk % IDX_RING) * T * BLOCK_M;
      // lanes 0-15 fetch tile t, lanes 16-31 tile t+1: the warp's 16 rows of each
      for (int t = lane / ROWS_PER_WARP; t < t_eff; t += TILES_PER_IDX_STEP) {
        const int64_t row = (group * T + t) * BLOCK_M + warp * ROWS_PER_WARP + (lane % ROWS_PER_WARP);
        int* d = dst + t * BLOCK_M + warp * ROWS_PER_WARP + (lane % ROWS_PER_WARP);
        if (row < p.n_out) {
          if (p.nbr) cp_async4(smem_u32(d), p.nbr + (int64_t)k * p.n_out + row);
          else *d = (int)row;
        } else {
          *d = -1;
        }
      }
      cp_async_commit();
    };
    const int64_t num_items = pl.num_items;
    // position `it` at the first offset of work item v
    auto enter = [&](SlotIt& it, int64_t v) {
      it.v = v;
      it.valid = v < num_items;
      if (it.valid) {
        it.group = item_group(p, v);
        it.k = item_ks(p, v) * p.kchunk;
        it.k1 = it.k + p.kchunk < p.K ? it.k + p.kchunk : p.K;
        it.t_eff = T;              // padded to T tiles (see role_consumer)
      }
    };
    auto advance = [&](SlotIt& it) {
      if (++it.t < it.t_eff) return;
      it.t = 0;
      if (++it.kb < KB) return;
      it.kb = 0;
      ++it.gk;
      if (++it.k < it.k1) return;
      enter(it, it.v + gridDim.x);
    };
    // the (work item, k) pair that follows `it`'s by `ahead` steps, for index prefetch
    auto prefetch_ahead = [&](const SlotIt& it, int ahead) {
      int64_t v = it.v;
      int k = it.k + ahead, k1 = it.k1;
      const int gk = it.gk + ahead;
      while (v < num_items && k >= k1) {
        const int over = k - k1;
        v += gridDim.x;
        if (v >= num_items) break;
        const int k0 = item_ks(p, v) * p.kchunk;
        k1 = k0 + p.kchunk < p.K ? k0 + p.kchunk : p.K;
        k = k0 + over;
      }
      if (v < num_items) {
        const int64_t g = item_group(p, v);
        prefetch_idx(g, k, gk, T);
      } else {
        cp_async_commit();  // keep the group count uniform
      }
    };

    SlotIt ld;
    ld.gk = 0; ld.kb = 0; ld.t = 0; ld.group = 0; ld.k = 0; ld.k1 = 0; ld.t_eff = 0;
    enter(ld, blockIdx.x);
    if (ld.valid) {
      // prime the index ring: entries 0 .. IDX_RING-2
      for (int a = 0; a < IDX_RING - 1; ++a) prefetch_ahead(ld, a);
    }
    SlotIt st = ld;
    int stage = 0;
    uint32_t phase = 0;

    float4 va[LOADS_PER_SLOT], vb[LOADS_PER_SLOT];
    uint32_t valid_a = 0, valid_b = 0;

    // issue the 16 row-segment loads of one slot into registers
    auto issue = [&](SlotIt& it, float4 (&v)[LOADS_PER_SLOT], uint32_t& valid) {
      if (it.kb == 0 && it.t == 0) {
        // first use of ring entry gk: it was prefetched IDX_RING-1 entries ago; keep the ring primed
        cp_async_wait<IDX_RING - 2>();
        __syncwarp();
        prefetch_ahead(it, IDX_RING - 1);
      }
      const int* irow = idx_ring + (it.gk % IDX_RING) * T * BLOCK_M + it.t * BLOCK_M + warp * ROWS_PER_WARP;
      const int cbase = it.kb * KBLK + chunk * 4;
      valid = 0;
      int srcs[LOADS_PER_SLOT];
#pragma unroll
      for (int i = 0; i < LOADS_PER_SLOT; ++i) srcs[i] = irow[i * 2 + rsub];
#pragma unroll
      for (int i = 0; i < LOADS_PER_SLOT; ++i) {
        v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (srcs[i] >= 0) {
          v[i] = __ldg(reinterpret_cast<const float4*>(p.in + (int64_t)srcs[i] * p.in_pitch + cbase));
          valid |= 1u << i;
        }
      }
    };
    // convert + store one slot into its A stage and publish it
    auto store = [&](const SlotIt& it, float4 (&v)[LOADS_PER_SLOT], uint32_t valid) {
      mbar_wait(smem_u32(aempty + stage), phase ^ 1);
      uint8_t* dst = a_smem + (size_t)stage * a_stage_bytes;
      float4 sc = make_float4(1.f, 1.f, 1.f, 1.f), sh = make_float4(0.f, 0.f, 0.f, 0.f);
      if (PROLOGUE && affine) {
        const int cbase = it.kb * KBLK + chunk * 4;
        sc = __ldg(reinterpret_cast<const float4*>(p.in_scale + cbase));
        sh = __ldg(reinterpret_cast<const float4*>(p.in_shift + cbase));
      }
      // byte offset of (row warp*16 + rsub, 16-byte chunk) inside the swizzled tile; row i*2 adds i*256 and flips
      // the chunk by (i*2 & 7)
      const uint32_t row_base = (uint32_t)(warp * ROWS_PER_WARP + rsub);
#pragma unroll
      for (int i = 0; i < LOADS_PER_SLOT; ++i) {
        float4 x = v[i];
        if (PROLOGUE && ((valid >> i) & 1u)) {
          x.x = act_apply(fmaf(x.x, sc.x, sh.x), p.in_act);
          x.y = act_apply(fmaf(x.y, sc.y, sh.y), p.in_act);
          x.z = act_apply(fmaf(x.z, sc.z, sh.z), p.in_act);
          x.w = act_apply(fmaf(x.w, sc.w, sh.w), p.in_act);
        }
        const uint32_t trow = row_base + i * 2;
        const uint32_t off = trow * 128u + ((((uint32_t)chunk >> 1) ^ (trow & 7u)) << 4) + (((uint32_t)chunk & 1u) << 3);
        if (NSPLIT == 3) {
          uint2 hi, lo;
          split4(x, hi, lo);
          *reinterpret_cast<uint2*>(dst + off) = hi;
          *reinterpret_cast<uint2*>(dst + A_TILE_BYTES + off) = lo;
        } else {
          *reinterpret_cast<uint2*>(dst + off) = to_bf16x4(x);
        }
      }
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(afull + stage));
      if (++stage == p.sa) {
        stage = 0;
        phase ^= 1;
      }
    };

    if (ld.valid) {
      issue(ld, va, valid_a);
      advance(ld);
      while (st.valid) {
        if (ld.valid) {
          issue(ld, vb, valid_b);
          advance(ld);
        }
        store(st, va, valid_a);
        advance(st);
        if (!st.valid) break;
        if (ld.valid) {
          issue(ld, va, valid_a);
          advance(ld);
        }
        store(st, vb, valid_b);
        advance(st);
      }
    }
    cp_async_wait<0>();
  } else if (warp >= LOAD_WARP) {
    reg_dealloc<LOAD_REGS>();
    if (warp == LOAD_WARP && lane == 0) role_weight_loader(p, pl, n_op);
  } else {
    reg_alloc<TC_CONS_REGS>();
    run_consumer<NSPLIT, false>(p, pl, warp, lane);
  }
}

// ------------------------------------------------------------------------------------------------------------
// Plane-gather variant: the input arrives PRE-SPLIT as bf16 planes (hi [+ lo]) and the producers only move bytes
// ------------------------------------------------------------------------------------------------------------
// In k_conv_tc every gathered fp32 value crosses the register file and is converted once per kernel offset.  Here the
// split x = hi + lo is done ONCE per tensor by the producing pass (k_split_planes / the BatchNorm apply), and a gather
// warp issues 16-byte cp.async (LDGSTS) copies straight from the plane rows into the 128-byte-swizzled operand tile:
//   * no registers on the data path, so whole A stages (32 KB each in fp32 mode) are in flight per SM;
//   * a missing neighbour is a ZERO-FILL copy (src-size 0): no global or L2 traffic for (row, offset) pairs that have
//     no neighbour;
//   * 8 copies per lane per slot instead of ~600 gather/convert/store instructions.
// Completion is tracked by the hardware: after issuing the copies of a slot every lane of the filling warp executes
// cp.async.mbarrier.arrive.noinc on the slot's "full" barrier (expected count = 32), so the barrier completes when the
// last copy has landed — no wait_group, no software publish step, and the producers run up to `sa` slots ahead of the
// MMA.  The consumers add a generic→async proxy fence after their barrier wait.
__device__ __forceinline__ void cp_async16_zfill(uint32_t dst_smem, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst_smem), "l"(src), "r"(src_bytes) : "memory");
}
// the mbarrier receives one arrival from this thread once all its cp.async copies issued so far have completed
__device__ __forceinline__ void cp_async_mbar_arrive_noinc(uint32_t bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
}

template <int NSPLIT>
__global__ void __launch_bounds__(NUM_THREADS, 1) k_conv_pl(const __grid_constant__ ConvParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  constexpr int n_op = (NSPLIT == 3) ? 2 : 1;
  const int b_tile = p.ncols * 128;
  const int a_stage_bytes = n_op * A_TILE_BYTES;
  const int b_stage_bytes = n_op * b_tile;
  const int T = p.tiles_per_group;
  uint8_t* a_smem = smem;                                           // [sa][A_hi | A_lo]
  uint8_t* b_smem = smem + (size_t)p.sa * a_stage_bytes;            // [sb][B_hi | B_lo]
  uint64_t* bars = reinterpret_cast<uint64_t*>(b_smem + (size_t)p.sb * b_stage_bytes);
  uint64_t* afull = bars;                         // [MAX_STAGES]
  uint64_t* aempty = bars + MAX_STAGES;           // [MAX_STAGES]
  uint64_t* bfull = bars + 2 * MAX_STAGES;        // [MAX_STAGES]
  uint64_t* bempty = bars + 3 * MAX_STAGES;       // [MAX_STAGES]
  double* stat_acc = p.stats ? reinterpret_cast<double*>(bars + 4 * MAX_STAGES) : nullptr;   // [2*Cout]

  const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x, 0) >> 5, lane = threadIdx.x & 31;   // provably warp-uniform, else ptxas serializes the wgmma
  const int KB = p.Cin / KBLK;
  const int64_t num_tiles = (p.n_out + BLOCK_M - 1) / BLOCK_M;
  const int64_t num_groups = (num_tiles + T - 1) / T;

  if (stat_acc)
    for (int i = threadIdx.x; i < 2 * p.Cout; i += NUM_THREADS) stat_acc[i] = 0.0;
  if (threadIdx.x == 0) {
    for (int s = 0; s < MAX_STAGES; ++s) {
      mbar_init(smem_u32(afull + s), 32);   // one cp.async arrival per lane of the warp that fills the slot
      mbar_init(smem_u32(aempty + s), NUM_CONS_WARPS);
      mbar_init(smem_u32(bfull + s), 1);
      mbar_init(smem_u32(bempty + s), NUM_CONS_WARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();
  Pipe pl;
  pl.a_smem = a_smem; pl.b_smem = b_smem;
  pl.afull = afull; pl.aempty = aempty; pl.bfull = bfull; pl.bempty = bempty;
  pl.stat_acc = stat_acc;
  pl.a_stage_bytes = a_stage_bytes; pl.b_tile = b_tile;
  pl.KB = KB; pl.T = T; pl.num_tiles = num_tiles; pl.num_groups = num_groups;
  pl.num_items = num_groups * p.ksplit * p.nsplit;

  if (warp < NUM_GATHER_WARPS) {
    reg_alloc<PL_GATHER_REGS>();
    // ===================================== plane-gather producers =====================================
    // ONE WARP PER SLOT: warp w fills the slots n ≡ w (mod 8) of the CTA's slot sequence (work item → k → kb → tile),
    // all 128 rows of the tile.  (A first version let every warp fill 16 rows of EVERY slot: ncu showed ~300
    // instructions of per-slot bookkeeping per warp for 8 copies, 900 cycles per slot against 384 cycles of MMA.)
    // One copy instruction moves 4 rows: lane = (row sub-index 0..3, 16-byte chunk 0..7 of the 128-byte row); 32
    // instructions per plane per slot.  Lane l holds the neighbour indices of rows l, l+32, l+64, l+96 (four coalesced
    // 128-byte loads, fetched two of the warp's slots = 16 CTA slots ahead), distributed by one shuffle per instruction.
    const int ch = lane & 7, sub = lane >> 3;
    const int64_t num_items = pl.num_items;
    struct It {
      int64_t v, group;
      int k, k1, kb, t, t_eff;
      bool valid;
    };
    auto enter = [&](It& it, int64_t v) {
      it.v = v;
      it.valid = v < num_items;
      it.kb = 0; it.t = 0;
      if (it.valid) {
        it.group = item_group(p, v);
        it.k = item_ks(p, v) * p.kchunk;
        it.k1 = it.k + p.kchunk < p.K ? it.k + p.kchunk : p.K;
        it.t_eff = T;              // padded to T tiles (see role_consumer)
      }
    };
    auto advance = [&](It& it) {
      if (++it.t < it.t_eff) return;
      it.t = 0;
      if (++it.kb < KB) return;
      it.kb = 0;
      if (++it.k < it.k1) return;
      enter(it, it.v + gridDim.x);
    };
    auto advance_n = [&](It& it, int n) {
      for (int i = 0; i < n && it.valid; ++i) advance(it);
    };
    struct Idx4 { int v[4]; };
    auto load_idx = [&](const It& it) -> Idx4 {
      Idx4 r;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        r.v[j] = -1;
        if (it.valid) {
          const int64_t row = (it.group * T + it.t) * BLOCK_M + j * 32 + lane;
          if (row < p.n_out) r.v[j] = p.nbr ? __ldg(p.nbr + (int64_t)it.k * p.n_out + row) : (int)row;
        }
      }
      return r;
    };
    // Ownership: W = min(8, sa) producer warps are active and warp w fills the slots n = w, w + W, w + 2W, ...  A warp
    // waits only on the "empty" barriers of its own slots; the parity wait is sound because its previous wait (slot
    // n - W) already required slot n - W - sa >= n - 2 sa to be consumed (W <= sa), so it is never two ring revolutions
    // ahead of the barrier, and it cannot be behind it either (the next completion needs this very slot filled).
    // (Two earlier variants deadlocked: a stride of 8 with a ring of 6 lets a warp run two revolutions ahead; letting
    // every warp observe every slot's barrier fails the other way round — a slow observer falls a revolution BEHIND
    // and then waits for a completion that depends on its own slot.  tools/pipeline_sim.py replays both.)
    const int W = NUM_GATHER_WARPS < p.sa ? NUM_GATHER_WARPS : p.sa;
    It it0, it1, it2;
    enter(it0, blockIdx.x);
    if (warp >= W) it0.valid = false;
    advance_n(it0, warp);
    it1 = it0;
    advance_n(it1, W);
    it2 = it1;
    advance_n(it2, W);
    Idx4 q0 = load_idx(it0), q1 = load_idx(it1);
    const uint8_t* base_hi = reinterpret_cast<const uint8_t*>(p.pl_hi);
    const uint8_t* base_lo = reinterpret_cast<const uint8_t*>(p.pl_lo);
    const int64_t pitch_b = p.pl_pitch * 2;
    int stage = warp;                               // ring position of this warp's current slot (warp < W <= sa)
    uint32_t phase = 0;
    auto observe = [&]() {                          // wait until the slot's stage is free
      mbar_wait(smem_u32(aempty + stage), phase ^ 1);
    };
    auto next_stage = [&]() {                       // this warp's next slot is W slots on (at most one wrap: W <= sa)
      stage += W;
      if (stage >= p.sa) {
        stage -= p.sa;
        phase ^= 1;
      }
    };
    while (it0.valid) {
      const Idx4 q2 = load_idx(it2);                // indices of this warp's slot after next
      observe();
      const uint32_t dst0 = smem_u32(a_smem + (size_t)stage * a_stage_bytes) + (uint32_t)sub * 128u;
      const int64_t coff_b = ((int64_t)it0.kb * KBLK + ch * 8) * 2;
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        // tile row r = 4i + sub; its index lives in register (i / 8) of lane (4 (i % 8) + sub)
        const int idx = __shfl_sync(0xffffffffu, q0.v[i >> 3], ((i & 7) << 2) + sub);
        const uint32_t nbytes = idx >= 0 ? 16u : 0u;
        const int64_t boff = (int64_t)(idx >= 0 ? idx : 0) * pitch_b + coff_b;
        // byte offset of (row r, chunk ch) in the swizzled tile: r*128 + ((ch ^ (r & 7)) << 4), r & 7 = 4 (i & 1) + sub
        const uint32_t off = (uint32_t)i * 512u + (((uint32_t)ch ^ (((uint32_t)(i & 1) << 2) + (uint32_t)sub)) << 4);
        cp_async16_zfill(dst0 + off, base_hi + boff, nbytes);
        if (NSPLIT == 3) cp_async16_zfill(dst0 + A_TILE_BYTES + off, base_lo + boff, nbytes);
      }
      cp_async_mbar_arrive_noinc(smem_u32(afull + stage));
      next_stage();
      it0 = it1; it1 = it2;
      advance_n(it2, W);
      q0 = q1; q1 = q2;
    }
    cp_async_commit();
    cp_async_wait<0>();
  } else if (warp >= LOAD_WARP) {
    reg_dealloc<LOAD_REGS>();
    if (warp == LOAD_WARP && lane == 0) role_weight_loader(p, pl, n_op);
  } else {
    reg_alloc<PL_CONS_REGS>();
    run_consumer<NSPLIT, true>(p, pl, warp, lane);
  }
}

}  // namespace

extern "C" int64_t pasco_conv_packed_bytes(int32_t K, int32_t Cin, int32_t Cout) {
  return (int64_t)K * Cin * Cout * 4;
}

extern "C" int pasco_conv_pack_weights(const float* W, int32_t K, int32_t Cin, int32_t Cout, int32_t transpose,
                                       void* packed, pasco_stream_t s) {
  const int N = transpose ? Cin : Cout, Kc = transpose ? Cout : Cin;
  PASCO_CHECK_ARG(Kc % KBLK == 0, "pasco_conv_pack_weights: contraction channels (%d) must be a multiple of 64", Kc);
  PASCO_CHECK_ARG(N % 16 == 0 && N >= 16 && N <= 256, "pasco_conv_pack_weights: output channels (%d) must be a multiple of 16 in [16,256]", N);
  int64_t total = (int64_t)K * (Kc / KBLK) * N * 8;
  k_pack_weights<<<grid_for(total, 256), 256, 0, (cudaStream_t)s>>>(W, K, Cin, Cout, transpose, (uint8_t*)packed);
  PASCO_CHECK_LAUNCH("pasco_conv_pack_weights");
  return 0;
}

namespace {

// output column ranges: up to 128 columns (the register accumulators of a consumer warpgroup) per work item, and
// the tiles per group whose accumulators fit beside each other; small inputs spread tiles over more SMs instead
void column_plan(int Cout, int64_t tiles, int& nsplit, int& ncols, int& T) {
  nsplit = (Cout + ACC_COLS - 1) / ACC_COLS;
  ncols = nsplit > 1 ? ACC_COLS : Cout;
  T = ACC_COLS / ncols;
  if (T > 4) T = 4;
  while (T > 1 && tiles < (int64_t)T * num_sms()) T >>= 1;
}

// split-K plan: few output tiles and many offsets (the dense bottleneck: 32 tiles x 245 offsets) leave most SMs idle with
// one CTA per tile; cut the offsets into `ksplit` ranges so that ~2 x #SM work items exist.  1 = no split.
int splitk_plan(int K, int64_t n_out) {
  const int64_t tiles = (n_out + BLOCK_M - 1) / BLOCK_M;
  if (K < 18 || tiles * 2 > num_sms()) return 1;
  int ks = (int)((2 * (int64_t)num_sms() + tiles - 1) / tiles);
  if (ks > K / 6) ks = K / 6;                       // at least 6 offsets per work item
  return ks < 2 ? 1 : ks;
}

// out[r, :] = bias + Σ_s part[s, r, :]   (deterministic reduction of the split-K partial outputs)
__global__ void k_splitk_reduce(const float* __restrict__ part, int ksplit, int64_t n, int C, const float* __restrict__ bias,
                                float* __restrict__ out, int64_t out_pitch) {
  const int cv = C >> 2;
  const int64_t total = n * cv;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / cv;
    const int c = (int)(t - r * cv) << 2;
    float4 acc = bias ? __ldg(reinterpret_cast<const float4*>(bias + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
    for (int s = 0; s < ksplit; ++s) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(part + ((int64_t)s * n + r) * C + c));
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    *reinterpret_cast<float4*>(out + r * out_pitch + c) = acc;
  }
}

int conv_forward_impl(const float* in, int64_t n_in, const int32_t* nbr, int32_t K, int64_t n_out,
                                     int32_t Cin, int32_t Cout, const void* packed_w, const int32_t* koff_map,
                                     const float* bias, const float* in_scale, const float* in_shift, int32_t in_act,
                                     double* stats, float* out, int32_t precision, int64_t in_pitch, int64_t out_pitch,
                                     int ksplit, float* workspace, pasco_stream_t s) {
  PASCO_CHECK_ARG(precision == 1 || precision == 3, "pasco_conv_forward_tc: precision must be 1 (bf16) or 3 (bf16x3)");
  PASCO_CHECK_ARG(Cin % KBLK == 0, "pasco_conv_forward_tc: Cin (%d) must be a multiple of 64", Cin);
  PASCO_CHECK_ARG(Cout % 16 == 0 && Cout >= 16 && Cout <= 256, "pasco_conv_forward_tc: Cout (%d) must be a multiple of 16 in [16,256]", Cout);
  PASCO_CHECK_ARG(K >= 1 && K <= 1024, "pasco_conv_forward_tc: K (%d) out of range", K);
  PASCO_CHECK_ARG((((uintptr_t)in | (uintptr_t)out | (uintptr_t)packed_w) & 15) == 0, "pasco_conv_forward_tc: pointers must be 16-byte aligned");
  if (n_out == 0) return 0;
  int dev = 0, smem_optin = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  const int n_op = precision == 3 ? 2 : 1;
  int64_t tiles = (n_out + BLOCK_M - 1) / BLOCK_M;
  int nsplit, ncols, T;
  column_plan(Cout, tiles, nsplit, ncols, T);
  if (ksplit > 1) T = 1;
  const int a_stage = n_op * A_TILE_BYTES, b_stage = n_op * ncols * 128;
  const int idx_bytes = IDX_RING * T * BLOCK_M * 4;
  const int fixed = 1024 /*align slack*/ + idx_bytes + 4 * MAX_STAGES * 8 + (stats ? 2 * Cout * 8 : 0);
  int sb = 2;
  int sa = (smem_optin - fixed - sb * b_stage) / a_stage;
  if (sa > 5) {  // room to spare: deepen the weight ring first
    sb = 3;
    sa = (smem_optin - fixed - sb * b_stage) / a_stage;
  }
  if (sa > MAX_STAGES) sa = MAX_STAGES;
  PASCO_CHECK_ARG(sa >= 3, "pasco_conv_forward_tc: not enough shared memory (Cout=%d)", Cout);   // see role_consumer
  ConvParams p;
  p.in = in; p.nbr = nbr; p.wpk = (const uint8_t*)packed_w; p.bias = bias;
  p.in_scale = in_scale; p.in_shift = in_shift; p.out = out; p.stats = stats;
  p.n_out = n_out;
  p.out_pitch = out_pitch > 0 ? out_pitch : Cout;
  p.ksplit = 1; p.kchunk = K;
  if (ksplit > 1) {       // partial outputs [ksplit, n_out, Cout] into the workspace, bias added by the reduction
    p.ksplit = ksplit; p.kchunk = (K + ksplit - 1) / ksplit;
    p.ksplit = (K + p.kchunk - 1) / p.kchunk;       // no empty ranges
    p.out = workspace; p.out_pitch = Cout; p.bias = nullptr; p.stats = nullptr;
  }
  p.in_pitch = in_pitch > 0 ? in_pitch : Cin;
  PASCO_CHECK_ARG(p.out_pitch % 4 == 0 && p.in_pitch % 4 == 0, "pasco_conv_forward_tc: pitches must be multiples of 4 floats");
  p.K = K; p.Cin = Cin; p.Cout = Cout; p.in_act = in_act;
  p.pl_hi = nullptr; p.pl_lo = nullptr; p.pl_pitch = 0;
  p.sa = sa; p.sb = sb; p.tiles_per_group = T; p.nsplit = nsplit; p.ncols = ncols;
  p.koff_base = 0; p.koff_step = 1;
  if (koff_map) {
    bool ident = true, rev = true;
    for (int k = 0; k < K; ++k) {
      ident = ident && koff_map[k] == k;
      rev = rev && koff_map[k] == K - 1 - k;
    }
    PASCO_CHECK_ARG(ident || rev, "pasco_conv_forward_tc: koff_map must be the identity or the reversal");
    if (!ident) { p.koff_base = K - 1; p.koff_step = -1; }
  }
  const size_t smem = (size_t)sa * a_stage + (size_t)sb * b_stage + fixed;
  const int64_t items = (tiles + T - 1) / T * p.ksplit * nsplit;
  const int grid = (int)(items < num_sms() ? items : num_sms());
  cudaError_t e;
  const bool prologue = in_scale != nullptr || in_act != 0;
  auto launch = [&](auto kern) {
    cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (err == cudaSuccess) kern<<<grid, NUM_THREADS, smem, (cudaStream_t)s>>>(p);
    return err;
  };
  if (precision == 3) e = prologue ? launch(k_conv_tc<3, true>) : launch(k_conv_tc<3, false>);
  else e = prologue ? launch(k_conv_tc<1, true>) : launch(k_conv_tc<1, false>);
  if (e != cudaSuccess) {
    set_error("pasco_conv_forward_tc: cudaFuncSetAttribute(%zu bytes) failed: %s", smem, cudaGetErrorString(e));
    return -1;
  }
  PASCO_CHECK_LAUNCH("pasco_conv_forward_tc");
  if (p.ksplit > 1) {
    k_splitk_reduce<<<grid_for(n_out * (Cout / 4), 256), 256, 0, (cudaStream_t)s>>>(workspace, p.ksplit, n_out, Cout, bias, out,
                                                                                out_pitch > 0 ? out_pitch : Cout);
    PASCO_CHECK_LAUNCH("pasco_conv_forward_tc(split-K reduce)");
  }
  return 0;
}

}  // namespace

extern "C" int pasco_conv_forward_tc(const float* in, int64_t n_in, const int32_t* nbr, int32_t K, int64_t n_out,
                                     int32_t Cin, int32_t Cout, const void* packed_w, const int32_t* koff_map,
                                     const float* bias, const float* in_scale, const float* in_shift, int32_t in_act,
                                     double* stats, float* out, int32_t precision, int64_t in_pitch, int64_t out_pitch,
                                     pasco_stream_t s) {
  return conv_forward_impl(in, n_in, nbr, K, n_out, Cin, Cout, packed_w, koff_map, bias, in_scale, in_shift, in_act, stats, out,
                           precision, in_pitch, out_pitch, 1, nullptr, s);
}

extern "C" int pasco_conv_forward_planes(const void* hi, const void* lo, int64_t n_in, const int32_t* nbr, int32_t K,
                                         int64_t n_out, int32_t Cin, int32_t Cout, const void* packed_w,
                                         const int32_t* koff_map, const float* bias, double* stats, float* out,
                                         int32_t precision, int64_t plane_pitch, int64_t out_pitch, pasco_stream_t s) {
  PASCO_CHECK_ARG(precision == 1 || precision == 3, "pasco_conv_forward_planes: precision must be 1 or 3");
  PASCO_CHECK_ARG(hi != nullptr && (precision == 1 || lo != nullptr), "pasco_conv_forward_planes: missing plane (precision 3 needs hi and lo)");
  PASCO_CHECK_ARG(Cin % KBLK == 0, "pasco_conv_forward_planes: Cin (%d) must be a multiple of 64", Cin);
  PASCO_CHECK_ARG(Cout % 16 == 0 && Cout >= 16 && Cout <= 256, "pasco_conv_forward_planes: Cout (%d) must be a multiple of 16 in [16,256]", Cout);
  PASCO_CHECK_ARG(K >= 1 && K <= 1024, "pasco_conv_forward_planes: K (%d) out of range", K);
  const int64_t pitch = plane_pitch > 0 ? plane_pitch : Cin;
  PASCO_CHECK_ARG(pitch % 8 == 0 && (((uintptr_t)hi | (uintptr_t)lo | (uintptr_t)out | (uintptr_t)packed_w) & 15) == 0,
                  "pasco_conv_forward_planes: planes must be 16-byte aligned with a pitch multiple of 8 elements");
  (void)n_in;
  if (n_out == 0) return 0;
  int dev = 0, smem_optin = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  const int n_op = precision == 3 ? 2 : 1;
  const int64_t tiles = (n_out + BLOCK_M - 1) / BLOCK_M;
  int nsplit, ncols, T;
  column_plan(Cout, tiles, nsplit, ncols, T);
  const int a_stage = n_op * A_TILE_BYTES, b_stage = n_op * ncols * 128;
  const int fixed = 1024 + 4 * MAX_STAGES * 8 + (stats ? 2 * Cout * 8 : 0);
  int sb = 2;
  int sa = (smem_optin - fixed - sb * b_stage) / a_stage;
  if (sa > MAX_STAGES) sa = MAX_STAGES;
  static const int sa_env = [] { const char* e = getenv("PASCO_PL_SA"); return e ? atoi(e) : 0; }();
  if (sa_env >= 3 && sa_env < sa) sa = sa_env;
  PASCO_CHECK_ARG(sa >= 3, "pasco_conv_forward_planes: not enough shared memory (Cout=%d)", Cout);   // see role_consumer
  ConvParams p;
  p.in = nullptr; p.nbr = nbr; p.wpk = (const uint8_t*)packed_w; p.bias = bias;
  p.in_scale = nullptr; p.in_shift = nullptr; p.out = out; p.stats = stats;
  p.n_out = n_out;
  p.out_pitch = out_pitch > 0 ? out_pitch : Cout;
  p.in_pitch = Cin;
  PASCO_CHECK_ARG(p.out_pitch % 4 == 0, "pasco_conv_forward_planes: out_pitch must be a multiple of 4 floats");
  p.K = K; p.Cin = Cin; p.Cout = Cout; p.in_act = 0;
  p.sa = sa; p.sb = sb; p.tiles_per_group = T; p.nsplit = nsplit; p.ncols = ncols;
  p.ksplit = 1; p.kchunk = K;
  p.koff_base = 0; p.koff_step = 1;
  if (koff_map) {
    bool ident = true, rev = true;
    for (int k = 0; k < K; ++k) {
      ident = ident && koff_map[k] == k;
      rev = rev && koff_map[k] == K - 1 - k;
    }
    PASCO_CHECK_ARG(ident || rev, "pasco_conv_forward_planes: koff_map must be the identity or the reversal");
    if (!ident) { p.koff_base = K - 1; p.koff_step = -1; }
  }
  p.pl_hi = (const uint16_t*)hi; p.pl_lo = (const uint16_t*)lo; p.pl_pitch = pitch;
  const size_t smem = (size_t)sa * a_stage + (size_t)sb * b_stage + fixed;
  const int64_t items = (tiles + T - 1) / T * nsplit;
  const int grid = (int)(items < num_sms() ? items : num_sms());
  auto launch = [&](auto kern) {
    cudaError_t err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (err == cudaSuccess) kern<<<grid, NUM_THREADS, smem, (cudaStream_t)s>>>(p);
    return err;
  };
  const cudaError_t e = precision == 3 ? launch(k_conv_pl<3>) : launch(k_conv_pl<1>);
  if (e != cudaSuccess) {
    set_error("pasco_conv_forward_planes: cudaFuncSetAttribute(%zu bytes) failed: %s", smem, cudaGetErrorString(e));
    return -1;
  }
  PASCO_CHECK_LAUNCH("pasco_conv_forward_planes");
  return 0;
}

extern "C" int64_t pasco_conv_splitk_workspace_bytes(int32_t K, int64_t n_out, int32_t Cout) {
  const int ks = splitk_plan(K, n_out);
  return ks > 1 ? (int64_t)ks * n_out * Cout * 4 : 0;
}

extern "C" int pasco_conv_forward_splitk(const float* in, int64_t n_in, const int32_t* nbr, int32_t K, int64_t n_out,
                                         int32_t Cin, int32_t Cout, const void* packed_w, const int32_t* koff_map,
                                         const float* bias, const float* in_scale, const float* in_shift, int32_t in_act,
                                         float* out, int32_t precision, int64_t in_pitch, int64_t out_pitch, void* workspace,
                                         int64_t workspace_bytes, pasco_stream_t s) {
  const int ks = splitk_plan(K, n_out);
  PASCO_CHECK_ARG(ks > 1, "pasco_conv_forward_splitk: this shape is not split (workspace_bytes = 0): call pasco_conv_forward_tc");
  PASCO_CHECK_ARG(workspace != nullptr && workspace_bytes >= (int64_t)ks * n_out * Cout * 4,
                  "pasco_conv_forward_splitk: workspace too small (%lld bytes)", (long long)workspace_bytes);
  PASCO_CHECK_ARG(((uintptr_t)workspace & 15) == 0, "pasco_conv_forward_splitk: workspace must be 16-byte aligned");
  return conv_forward_impl(in, n_in, nbr, K, n_out, Cin, Cout, packed_w, koff_map, bias, in_scale, in_shift, in_act, nullptr, out,
                           precision, in_pitch, out_pitch, ks, (float*)workspace, s);
}
