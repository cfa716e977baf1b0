// Weight gradient of the sparse convolution on the Hopper tensor cores (wgmma), sm_90a.
//
//   dW[k] = Σ_o in[nbr[k,o], :]^T @ gout[o, :]
//
// MMA view: D[M = 64 input channels][N = columns of gout] += A^T · G with the voxel rows as the contraction dimension,
// so both operands are MN-major: the very same gathered [rows][64 ch] swizzled tiles the forward kernel builds serve
// as A and the gout tile as B.  "sub-tile" s = (offset k, 64-channel block cb); a unit = two consecutive sub-tiles x
// one range of UC output columns (UC = Cout up to 128); consumer warpgroup h accumulates sub-tile h of the CTA's units
// in registers (at most 128 columns per thread set), walks its share of 64-row tiles, and finally stores its partial
// dW into its own workspace slot; k_wgrad_sum adds the slots of a pass in CTA order (deterministic, no atomics).
#include "common.cuh"
#include "gmma.cuh"

using namespace pasco;
using namespace gmma;

namespace {

constexpr int NUM_GATHER_WARPS = 8;                 // 8 tile rows each
constexpr int CONS_WARP0 = NUM_GATHER_WARPS;         // warps 8-15: consumer warpgroups 0 and 1 (sub-tile 0 / 1 of a unit)
constexpr int NUM_CONS_WARPS = 8;
constexpr int NUM_THREADS = (CONS_WARP0 + NUM_CONS_WARPS) * 32;   // 512
constexpr int ACC_COLS = 128;                        // accumulator columns per consumer thread set (64 registers)
constexpr int WROWS = 64 / NUM_GATHER_WARPS;         // rows of a 64-row tile per gather warp
constexpr int WLOADS = WROWS / 2;                    // float4 loads per lane per sub-tile
constexpr int MAX_STAGES = 8;             // unit (A) ring
constexpr int MAX_GSTAGES = 4;            // gout ring
constexpr int WG_R = 64;                  // voxel rows per tile (contraction block)
constexpr int WG_SUB_BYTES = WG_R * 128;  // one [64 rows][64 ch] bf16 tile = 8 KB

struct WgradParams {
  const float* in;                // k_wgrad_tc: fp32 rows of the layer input and of the output gradient
  const float* gout;
  const uint16_t* in_hi;          // k_wgrad_pl: the same as pre-split bf16 planes (hi [+ lo])
  const uint16_t* in_lo;
  const uint16_t* g_hi;
  const uint16_t* g_lo;
  const int32_t* nbr;
  int64_t n_out;
  int64_t in_pitch, gout_pitch;   // row strides (floats, or elements of the planes)
  int K, Cin, Cout;
  int stages, gstages;            // depths of the unit ring and of the gout ring
  int gblocks;                    // 64-column blocks of gout per gout tile (see gout_block)
  int units_per_pass, num_units, num_subs, passes, ctas_per_pass;
  int uc, ncr;                    // columns per unit, column ranges (unit u = sub-tile pair u / ncr, columns of range u % ncr)
  float* part;                    // [grid][slot]: partial dW of CTA b = cta_in_pass * passes + pass
  int64_t slot;                   // units_per_pass * 128 * uc floats
};

constexpr int IDX_RING = 16;   // unit slots are short: fetch neighbour indices 15 slots ahead (HBM-latency bound otherwise)

// One [WG_R rows][64 ch] sub-tile is gathered by 8 warps x 8 rows; lanes (l & 7) of a warp hold the source row of
// tile row w*8 + (l & 7).  Loads and the convert+store are separate so several sub-tiles can be in flight.
struct SubRegs {
  float4 v[WLOADS];
};

__device__ __forceinline__ void sub_load(SubRegs& r, const float* __restrict__ src, int ld, int cbase_blk, int idx, int lane) {
  const int chunk = lane & 15, rsub = lane >> 4;
  const int cbase = cbase_blk + chunk * 4;
#pragma unroll
  for (int i = 0; i < WLOADS; ++i) {
    const int s = __shfl_sync(0xffffffffu, idx, i * 2 + rsub);
    r.v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (s >= 0) r.v[i] = __ldg(reinterpret_cast<const float4*>(src + (int64_t)s * ld + cbase));
  }
}

template <int NSPLIT>
__device__ __forceinline__ void sub_store(const SubRegs& r, uint8_t* dst_hi, uint8_t* dst_lo, int warp, int lane) {
  const int chunk = lane & 15, rsub = lane >> 4;
#pragma unroll
  for (int i = 0; i < WLOADS; ++i) {
    const float4 x = r.v[i];
    const uint32_t trow = (uint32_t)(warp * WROWS + i * 2 + rsub);
    const uint32_t off = trow * 128u + ((((uint32_t)chunk >> 1) ^ (trow & 7u)) << 4) + (((uint32_t)chunk & 1u) << 3);
    if (NSPLIT == 3) {
      uint2 hi, lo;
      split4(x, hi, lo);
      *reinterpret_cast<uint2*>(dst_hi + off) = hi;
      *reinterpret_cast<uint2*>(dst_lo + off) = lo;
    } else {
      *reinterpret_cast<uint2*>(dst_hi + off) = to_bf16x4(x);
    }
  }
}

// The gout tile of a row tile holds only the 64-column blocks of gout that the CTA's units read, hi blocks then lo
// blocks: with uc = 128 (one unit per pass) the unit's two blocks, with uc = 64 the block of each unit (one block when
// Cout = 64, where both units share it).  Block b of the tile is gout column block gout_block(p, unit0, b).
__device__ __forceinline__ int gout_block(const WgradParams& p, int unit0, int b) {
  return p.uc == 128 ? (unit0 % p.ncr) * 2 + b : (unit0 + b) % p.ncr;
}
// 64-column blocks of gout one CTA copies per row tile (at most gblocks)
__device__ __forceinline__ int gout_nblocks(const WgradParams& p, int nunits) {
  return p.uc == 128 ? 2 : (p.ncr > 1 ? nunits : 1);
}

// Consumer warpgroup hh (0 / 1) accumulates sub-tile hh of every unit of the CTA's pass: acc[q] holds columns
// [64 q, 64 q + 64) of the pass's accumulator, i.e. column block q % (UC / 64) of unit q / (UC / 64).  Every consumer
// warp arrives on the ring "empty" barriers (expected count 8).  After the CTA's last row tile it stores its partial dW
// into its workspace slot: row (u * 128 + 64 hh + channel), column within the unit.
// Retire: one wgmma group stays in flight, as in the convolution consumer.  After committing slot n the warpgroup waits
// for slot n - 1 (wait_group 1) and only then releases slot n - 1's A stage, and the row tile's gout buffer when slot
// n - 1 was the tile's last unit.  The last slot is drained (wait_group 0) before the partial dW is stored.  Each slot's
// MMA chain and its commit sit in one basic block (else ptxas commits an empty group and the wait drains the real MMAs).
template <int NSPLIT, bool CPASYNC, int UC>
__device__ __forceinline__ void wgrad_consumer(const WgradParams& p, const uint8_t* g_smem, const uint8_t* a_smem, int g_bytes, int a_bytes,
                                               uint64_t* full_bar, uint64_t* empty_bar, uint64_t* gfull_bar, uint64_t* gempty_bar,
                                               int unit0, int nunits, int cta_in_pass, int64_t num_rt, int hh, int wq, int lane) {
  constexpr int UNB = UC / 64;
  float acc[2][32];
#pragma unroll
  for (int q = 0; q < 2; ++q)
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[q][i] = 0.f;
  int stage = 0, gb = 0;
  uint32_t phase = 0, gphase = 0;
  int held = -1, held_g = -1;     // A stage and gout buffer of the slot whose MMAs may still be in flight (-1: none)
  auto release_held = [&]() {
    __syncwarp();
    if (lane == 0) {
      if (held >= 0) mbar_arrive(smem_u32(empty_bar + held));
      if (held_g >= 0) mbar_arrive(smem_u32(gempty_bar + held_g));
    }
    held = held_g = -1;
  };
  const uint32_t g_lo_off = p.gblocks * WG_SUB_BYTES;
  for (int64_t rt = cta_in_pass; rt < num_rt; rt += p.ctas_per_pass) {
    mbar_wait(smem_u32(gfull_bar + gb), gphase);
    if (CPASYNC) fence_proxy_async_smem();     // tiles were written by cp.async copies (generic proxy)
    const uint32_t g_hi = smem_u32(g_smem + (size_t)gb * g_bytes);
    for (int u = 0; u < nunits; ++u) {
      mbar_wait(smem_u32(full_bar + stage), phase);
      if (CPASYNC) fence_proxy_async_smem();
      const uint32_t a_hi = smem_u32(a_smem + (size_t)stage * a_bytes) + (uint32_t)hh * WG_SUB_BYTES;
      const uint32_t a_lo = a_hi + 2 * WG_SUB_BYTES;
      const uint64_t da_hi = make_desc_sw128(a_hi, WG_SUB_BYTES, 1024), da_lo = make_desc_sw128(a_lo, WG_SUB_BYTES, 1024);
      // the unit's first block in the gout tile: uc = 128 reads blocks 0-1, uc = 64 the block of unit u
      const uint32_t b = g_hi + (uint32_t)(UC == 128 || p.ncr == 1 ? 0 : u) * WG_SUB_BYTES;
      const uint64_t db_hi = make_desc_sw128(b, WG_SUB_BYTES, 1024), db_lo = make_desc_sw128(b + g_lo_off, WG_SUB_BYTES, 1024);
      // k-step j (16 rows = 2048 bytes = 128 address units); every column adds hi·hi, lo·hi, hi·lo for j = 0, 1, ...
      auto mma_chain = [&](auto& a) {
#pragma unroll
        for (int j = 0; j < WG_R / 16; ++j) {
          if constexpr (UC == 128) {     // one MMA spans the unit's two gout blocks (LBO = the block distance)
            wgmma_n128<1, 1>(a, da_hi + 128 * j, db_hi + 128 * j);
            if (NSPLIT == 3) {
              wgmma_n128<1, 1>(a, da_lo + 128 * j, db_hi + 128 * j);
              wgmma_n128<1, 1>(a, da_hi + 128 * j, db_lo + 128 * j);
            }
          } else {
            wgmma_n64<1, 1>(a, da_hi + 128 * j, db_hi + 128 * j);
            if (NSPLIT == 3) {
              wgmma_n64<1, 1>(a, da_lo + 128 * j, db_hi + 128 * j);
              wgmma_n64<1, 1>(a, da_hi + 128 * j, db_lo + 128 * j);
            }
          }
        }
      };
      wg_fence();
      if constexpr (UC == 128) {           // one unit per pass: the chain is unconditional
        mma_chain(reinterpret_cast<float(&)[64]>(acc));
        wg_commit();
      } else {                             // unit u accumulates into acc[u]: each chain is committed in its own branch
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          if (q == u) {
            mma_chain(acc[q]);
            wg_commit();
          }
        }
      }
      wg_wait<1>();                        // the previous slot's MMAs are complete
      release_held();
      held = stage;
      held_g = u == nunits - 1 ? gb : -1;  // the gout buffer is free after the row tile's last unit
      if (++stage == p.stages) {
        stage = 0;
        phase ^= 1;
      }
    }
    if (++gb == p.gstages) {
      gb = 0;
      gphase ^= 1;
    }
  }
  wg_wait<0>();
  release_held();
  float* slot = p.part + (int64_t)blockIdx.x * p.slot;
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    const int u = q / UNB;
    if (u >= nunits) continue;
    const int col0 = (q % UNB) * 64;
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int ch = frag_row(i, wq, lane), col = col0 + frag_col(i, lane);
      *reinterpret_cast<float2*>(slot + (int64_t)(u * 128 + hh * 64 + ch) * UC + col) = make_float2(acc[q][i], acc[q][i + 1]);
    }
  }
}

template <int NSPLIT, bool CPASYNC>
__device__ __forceinline__ void run_wgrad_consumer(const WgradParams& p, const uint8_t* g_smem, const uint8_t* a_smem, int g_bytes,
                                                   int a_bytes, uint64_t* bars, int unit0, int nunits, int cta_in_pass,
                                                   int64_t num_rt, int warp, int lane) {
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + MAX_STAGES;
  uint64_t* gfull_bar = bars + 2 * MAX_STAGES;
  uint64_t* gempty_bar = bars + 2 * MAX_STAGES + MAX_GSTAGES;
  const int hh = (warp - CONS_WARP0) >> 2, wq = (warp - CONS_WARP0) & 3;
  if (p.uc == 128)
    wgrad_consumer<NSPLIT, CPASYNC, 128>(p, g_smem, a_smem, g_bytes, a_bytes, full_bar, empty_bar, gfull_bar, gempty_bar,
                                         unit0, nunits, cta_in_pass, num_rt, hh, wq, lane);
  else
    wgrad_consumer<NSPLIT, CPASYNC, 64>(p, g_smem, a_smem, g_bytes, a_bytes, full_bar, empty_bar, gfull_bar, gempty_bar,
                                        unit0, nunits, cta_in_pass, num_rt, hh, wq, lane);
}

// dW[k][ci][co] += Σ_c part[c * passes + pass][...] over the CTAs c of the pass that owns (k, ci, co), in CTA order
__global__ void k_wgrad_sum(const WgradParams p, float* __restrict__ dW) {
  const int CB = p.Cin / 64;
  const int64_t total = (int64_t)p.K * p.Cin * p.Cout;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t kc = e / p.Cout;
    const int col = (int)(e - kc * p.Cout);
    const int k = (int)(kc / p.Cin), ci = (int)(kc - (int64_t)k * p.Cin);
    const int sub = k * CB + ci / 64, hh = sub & 1;
    const int unit = (sub >> 1) * p.ncr + col / p.uc;
    const int pass = unit / p.units_per_pass, u = unit - pass * p.units_per_pass;
    const float* src = p.part + (int64_t)pass * p.slot + (int64_t)(u * 128 + hh * 64 + (ci & 63)) * p.uc + col % p.uc;
    float acc = 0.f;
    for (int c = 0; c < p.ctas_per_pass; ++c) acc += __ldg(src + (int64_t)c * p.passes * p.slot);
    dW[e] += acc;
  }
}

template <int NSPLIT>
__global__ void __launch_bounds__(NUM_THREADS, 1) k_wgrad_tc(const __grid_constant__ WgradParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int n_op = (NSPLIT == 3) ? 2 : 1;
  const int g_bytes = n_op * p.gblocks * WG_SUB_BYTES;   // one gout tile (hi blocks [+ lo blocks])
  const int a_bytes = n_op * 2 * WG_SUB_BYTES;           // one stage: two sub-tiles (hi [+ lo])
  uint8_t* g_smem = smem;                                // [gstages][g_bytes]
  uint8_t* a_smem = smem + (size_t)p.gstages * g_bytes;  // [stages][a_bytes]
  uint64_t* bars = reinterpret_cast<uint64_t*>(a_smem + (size_t)p.stages * a_bytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + MAX_STAGES;
  uint64_t* gfull_bar = bars + 2 * MAX_STAGES;
  uint64_t* gempty_bar = bars + 2 * MAX_STAGES + MAX_GSTAGES;

  const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x, 0) >> 5, lane = threadIdx.x & 31;   // provably warp-uniform, else ptxas serializes the wgmma
  const int CB = p.Cin / 64;
  const int pass = blockIdx.x % p.passes;
  const int cta_in_pass = blockIdx.x / p.passes;
  const int unit0 = pass * p.units_per_pass;
  const int nunits = min(p.units_per_pass, p.num_units - unit0);
  const int64_t num_rt = (p.n_out + WG_R - 1) / WG_R;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(smem_u32(full_bar + s), NUM_GATHER_WARPS);
      mbar_init(smem_u32(empty_bar + s), NUM_CONS_WARPS);
    }
    for (int b = 0; b < p.gstages; ++b) {
      mbar_init(smem_u32(gfull_bar + b), NUM_GATHER_WARPS);
      mbar_init(smem_u32(gempty_bar + b), NUM_CONS_WARPS);
    }
    fence_barrier_init();
  }
  // slot descriptor table: [j][0]=type (0 gout, 1 unit), [1],[2]=column bases of the two sub-tiles (-1 = none),
  // [3],[4]=kernel offset of the two sub-tiles (-1 = padding)
  int* idx_ring = reinterpret_cast<int*>(bars + 2 * (MAX_STAGES + MAX_GSTAGES));   // [IDX_RING][2][WG_R]
  int* desc = idx_ring + IDX_RING * 2 * WG_R;                                    // [<=16][8]
  {
    for (int j = threadIdx.x; j < 1 + nunits; j += NUM_THREADS) {
      int* dj = desc + j * 8;
      if (j == 0) {                          // the gout slot: the tile's one or two column blocks
        dj[0] = 0; dj[1] = gout_block(p, unit0, 0) * 64;
        dj[2] = gout_nblocks(p, nunits) > 1 ? gout_block(p, unit0, 1) * 64 : -1; dj[3] = -1; dj[4] = -1;
      } else {
        dj[0] = 1;
        for (int h = 0; h < 2; ++h) {
          const int sub = ((unit0 + (j - 1)) / p.ncr) * 2 + h;
          const bool ok = sub < p.num_subs;
          dj[1 + h] = ok ? (sub % CB) * 64 : 0;
          dj[3 + h] = ok ? sub / CB : -1;
        }
      }
    }
  }
  __syncthreads();
  const int spr = 1 + nunits;               // slots per row tile

  if (warp < NUM_GATHER_WARPS) {
    // Flat slot sequence per row tile:  one gout slot (the tile's one or two 64-column blocks), then one slot per unit
    // (two gathered sub-tiles).  Every slot = 2 x WLOADS float4 loads per lane; the loads of slot s+1 are in flight in
    // registers while slot s is converted and stored; neighbour indices arrive through a cp.async ring PF_DIST slots
    // ahead.  Slot geometry comes from a small descriptor table in shared memory (no divisions in the loop).
    const int my_r = warp * WROWS + (lane & (WROWS - 1));          // this lane's row inside the 64-row tile
    const int64_t stride_rt = p.ctas_per_pass;
    constexpr int PF_DIST = 12;

    auto prefetch = [&](int64_t rt, int j, int g) {              // indices of slot (rt, j) → ring entry g
      if (lane < 16) {
        const int h = lane >> 3;
        const int k = desc[j * 8 + 3 + h];
        int* d = idx_ring + ((g & (IDX_RING - 1)) * 2 + h) * WG_R + warp * WROWS + (lane & 7);
        const int64_t row = rt * WG_R + warp * WROWS + (lane & 7);
        if (p.nbr && k >= 0 && rt < num_rt && row < p.n_out) cp_async4(smem_u32(d), p.nbr + (int64_t)k * p.n_out + row);
        else *d = (k >= 0 && rt < num_rt && row < p.n_out) ? (int)row : -1;
      }
      cp_async_commit();
    };
    auto issue = [&](int64_t rt, int j, int g, SubRegs (&r)[2]) {
      cp_async_wait<PF_DIST - 1>();
      __syncwarp();
      const int* dj = desc + j * 8;
      const int64_t row = rt * WG_R + my_r;
      if (dj[0] == 0) {                                            // gout slot: identity rows
        int gidx = row < p.n_out ? (int)row : -1;
        sub_load(r[0], p.gout, (int)p.gout_pitch, dj[1], gidx, lane);
        if (dj[2] >= 0) sub_load(r[1], p.gout, (int)p.gout_pitch, dj[2], gidx, lane);
      } else {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          int idx = idx_ring[((g & (IDX_RING - 1)) * 2 + h) * WG_R + my_r];
          if (!p.nbr && idx >= 0) idx = (int)row;
          sub_load(r[h], p.in, (int)p.in_pitch, dj[1 + h], idx, lane);
        }
      }
    };
    int stage = 0, gb = 0;
    uint32_t phase = 0, gphase = 0;
    auto store = [&](int j, SubRegs (&r)[2]) {
      const int* dj = desc + j * 8;
      if (dj[0] == 0) {
        mbar_wait(smem_u32(gempty_bar + gb), gphase ^ 1);
        uint8_t* g = g_smem + (size_t)gb * g_bytes;
        const int GB = p.gblocks;
        sub_store<NSPLIT>(r[0], g, g + (size_t)GB * WG_SUB_BYTES, warp, lane);
        if (dj[2] >= 0) sub_store<NSPLIT>(r[1], g + WG_SUB_BYTES, g + (size_t)(GB + 1) * WG_SUB_BYTES, warp, lane);
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(gfull_bar + gb));
        if (++gb == p.gstages) {
          gb = 0;
          gphase ^= 1;
        }
      } else {
        mbar_wait(smem_u32(empty_bar + stage), phase ^ 1);
        uint8_t* a = a_smem + (size_t)stage * a_bytes;
#pragma unroll
        for (int h = 0; h < 2; ++h) sub_store<NSPLIT>(r[h], a + (size_t)h * WG_SUB_BYTES, a + (size_t)(2 + h) * WG_SUB_BYTES, warp, lane);
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(full_bar + stage));
        if (++stage == p.stages) {
          stage = 0;
          phase ^= 1;
        }
      }
    };

    // three cursors over the same slot sequence: prefetch (PF_DIST ahead), load, store
    int64_t p_rt = cta_in_pass, l_rt = cta_in_pass, s_rt = cta_in_pass;
    int p_j = 0, l_j = 0, s_j = 0, p_g = 0, l_g = 0;
#define WG_ADV(rt, j) do { if (++(j) == spr) { (j) = 0; (rt) += stride_rt; } } while (0)
    if (l_rt < num_rt) {
      for (int a = 0; a < PF_DIST; ++a) {
        prefetch(p_rt, p_j, p_g);
        ++p_g;
        WG_ADV(p_rt, p_j);
      }
      SubRegs ra[2], rb[2];
      auto issue_next = [&](SubRegs (&r)[2]) {
        issue(l_rt, l_j, l_g, r);
        prefetch(p_rt, p_j, p_g);
        ++p_g;
        WG_ADV(p_rt, p_j);
        ++l_g;
        WG_ADV(l_rt, l_j);
      };
      auto store_next = [&](SubRegs (&r)[2]) {
        store(s_j, r);
        if (++s_j == spr) {
          s_j = 0;
          s_rt += stride_rt;
        }
      };
      issue_next(ra);
      while (s_rt < num_rt) {
        if (l_rt < num_rt) issue_next(rb);
        store_next(ra);
        if (s_rt >= num_rt) break;
        if (l_rt < num_rt) issue_next(ra);
        store_next(rb);
      }
    }
#undef WG_ADV
    cp_async_wait<0>();
  } else {
    run_wgrad_consumer<NSPLIT, false>(p, g_smem, a_smem, g_bytes, a_bytes, bars, unit0, nunits, cta_in_pass, num_rt, warp, lane);
  }
}

// ------------------------------------------------------------------------------------------------------------
// Plane-gather variant of the weight gradient: both operands arrive as pre-split bf16 planes
// ------------------------------------------------------------------------------------------------------------
// Same MMA view, consumers, passes and epilogue as k_wgrad_tc; the producers only move bytes: 16-byte cp.async
// copies from the `in` planes (gathered rows; a missing neighbour is a zero-fill copy that touches no memory) and from
// the `gout` planes (contiguous rows) straight into the 128-byte-swizzled tiles.  Slot 0 of a row tile = the whole gout
// tile, slots 1.. = one unit of two gathered sub-tiles each; every producer thread arrives on the slot's "full" barrier
// with cp.async.mbarrier.arrive.noinc (count = 32 lanes of the filling warp), so the hardware completes it when the last
// copy has landed and the producers run a whole ring ahead of the MMA.
template <int NSPLIT>
__global__ void __launch_bounds__(NUM_THREADS, 1) k_wgrad_pl(const __grid_constant__ WgradParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int n_op = (NSPLIT == 3) ? 2 : 1;
  const int g_bytes = n_op * p.gblocks * WG_SUB_BYTES;   // one gout tile (hi blocks [+ lo blocks])
  const int a_bytes = n_op * 2 * WG_SUB_BYTES;           // one stage: two sub-tiles (hi, hi [, lo, lo])
  uint8_t* g_smem = smem;                                // [gstages][g_bytes]
  uint8_t* a_smem = smem + (size_t)p.gstages * g_bytes;  // [stages][a_bytes]
  uint64_t* bars = reinterpret_cast<uint64_t*>(a_smem + (size_t)p.stages * a_bytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + MAX_STAGES;
  uint64_t* gfull_bar = bars + 2 * MAX_STAGES;
  uint64_t* gempty_bar = bars + 2 * MAX_STAGES + MAX_GSTAGES;

  const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x, 0) >> 5, lane = threadIdx.x & 31;   // provably warp-uniform, else ptxas serializes the wgmma
  const int CB = p.Cin / 64;
  const int pass = blockIdx.x % p.passes;
  const int cta_in_pass = blockIdx.x / p.passes;
  const int unit0 = pass * p.units_per_pass;
  const int nunits = min(p.units_per_pass, p.num_units - unit0);
  const int64_t num_rt = (p.n_out + WG_R - 1) / WG_R;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(smem_u32(full_bar + s), 32);    // one cp.async arrival per lane of the warp that fills the slot
      mbar_init(smem_u32(empty_bar + s), NUM_CONS_WARPS);
    }
    for (int b = 0; b < p.gstages; ++b) {
      mbar_init(smem_u32(gfull_bar + b), 32);
      mbar_init(smem_u32(gempty_bar + b), NUM_CONS_WARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < NUM_GATHER_WARPS) {
    // ONE WARP PER SLOT, ownership split by resource:
    //   * warp 7 fills every gout tile (a ring of gstages buffers, filled in order by the same warp, so its parity wait
    //     on a "gout empty" barrier is never more than one phase away from the barrier);
    //   * warps 0 .. Wu-1 (Wu = min(7, stages)) fill the unit slots ord = w, w + Wu, ... of the CTA's unit sequence
    //     (row tile major): the stride Wu <= stages keeps a warp within one revolution of the unit ring.
    // A warp waits only on barriers of slots it owns.  (Letting all 8 warps take slots round-robin across both rings, or
    // letting every warp observe every barrier, deadlocks: a parity wait is only sound when the waiter is neither two
    // revolutions ahead of nor one revolution behind the barrier — tools/pipeline_sim.py replays the three schemes.)
    // lane = (row sub-index 0..3, 16-byte chunk 0..7): one copy instruction moves 4 tile rows.  For a unit slot lane l
    // holds the neighbour indices of rows l and l+32 of both sub-tiles (four coalesced 128-byte loads, fetched one of
    // the warp's slots ahead), distributed by one shuffle per instruction.
    const int ch = lane & 7, sub = lane >> 3;
    const int64_t stride_rt = p.ctas_per_pass;
    const int64_t my_rts = cta_in_pass < num_rt ? (num_rt - cta_in_pass + stride_rt - 1) / stride_rt : 0;   // row tiles of this CTA
    const uint8_t* in_hi = reinterpret_cast<const uint8_t*>(p.in_hi);
    const uint8_t* in_lo = reinterpret_cast<const uint8_t*>(p.in_lo);
    const uint8_t* gp_hi = reinterpret_cast<const uint8_t*>(p.g_hi);
    const uint8_t* gp_lo = reinterpret_cast<const uint8_t*>(p.g_lo);
    // unit producers: Wu = the largest divisor of `stages` that is <= 7, so that warp w always fills the same stages
    // (w, w + Wu, ...) and sees every phase of their "empty" barriers
    int Wu = 1;
    for (int c = 2; c <= NUM_GATHER_WARPS - 1; ++c)
      if (p.stages % c == 0) Wu = c;
    // gout producers: the last Wg warps, Wg = the largest divisor of `gstages` that the unit producers leave free; warp
    // 8 - Wg + i fills the row tiles i, i + Wg, ... and so always the same gout buffers
    int Wg = 1;
    for (int c = 2; c <= NUM_GATHER_WARPS - Wu; ++c)
      if (p.gstages % c == 0) Wg = c;
    if (warp >= NUM_GATHER_WARPS - Wg) {
      // ---- gout tiles: [64 rows][the units' 64-column blocks] per plane, contiguous rows ----
      const int GB = p.gblocks, gn = gout_nblocks(p, nunits);
      const int64_t gcol0 = gout_block(p, unit0, 0) * 64 * 2, gcol1 = gout_block(p, unit0, gn - 1) * 64 * 2;   // bytes
      int gb = warp - (NUM_GATHER_WARPS - Wg);     // < Wg <= gstages
      uint32_t gphase = 0;
      for (int64_t rti = gb; rti < my_rts; rti += Wg) {
        const int64_t rt = cta_in_pass + rti * stride_rt;
        mbar_wait(smem_u32(gempty_bar + gb), gphase ^ 1);
        const uint32_t g0 = smem_u32(g_smem + (size_t)gb * g_bytes) + (uint32_t)sub * 128u;
#pragma unroll 4
        for (int i = 0; i < WG_R / 4; ++i) {
          const int64_t row = rt * WG_R + i * 4 + sub;
          const uint32_t nbytes = row < p.n_out ? 16u : 0u;
          const int64_t boff = ((row < p.n_out ? row : 0) * p.gout_pitch + ch * 8) * 2;
          const uint32_t off = (uint32_t)i * 512u + (((uint32_t)ch ^ (((uint32_t)(i & 1) << 2) + (uint32_t)sub)) << 4);
          for (int b = 0; b < gn; ++b) {
            const int64_t src = boff + (b == 0 ? gcol0 : gcol1);
            cp_async16_zfill(g0 + (uint32_t)b * WG_SUB_BYTES + off, gp_hi + src, nbytes);
            if (NSPLIT == 3) cp_async16_zfill(g0 + (uint32_t)(GB + b) * WG_SUB_BYTES + off, gp_lo + src, nbytes);
          }
        }
        cp_async_mbar_arrive_noinc(smem_u32(gfull_bar + gb));
        gb += Wg;                                   // at most one wrap: Wg <= gstages
        if (gb >= p.gstages) {
          gb -= p.gstages;
          gphase ^= 1;
        }
      }
    } else if (warp < Wu) {
      // ---- units: two gathered [64 rows][64 ch] sub-tiles each ----
      const int64_t total_units = my_rts * nunits;
      struct Idx4 { int v[4]; };                    // [sub-tile h][row half]
      auto load_idx = [&](int64_t ord) -> Idx4 {
        Idx4 r;
        r.v[0] = r.v[1] = r.v[2] = r.v[3] = -1;
        if (ord < total_units) {
          const int64_t rt = cta_in_pass + (ord / nunits) * stride_rt;
          const int u = (int)(ord % nunits);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int sbi = ((unit0 + u) / p.ncr) * 2 + h;
#pragma unroll
            for (int q = 0; q < 2; ++q) {
              const int64_t row = rt * WG_R + q * 32 + lane;
              if (sbi < p.num_subs && row < p.n_out)
                r.v[h * 2 + q] = p.nbr ? __ldg(p.nbr + (int64_t)(sbi / CB) * p.n_out + row) : (int)row;
            }
          }
        }
        return r;
      };
      int stage = warp;                             // warp < Wu <= stages
      uint32_t phase = 0;
      Idx4 q0 = load_idx(warp);
      for (int64_t ord = warp; ord < total_units; ord += Wu) {
        const Idx4 q1 = load_idx(ord + Wu);         // indices of this warp's next unit
        const int u = (int)(ord % nunits);
        mbar_wait(smem_u32(empty_bar + stage), phase ^ 1);
        const uint32_t a0 = smem_u32(a_smem + (size_t)stage * a_bytes) + (uint32_t)sub * 128u;
        const int sb0 = ((unit0 + u) / p.ncr) * 2;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int sbi = sb0 + h;
          const int64_t coff_b = ((int64_t)(sbi < p.num_subs ? sbi % CB : 0) * 64 + ch * 8) * 2;
#pragma unroll
          for (int i = 0; i < WG_R / 4; ++i) {
            const int idx = __shfl_sync(0xffffffffu, q0.v[h * 2 + (i >> 3)], ((i & 7) << 2) + sub);
            const uint32_t nbytes = idx >= 0 ? 16u : 0u;
            const int64_t boff = (int64_t)(idx >= 0 ? idx : 0) * p.in_pitch * 2 + coff_b;
            const uint32_t off = (uint32_t)i * 512u + (((uint32_t)ch ^ (((uint32_t)(i & 1) << 2) + (uint32_t)sub)) << 4);
            cp_async16_zfill(a0 + (uint32_t)h * WG_SUB_BYTES + off, in_hi + boff, nbytes);
            if (NSPLIT == 3) cp_async16_zfill(a0 + (uint32_t)(2 + h) * WG_SUB_BYTES + off, in_lo + boff, nbytes);
          }
        }
        cp_async_mbar_arrive_noinc(smem_u32(full_bar + stage));
        stage += Wu;                                // at most one wrap: Wu <= stages
        if (stage >= p.stages) {
          stage -= p.stages;
          phase ^= 1;
        }
        q0 = q1;
      }
    }
    cp_async_commit();
    cp_async_wait<0>();
  } else {
    run_wgrad_consumer<NSPLIT, true>(p, g_smem, a_smem, g_bytes, a_bytes, bars, unit0, nunits, cta_in_pass, num_rt, warp, lane);
  }
}

// CTAs per pass: at least one per SM, and enough that no CTA sums more than WG_MAX_RT row tiles in its fp32 register
// accumulators before adding its partial dW (the rounding error of that sum grows with its length)
constexpr int64_t WG_MAX_RT = 128;
int ctas_per_pass(int64_t num_rt, int passes) {
  int64_t cpp = num_sms() / passes;
  const int64_t need = (num_rt + WG_MAX_RT - 1) / WG_MAX_RT;
  if (cpp < need) cpp = need;
  if (cpp > num_rt) cpp = num_rt;
  return cpp < 1 ? 1 : (int)cpp;
}

// unit geometry: uc columns per unit (the consumers' 128 accumulator columns hold 128 / uc units), ncr column ranges
void unit_plan(WgradParams& p, int K, int Cin, int Cout) {
  p.uc = Cout <= ACC_COLS ? Cout : (Cout % ACC_COLS == 0 ? ACC_COLS : 64);
  p.ncr = Cout / p.uc;
  p.num_subs = K * (Cin / 64);
  p.num_units = (p.num_subs + 1) / 2 * p.ncr;
  p.units_per_pass = ACC_COLS / p.uc;
  if (p.units_per_pass > p.num_units) p.units_per_pass = p.num_units;
  p.passes = (p.num_units + p.units_per_pass - 1) / p.units_per_pass;
  p.units_per_pass = (p.num_units + p.passes - 1) / p.passes;
}

// The host half of both weight-gradient launches.  The caller sets the operands of p: fp32 rows in / gout (register
// gather, k_wgrad_tc) or, when in_hi is set, their bf16 planes (plane gather, k_wgrad_pl), with row pitches (0 = Cin /
// Cout).  The per-CTA partials are summed in a fixed order into dW through a stream-ordered workspace.
int wgrad_launch(const char* fn, WgradParams& p, int64_t n_out, int32_t K, int32_t Cin, int32_t Cout, float* dW,
                 int32_t precision, pasco_stream_t s) {
  const bool planes = p.in_hi != nullptr;
  PASCO_CHECK_ARG(precision == 1 || precision == 3, "%s: precision must be 1 or 3", fn);
  PASCO_CHECK_ARG(Cin % 64 == 0 && Cout % 64 == 0 && Cout <= 256,
                  "%s: Cin (%d) and Cout (%d) must be multiples of 64, Cout <= 256", fn, Cin, Cout);
  if (p.in_pitch <= 0) p.in_pitch = Cin;
  if (p.gout_pitch <= 0) p.gout_pitch = Cout;
  if (planes)
    PASCO_CHECK_ARG(p.in_pitch % 8 == 0 && p.gout_pitch % 8 == 0 &&
                    (((uintptr_t)p.in_hi | (uintptr_t)p.in_lo | (uintptr_t)p.g_hi | (uintptr_t)p.g_lo) & 15) == 0,
                    "%s: planes must be 16-byte aligned with pitches multiple of 8 elements", fn);
  if (n_out == 0) return 0;
  int dev = 0, smem_optin = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  unit_plan(p, K, Cin, Cout);
  p.gblocks = p.uc == 128 ? 2 : (p.ncr > 1 ? p.units_per_pass : 1);
  // shared memory: the gout ring, the unit ring, barriers and, for k_wgrad_tc, its index ring and slot descriptors.
  // With one wgmma group in flight the consumers hold one buffer of each ring, so gstages - 1 gout tiles and stages - 1
  // unit slots (units_per_pass per row tile) can be filled ahead of the MMAs: the two depths are picked together for
  // the most row tiles filled ahead, then for the most unit stages.
  const int n_op = precision == 3 ? 2 : 1;
  const int g_bytes = n_op * p.gblocks * WG_SUB_BYTES;
  const int a_bytes = n_op * 2 * WG_SUB_BYTES;
  const int fixed = 1024 + 2 * (MAX_STAGES + MAX_GSTAGES) * 8 + (planes ? 0 : IDX_RING * 2 * WG_R * 4 + 16 * 8 * 4);
  const int upr = p.units_per_pass;
  int stages = 0, gstages = 0, best = -1;
  for (int gs = 2; gs <= MAX_GSTAGES; ++gs) {
    const int st = std::min(MAX_STAGES, (smem_optin - fixed - gs * g_bytes) / a_bytes);
    const int ahead = std::min((gs - 1) * upr, st - 1);     // row tiles filled ahead, times units_per_pass
    if (st >= 3 && ahead > best) {
      best = ahead;
      stages = st;
      gstages = gs;
    }
  }
  PASCO_CHECK_ARG(stages >= 3, "%s: not enough shared memory", fn);   // a stage is filled, one multiplied, one held back
  if (planes) {   // the stage count with the largest divisor <= 7 (= the number of unit producer warps, see k_wgrad_pl)
    int pick = stages, pick_w = 0;
    for (int st = stages; st >= 3; --st) {
      int w = 1;
      for (int c = 2; c <= 7; ++c)
        if (st % c == 0) w = c;
      if (w > pick_w) { pick_w = w; pick = st; }
    }
    stages = pick;
  }
  p.n_out = n_out; p.K = K; p.Cin = Cin; p.Cout = Cout;
  p.stages = stages;
  p.gstages = gstages;
  p.ctas_per_pass = ctas_per_pass((n_out + WG_R - 1) / WG_R, p.passes);
  p.slot = (int64_t)p.units_per_pass * 128 * p.uc;
  const size_t smem = (size_t)gstages * g_bytes + (size_t)stages * a_bytes + fixed;
  const int grid = p.passes * p.ctas_per_pass;
  const cudaStream_t st = (cudaStream_t)s;
  cudaError_t e = ws_alloc((void**)&p.part, (size_t)grid * p.slot * sizeof(float), st);
  if (e != cudaSuccess) {
    set_error("%s: workspace of %lld bytes: %s", fn, (long long)grid * p.slot * 4, cudaGetErrorString(e));
    return -1;
  }
  void (*kern)(WgradParams) = planes ? (precision == 3 ? k_wgrad_pl<3> : k_wgrad_pl<1>)
                                     : (precision == 3 ? k_wgrad_tc<3> : k_wgrad_tc<1>);
  e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e == cudaSuccess) {
    kern<<<grid, NUM_THREADS, smem, st>>>(p);
    k_wgrad_sum<<<grid_for((int64_t)K * Cin * Cout, 256), 256, 0, st>>>(p, dW);
  }
  cudaFreeAsync(p.part, st);
  if (e != cudaSuccess) {
    set_error("%s: cudaFuncSetAttribute failed: %s", fn, cudaGetErrorString(e));
    return -1;
  }
  PASCO_CHECK_LAUNCH(fn);
  return 0;
}

}  // namespace

extern "C" int pasco_conv_wgrad_tc(const float* in, int64_t /*n_in*/, const int32_t* nbr, int32_t K, int64_t n_out,
                                   int32_t Cin, int32_t Cout, const float* gout, float* dW, int32_t precision,
                                   int64_t in_pitch, int64_t gout_pitch, pasco_stream_t s) {
  WgradParams p = {};
  p.in = in; p.gout = gout; p.nbr = nbr; p.in_pitch = in_pitch; p.gout_pitch = gout_pitch;
  return wgrad_launch("pasco_conv_wgrad_tc", p, n_out, K, Cin, Cout, dW, precision, s);
}

extern "C" int pasco_conv_wgrad_planes(const void* in_hi, const void* in_lo, int64_t /*n_in*/, const int32_t* nbr, int32_t K,
                                       int64_t n_out, int32_t Cin, int32_t Cout, const void* g_hi, const void* g_lo,
                                       float* dW, int32_t precision, int64_t in_pitch, int64_t gout_pitch, pasco_stream_t s) {
  PASCO_CHECK_ARG(in_hi && g_hi && (precision == 1 || (in_lo && g_lo)), "pasco_conv_wgrad_planes: missing plane");
  WgradParams p = {};
  p.in_hi = (const uint16_t*)in_hi; p.in_lo = (const uint16_t*)in_lo; p.g_hi = (const uint16_t*)g_hi; p.g_lo = (const uint16_t*)g_lo;
  p.nbr = nbr; p.in_pitch = in_pitch; p.gout_pitch = gout_pitch;
  return wgrad_launch("pasco_conv_wgrad_planes", p, n_out, K, Cin, Cout, dW, precision, s);
}
