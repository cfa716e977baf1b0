// Test-time post-processing of PaSCo (sm_90a): the M-subnet ensemble of ensembler.py:20-187 and the panoptic inference
// of helper.py:91-303, on sparse rows of the 256x256x32 reference grid instead of dense [Q, 256, 256, 32] volumes.
//
// Every kernel is memory-bound and deterministic: no floating-point atomics.  Column sums are written as per-CTA
// partials and added in CTA order (k_colsum_reduce); the panoptic areas are integer histograms, exact in any order.
// Arithmetic that the reference performs as separate fp32 tensor operations is written with __fmul_rn / __fadd_rn /
// __fdiv_rn so that nvcc cannot contract it into a fused multiply-add.
#include "common.cuh"
#include "gmma.cuh"
#include "semantic.cuh"

using namespace pasco;

namespace {

// ------------------------------------------------------------------------------------------------
// pose lookup: reference cell → row of the subnet's sparse tensor (transform_utils.py:55-76,160-181)
// ------------------------------------------------------------------------------------------------
struct Pose {
  float t[12];   // rows 0-2 of the 4x4 pose, row-major
};

__global__ void k_pose_lookup(const uint64_t* __restrict__ keys, const int32_t* __restrict__ vals, uint32_t mask,
                              const Pose T, int X, int Y, int Z, int32_t* __restrict__ cell_row,
                              uint8_t* __restrict__ cell_mask) {
  const int64_t cells = (int64_t)X * Y * Z;
  const float lo[3] = {0.f, -25.6f, -2.f};
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < cells; i += (int64_t)gridDim.x * blockDim.x) {
    const int c[3] = {(int)(i / ((int64_t)Y * Z)), (int)((i / Z) % Y), (int)(i % Z)};
    float p[3], q[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) p[d] = __fadd_rn(__fadd_rn(__fmul_rn((float)c[d], 0.2f), 0.1f), lo[d]);
    bool ok = true;
    int v[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      q[d] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T.t[4 * d], p[0]), __fmul_rn(T.t[4 * d + 1], p[1])),
                                 __fmul_rn(T.t[4 * d + 2], p[2])), T.t[4 * d + 3]);
      const float r = rintf(__fdiv_rn(__fsub_rn(__fsub_rn(q[d], lo[d]), 0.1f), 0.2f));   // torch.round: half to even
      ok = ok && r >= -32768.f && r <= 32767.f;
      v[d] = ok ? (int)r : 0;
    }
    const int row = ok ? table_find(keys, vals, mask, pack_key(0, v[0], v[1], v[2])) : -1;
    cell_row[i] = row;
    if (cell_mask) cell_mask[i] = row >= 0;
  }
}

__global__ void k_cell_mask_or(const int32_t* __restrict__ cell_row, int64_t n, uint8_t* __restrict__ mask) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    if (__ldg(cell_row + i) >= 0) mask[i] = 1;
}

__global__ void k_lookup_rows(const int32_t* __restrict__ cell_row, const int32_t* __restrict__ lin, int64_t n,
                              int32_t* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = __ldg(cell_row + __ldg(lin + i));
}

// subnet box (net_panoptic_sparse.py:430-459): a row at (x, y, z) in [lo, hi] (inclusive) takes the cell (x, y, z) − lo of
// the X x Y x Z box.  A row outside [lo, hi], or at a cell another row already holds, is only counted; the per-warp
// counts reach counts[] as integer atomics.
struct BoxBounds {
  int lo[3], hi[3];
};

__global__ void k_box_cells(const int32_t* __restrict__ coords, int64_t n, const BoxBounds b, int X, int Y, int Z,
                            int32_t* __restrict__ cell_row, uint8_t* __restrict__ cell_mask, int32_t* __restrict__ counts) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int lane = threadIdx.x & 31;
  int outside = 0, taken = 0;
  // every lane of a warp runs the same trip count, so the whole warp reaches the reductions below
  for (int64_t base = blockIdx.x * (int64_t)blockDim.x + threadIdx.x - lane; base < n; base += stride) {
    const int64_t i = base + lane;
    if (i >= n) continue;
    int64_t c[3];
    bool in = true;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      const int v = __ldg(coords + 4 * i + 1 + d);
      in = in && v >= b.lo[d] && v <= b.hi[d];
      c[d] = (int64_t)v - b.lo[d];
    }
    if (!in) {
      ++outside;
      continue;
    }
    const int64_t cell = (c[0] * Y + c[1]) * Z + c[2];
    if (atomicCAS(cell_row + cell, -1, (int32_t)i) != -1) {
      ++taken;
      continue;
    }
    cell_mask[cell] = 1;
  }
  outside = __reduce_add_sync(0xffffffffu, outside);
  taken = __reduce_add_sync(0xffffffffu, taken);
  if (lane == 0) {
    if (outside) atomicAdd(counts, outside);
    if (taken) atomicAdd(counts + 1, taken);
  }
}

// ------------------------------------------------------------------------------------------------
// mask rows: sigmoid gather (MERGE = false) or matched running average (MERGE = true), with the bf16 hi/lo planes,
// the per-CTA column partial sums and the non-zero flag of every row.  Block (32, 8): lanes over columns, 8 row lanes;
// row lane y owns the shared partial sums s[y][:], so the partials need no atomics.
// ------------------------------------------------------------------------------------------------
struct MaskRowsParams {
  const float* a;          // gather: the source logits [*, C]; merge: the anchor probabilities [*, qa]
  const int32_t* rows;     // gather: source row of every output row
  const float* b;          // merge: the matched subnet's probabilities [*, qb]
  const int32_t* cell_a;   // merge: cell → anchor row / subnet row (−1 = none)
  const int32_t* cell_b;
  const int32_t* lin;      // merge: cell of every output row
  const int32_t* a_col;    // merge: anchor column of output column j
  const int32_t* b_col;    // merge: subnet column averaged into output column j (−1 = none)
  const uint8_t* gate;     // merge: cell → occupancy gate (NULL = none)
  int qa, qb;
  float w, w1;             // merge: the running-average weight i and i + 1
  int64_t n;
  int C, Cp;               // output columns, plane columns (C rounded up to 16)
  int64_t chunk;           // rows per CTA
  float* out;
  __nv_bfloat16* hi;
  __nv_bfloat16* lo;
  float* part;             // [gridDim.x, C] or NULL
  uint8_t* nz;
};

template <bool MERGE>
__global__ void __launch_bounds__(256) k_mask_rows(const __grid_constant__ MaskRowsParams p) {
  extern __shared__ float s_part[];                         // [8][C]
  const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * 32 + tx;
  if (p.part)
    for (int c = tid; c < 8 * p.C; c += 256) s_part[c] = 0.f;
  __syncthreads();
  const int64_t r0 = blockIdx.x * p.chunk, r1 = min(p.n, r0 + p.chunk);
  float* my = s_part + ty * p.C;
  for (int64_t r = r0 + ty; r < r1; r += 8) {
    int64_t ra = -1, rb = -1;
    float g = 1.f;
    if (MERGE) {
      const int cell = __ldg(p.lin + r);
      ra = __ldg(p.cell_a + cell);
      rb = p.cell_b ? __ldg(p.cell_b + cell) : -1;
      if (p.gate) g = (float)__ldg(p.gate + cell);
    } else {
      ra = __ldg(p.rows + r);
    }
    bool nz = false;
#pragma unroll 1
    for (int c = tx; c < p.Cp; c += 32) {
      float v = 0.f;
      if (c < p.C) {
        if (MERGE) {
          const float a = ra >= 0 ? __ldg(p.a + ra * p.qa + __ldg(p.a_col + c)) : 0.f;
          const int bc = p.b_col ? __ldg(p.b_col + c) : -1;
          if (bc >= 0) {                                     // b may be NULL when the subnet has no row at all
            const float b = rb >= 0 ? __ldg(p.b + rb * p.qb + bc) : 0.f;
            v = __fdiv_rn(__fadd_rn(__fmul_rn(a, p.w), b), p.w1);   // (a·i + b) / (i + 1)
          } else {
            v = a;
          }
          if (p.gate) v = __fmul_rn(v, g);
        } else {
          const float x = __ldg(p.a + ra * p.C + c);
          v = __frcp_rn(__fadd_rn(1.f, expf(-x)));             // 1 / (1 + e^-x), correctly rounded
        }
        if (p.out) p.out[r * p.C + c] = v;
        if (p.part) my[c] += v;
        nz = nz || v != 0.f;
      }
      if (p.hi) {
        const __nv_bfloat16 h = __float2bfloat16_rn(v);
        p.hi[r * p.Cp + c] = h;
        if (p.lo) p.lo[r * p.Cp + c] = __float2bfloat16_rn(v - __bfloat162float(h));
      }
    }
    nz = __any_sync(0xffffffffu, nz);
    if (p.nz && tx == 0) p.nz[r] = nz;
  }
  if (p.part) {
    __syncthreads();
    for (int c = tid; c < p.C; c += 256) {
      float acc = 0.f;
#pragma unroll
      for (int y = 0; y < 8; ++y) acc += s_part[y * p.C + c];
      p.part[(int64_t)blockIdx.x * p.C + c] = acc;
    }
  }
}

__global__ void k_colsum_reduce(const float* __restrict__ part, int G, int C, float* __restrict__ colsum) {
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < C; c += gridDim.x * blockDim.x) {
    float acc = 0.f;
    for (int g = 0; g < G; ++g) acc += __ldg(part + (int64_t)g * C + c);
    colsum[c] = acc;
  }
}

// softmax over the K channels of gathered rows (semantic logits); one warp per row
__global__ void k_softmax_rows(const float* __restrict__ src, const int32_t* __restrict__ rows, int64_t n, int K,
                               float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t w0 = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = w0; r < n; r += nw) {
    const float* x = src + (int64_t)__ldg(rows + r) * K;
    float m = -INFINITY;
    for (int c = lane; c < K; c += 32) m = fmaxf(m, __ldg(x + c));
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, d));
    float s = 0.f;
    for (int c = lane; c < K; c += 32) s += expf(__fsub_rn(__ldg(x + c), m));
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
    for (int c = lane; c < K; c += 32) out[r * K + c] = __fdiv_rn(expf(__fsub_rn(__ldg(x + c), m)), s);
  }
}

// ------------------------------------------------------------------------------------------------
// soft IoU from the intersections, with the threshold gate (utils.py:153-198, ensembler.py:78-86)
// ------------------------------------------------------------------------------------------------
__global__ void k_soft_iou(const float* __restrict__ inter, int Q, int64_t pitch, const float* __restrict__ sa,
                           const float* __restrict__ sb, float thr, float* __restrict__ gated) {
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < Q * Q; e += gridDim.x * blockDim.x) {
    const int qa = e / Q, qb = e - qa * Q;
    const float in = __ldg(inter + qa * pitch + qb);
    const float un = __fsub_rn(__fadd_rn(__ldg(sa + qa), __ldg(sb + qb)), in);
    const float iou = un != 0.f ? __fdiv_rn(in, fmaxf(un, 1e-30f)) : 0.f;
    gated[e] = iou > thr ? iou : __fmul_rn(iou, 0.f);
  }
}

// ------------------------------------------------------------------------------------------------
// semantic ensemble (ensembler.py:160-187 + net_panoptic_sparse.py:278-294 max_prob confidence)
// ------------------------------------------------------------------------------------------------
__global__ void k_sem_ensemble(const __grid_constant__ SemParams p, const int32_t* __restrict__ lin, int64_t n, int K,
                               int32_t* __restrict__ pred, float* __restrict__ conf, uint8_t* __restrict__ gate) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int cell = __ldg(lin + i);
    int64_t r[kMaxSubnets];
    sem_rows_at(p, cell, r);
    float best = -INFINITY;
    int arg = 0;
    for (int c = 0; c < K; ++c) {
      const float mean = sem_mean_prob(p, r, K, c);
      if (mean > best) {
        best = mean;
        arg = c;
      }
    }
    pred[i] = arg;
    conf[i] = best;
    if (gate) gate[cell] = arg != 0;
  }
}

// ------------------------------------------------------------------------------------------------
// panoptic inference (helper.py:135-263)
// ------------------------------------------------------------------------------------------------
// per query: class probability and label = max / first argmax over the K1 classes; kept when the label is neither the
// empty class 0 nor the dustbin K1 − 1 and the probability exceeds mask_thr
__device__ __forceinline__ bool query_kept(const float* __restrict__ qp, int q, int K1, float mask_thr, float& prob,
                                           int& label) {
  prob = __ldg(qp + (int64_t)q * K1);
  label = 0;
  for (int c = 1; c < K1; ++c) {
    const float v = __ldg(qp + (int64_t)q * K1 + c);
    if (v > prob) {
      prob = v;
      label = c;
    }
  }
  return label != 0 && label != K1 - 1 && prob > mask_thr;
}

// one warp per voxel; the kept-query list and class probabilities are built in shared memory by every CTA
__global__ void __launch_bounds__(256) k_panoptic_pass1(const float* __restrict__ probs, int64_t n, int Q,
                                                        const float* __restrict__ qp, int K1, float mask_thr,
                                                        float vox_thr, int32_t* __restrict__ win,
                                                        float* __restrict__ m_win, float* __restrict__ m_sum,
                                                        float* __restrict__ c_sum, int32_t* __restrict__ areas) {
  extern __shared__ int s_mem[];
  int* s_q = s_mem;                                            // [Q] kept query ids
  float* s_p = reinterpret_cast<float*>(s_mem + Q);            // [Q] their class probabilities
  int* s_orig = s_mem + 2 * Q;                                 // [Q] original_area by query id
  int* s_area = s_mem + 3 * Q;                                 // [Q] mask_area by query id
  __shared__ int s_kq;
  __shared__ int s_warp[8];
  // kept-query list in ascending order: every thread tests its queries, a block-wide ballot prefix places them
  if (threadIdx.x == 0) s_kq = 0;
  __syncthreads();
  for (int q0 = 0; q0 < Q; q0 += blockDim.x) {
    const int q = q0 + threadIdx.x;
    float pr = 0.f;
    int lb;
    const bool kept = q < Q && query_kept(qp, q, K1, mask_thr, pr, lb);
    if (q < Q) s_orig[q] = s_area[q] = 0;
    const unsigned bal = __ballot_sync(0xffffffffu, kept);
    const int w = threadIdx.x >> 5, ln = threadIdx.x & 31;
    if (ln == 0) s_warp[w] = __popc(bal);
    __syncthreads();
    int pos = s_kq + __popc(bal & ((1u << ln) - 1));
    for (int v = 0; v < w; ++v) pos += s_warp[v];
    if (kept) {
      s_q[pos] = q;
      s_p[pos] = pr;
    }
    __syncthreads();
    if (threadIdx.x == 0)
      for (int v = 0; v < 8; ++v) s_kq += s_warp[v];
    __syncthreads();
  }
  const int kq = s_kq;
  const int lane = threadIdx.x & 31;
  const int64_t w0 = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = w0; r < n; r += nw) {
    const float* row = probs + r * Q;
    float best = -INFINITY, bm = 0.f, sum = 0.f, csum = 0.f;
    int bk = 0x7fffffff;
    for (int k = lane; k < kq; k += 32) {
      const int q = s_q[k];
      const float m = __ldg(row + q);
      const float cmb = __fmul_rn(s_p[k], m);
      if (cmb > best) {                                         // ascending k per lane: the first maximum stays
        best = cmb;
        bk = k;
        bm = m;
      }
      sum = __fadd_rn(sum, m);
      csum = __fadd_rn(csum, cmb);
      if (m >= vox_thr) atomicAdd(s_orig + q, 1);
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, d), om = __shfl_xor_sync(0xffffffffu, bm, d);
      const int ok = __shfl_xor_sync(0xffffffffu, bk, d);
      if (ob > best || (ob == best && ok < bk)) {              // ties: the lowest filtered index wins
        best = ob;
        bk = ok;
        bm = om;
      }
      sum = __fadd_rn(sum, __shfl_xor_sync(0xffffffffu, sum, d));
      csum = __fadd_rn(csum, __shfl_xor_sync(0xffffffffu, csum, d));
    }
    if (lane == 0) {
      if (kq == 0) {
        win[r] = -1;
        m_win[r] = 0.f;
      } else {
        const int q = s_q[bk];                                  // kq > 0 and finite probabilities: bk < kq
        const bool strong = bm >= vox_thr;
        if (strong) atomicAdd(s_area + q, 1);
        win[r] = (q << 1) | (int)strong;
        m_win[r] = bm;
      }
      m_sum[r] = sum;
      if (c_sum) c_sum[r] = csum;
    }
  }
  __syncthreads();
  for (int q = threadIdx.x; q < Q; q += blockDim.x) {
    if (s_orig[q]) atomicAdd(areas + Q + q, s_orig[q]);        // integer counts: exact in any order
    if (s_area[q]) atomicAdd(areas + q, s_area[q]);
  }
}

// the sequential segment walk of helper.py:171-250 over the kept queries in ascending order; one thread
__global__ void k_panoptic_segments(const float* __restrict__ qp, int Q, int K1, float mask_thr, double overlap_thr,
                                    unsigned long long thing_mask, const int32_t* __restrict__ areas,
                                    int32_t* __restrict__ seg_of, int32_t* __restrict__ cls_of,
                                    int32_t* __restrict__ records, int32_t* __restrict__ kept) {
  __shared__ int stuff_id[64];                                 // segment id of every stuff class seen so far
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  for (int c = 0; c < 64; ++c) stuff_id[c] = 0;
  int cur = 0, kq = 0;
  for (int q = 0; q < Q; ++q) {
    seg_of[q] = 0;
    cls_of[q] = 0;
    float pr;
    int lb;
    if (!query_kept(qp, q, K1, mask_thr, pr, lb)) continue;
    if (kept) kept[1 + kq] = q;
    ++kq;
    const int ma = areas[q], oa = areas[Q + q];
    if (!(ma > 0 && oa > 0) || (double)ma / (double)oa < overlap_thr) continue;
    const bool isthing = (thing_mask >> lb) & 1ull;             // lb < K1 - 1 <= 64
    if (!isthing && stuff_id[lb]) {                 // merged stuff: the panoptic id only (helper.py:243-245)
      seg_of[q] = stuff_id[lb];
      cls_of[q] = -1;
      continue;
    }
    if (!isthing) stuff_id[lb] = cur + 1;
    ++cur;
    seg_of[q] = cur;
    cls_of[q] = lb;
    int32_t* rec = records + 1 + 4 * (cur - 1);
    rec[0] = q;
    rec[1] = lb;
    rec[2] = __float_as_int(pr);
    rec[3] = isthing;
  }
  records[0] = cur;
  if (kept) kept[0] = kq;
}

__global__ void k_panoptic_pass2(const int32_t* __restrict__ win, const float* __restrict__ m_win,
                                 const float* __restrict__ m_sum, int64_t n, const int32_t* __restrict__ seg_of,
                                 const int32_t* __restrict__ cls_of, int32_t* __restrict__ pan, int32_t* __restrict__ sem,
                                 float* __restrict__ conf) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int w = __ldg(win + i);
    int p = 0, s = 0;
    float cf = 0.f;
    if (w >= 0 && (w & 1)) {
      const int q = w >> 1, sg = __ldg(seg_of + q), cl = __ldg(cls_of + q);
      if (sg > 0) {
        p = sg;
        if (cl > 0) {
          s = cl;
          cf = __fdiv_rn(__ldg(m_win + i), __fadd_rn(__ldg(m_sum + i), 1e-8f));
        }
      }
    }
    pan[i] = p;
    sem[i] = s;
    conf[i] = cf;
  }
}

// ------------------------------------------------------------------------------------------------
// dense volumes of panoptic_inference (helper.py:206-281): rows → channel-first [C, X, Y, Z] at coord − min_c
// ------------------------------------------------------------------------------------------------
struct PanopticDenseParams {
  const int32_t* coords;                 // [n, 4] (batch, x, y, z)
  int64_t n;
  int min_c[3];
  int X, Y, Z;
  const int32_t* pan_row;                // pass 2
  const int32_t* sem_row;
  const float* conf_row;
  const int32_t* win;                    // pass 1
  const float* m_win;
  const float* c_sum;
  const float* qp;                       // [Q, K1]
  int K1;
  const float* probs;                    // [n, Q]
  int Q;
  const int32_t* kept;                   // [kq]: the query of every kept column, ascending
  int kq;
  int32_t* pan;                          // [X, Y, Z]
  int32_t* sem;
  float* conf;
  float* ins;
  float* vox;
  float* all;                            // [kq, X, Y, Z]
  int32_t* err;
};

// one thread per row, so rows in ascending cell order write every plane coalesced; the volumes are zeroed by the caller
__global__ void k_panoptic_dense(const __grid_constant__ PanopticDenseParams p) {
  const int64_t cells = (int64_t)p.X * p.Y * p.Z;
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < p.n; r += (int64_t)gridDim.x * blockDim.x) {
    const int32_t* c = p.coords + 4 * r;
    const int x = __ldg(c + 1) - p.min_c[0], y = __ldg(c + 2) - p.min_c[1], z = __ldg(c + 3) - p.min_c[2];
    if (__ldg(c) != 0 || x < 0 || x >= p.X || y < 0 || y >= p.Y || z < 0 || z >= p.Z) {
      *p.err = 1;
      continue;
    }
    const int64_t cell = ((int64_t)x * p.Y + y) * p.Z + z;
    const int s = __ldg(p.sem_row + r);
    p.pan[cell] = __ldg(p.pan_row + r);
    p.sem[cell] = s;
    p.conf[cell] = __ldg(p.conf_row + r);
    if (s == 0) continue;     // not painted by a segment of its own: class 0, merged stuff or no segment (all stay 0)
    const int q = __ldg(p.win + r) >> 1;
    float pr;
    int lb;
    query_kept(p.qp, q, p.K1, 0.f, pr, lb);
    p.ins[cell] = pr;
    // max_k(c_k / Σc) = max_k(c_k) / Σc: one rounding, monotone; the winner's c_k is pass 1's product
    p.vox[cell] = __fdiv_rn(__fmul_rn(pr, __ldg(p.m_win + r)), __ldg(p.c_sum + r));
    const float* row = p.probs + r * p.Q;
    for (int k = 0; k < p.kq; ++k) p.all[k * cells + cell] = __ldg(row + __ldg(p.kept + k));
  }
}

// ------------------------------------------------------------------------------------------------
// dense class distributions of ensemble_sem_compl (ensembler.py:159-187): one thread per cell, a loop over channels
// ------------------------------------------------------------------------------------------------
struct SemDenseOut {
  float* sub[kMaxSubnets];   // [K, cells] of subnet m: its softmax row, one-hot class 0 where it has none (NULL = skip)
  float* ens;                // [K, cells] the mean over the subnets (NULL = skip)
  uint8_t* gate;             // [cells] argmax of ens != 0 (NULL = skip)
};

__global__ void k_sem_dense(const __grid_constant__ SemParams p, const __grid_constant__ SemDenseOut o, int64_t cells,
                            int K) {
  for (int64_t cell = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; cell < cells;
       cell += (int64_t)gridDim.x * blockDim.x) {
    int64_t r[kMaxSubnets];
    sem_rows_at(p, cell, r);
#pragma unroll
    for (int m = 0; m < kMaxSubnets; ++m) {      // unrolled: r[] stays in registers
      if (m >= p.M || !o.sub[m]) continue;
      for (int c = 0; c < K; ++c)
        o.sub[m][c * cells + cell] = r[m] >= 0 ? __ldg(p.prob[m] + r[m] * K + c) : (c == 0 ? 1.f : 0.f);
    }
    if (!o.ens && !o.gate) continue;
    float best = -INFINITY;
    int arg = 0;
    for (int c = 0; c < K; ++c) {
      const float v = sem_mean_prob(p, r, K, c);       // the value k_sem_ensemble ranks, so the gates agree
      if (o.ens) o.ens[c * cells + cell] = v;
      if (v > best) {                                  // first maximum, as torch.argmax
        best = v;
        arg = c;
      }
    }
    if (o.gate) o.gate[cell] = arg != 0;
  }
}

// the occupancy gate of ensembler.py:102-105 from a given dense distribution [K, cells]: first argmax != 0
__global__ void k_class_gate(const float* __restrict__ dense, int64_t cells, int K, uint8_t* __restrict__ gate) {
  for (int64_t cell = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; cell < cells;
       cell += (int64_t)gridDim.x * blockDim.x) {
    float best = -INFINITY;
    int arg = 0;
    for (int c = 0; c < K; ++c) {
      const float v = __ldg(dense + c * cells + cell);
      if (v > best) {
        best = v;
        arg = c;
      }
    }
    gate[cell] = arg != 0;
  }
}

}  // namespace

extern "C" int pasco_pose_lookup(const uint64_t* table_keys, const int32_t* table_vals, int64_t capacity,
                                 const float T[12], int32_t X, int32_t Y, int32_t Z, int32_t* cell_row,
                                 uint8_t* cell_mask, pasco_stream_t s) {
  PASCO_CHECK_ARG(capacity > 0 && (capacity & (capacity - 1)) == 0, "pasco_pose_lookup: capacity must be a power of two");
  PASCO_CHECK_ARG(X > 0 && Y > 0 && Z > 0, "pasco_pose_lookup: empty grid");
  Pose P;
  for (int i = 0; i < 12; ++i) P.t[i] = T[i];
  const int64_t cells = (int64_t)X * Y * Z;
  k_pose_lookup<<<grid_for(cells, 256), 256, 0, (cudaStream_t)s>>>(table_keys, table_vals, (uint32_t)(capacity - 1), P, X,
                                                                   Y, Z, cell_row, cell_mask);
  PASCO_CHECK_LAUNCH("pasco_pose_lookup");
  return 0;
}

extern "C" int pasco_cell_mask_or(const int32_t* cell_row, int64_t n, uint8_t* mask, pasco_stream_t s) {
  if (n == 0) return 0;
  k_cell_mask_or<<<grid_for(n, 256), 256, 0, (cudaStream_t)s>>>(cell_row, n, mask);
  PASCO_CHECK_LAUNCH("pasco_cell_mask_or");
  return 0;
}

extern "C" int pasco_lookup_rows(const int32_t* cell_row, const int32_t* lin, int64_t n, int32_t* out, pasco_stream_t s) {
  if (n == 0) return 0;
  k_lookup_rows<<<grid_for(n, 256), 256, 0, (cudaStream_t)s>>>(cell_row, lin, n, out);
  PASCO_CHECK_LAUNCH("pasco_lookup_rows");
  return 0;
}

extern "C" int pasco_box_cells(const int32_t* coords, int64_t n, const int32_t lo[3], const int32_t hi[3], int32_t X,
                               int32_t Y, int32_t Z, int32_t* cell_row, uint8_t* cell_mask, int32_t* counts,
                               pasco_stream_t s) {
  PASCO_CHECK_ARG(X > 0 && Y > 0 && Z > 0, "pasco_box_cells: empty box");
  PASCO_CHECK_ARG((int64_t)X * Y * Z <= INT32_MAX, "pasco_box_cells: %d x %d x %d cells exceed the int32 cell maps", X, Y, Z);
  PASCO_CHECK_ARG(n <= INT32_MAX, "pasco_box_cells: %lld rows exceed the int32 cell map", (long long)n);
  BoxBounds b;
  const int32_t size[3] = {X, Y, Z};
  for (int d = 0; d < 3; ++d) {
    PASCO_CHECK_ARG((int64_t)hi[d] - lo[d] < size[d], "pasco_box_cells: bounds [%d, %d] exceed the box's %d cells on axis %d",
                    lo[d], hi[d], size[d], d);
    b.lo[d] = lo[d];
    b.hi[d] = hi[d];
  }
  if (n == 0) return 0;
  k_box_cells<<<grid_for(n, 256), 256, 0, (cudaStream_t)s>>>(coords, n, b, X, Y, Z, cell_row, cell_mask, counts);
  PASCO_CHECK_LAUNCH("pasco_box_cells");
  return 0;
}

// the CTA count of the mask-row kernels: a function of n alone on a given device, so the partial sums are too
static int mask_rows_grid(int64_t n, int64_t* chunk) {
  int64_t g = (n + 63) / 64;
  const int64_t cap = 2 * (int64_t)num_sms();
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  *chunk = (n + g - 1) / g;
  return (int)g;
}

static int mask_rows_launch(const char* name, MaskRowsParams& p, bool merge, float* colsum, cudaStream_t st) {
  PASCO_CHECK_ARG(p.C >= 1 && p.Cp >= p.C && (p.hi == nullptr || p.Cp % 16 == 0), "%s: bad column counts", name);
  PASCO_CHECK_ARG(8 * (int64_t)p.C * 4 <= 200 * 1024, "%s: %d columns exceed the shared-memory partial sums", name, p.C);
  if (p.n == 0) {
    if (colsum) cudaMemsetAsync(colsum, 0, sizeof(float) * p.C, st);
    PASCO_CHECK_LAUNCH(name);
    return 0;
  }
  const int G = mask_rows_grid(p.n, &p.chunk);
  float* part = nullptr;
  if (colsum) {
    cudaError_t e = ws_alloc((void**)&part, sizeof(float) * (size_t)G * p.C, st);
    if (e != cudaSuccess) {
      set_error("%s: workspace allocation failed: %s", name, cudaGetErrorString(e));
      return -1;
    }
  }
  p.part = part;
  const size_t smem = colsum ? sizeof(float) * 8 * p.C : 0;
  if (merge) {
    cudaFuncSetAttribute(k_mask_rows<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    k_mask_rows<true><<<G, dim3(32, 8), smem, st>>>(p);
  } else {
    cudaFuncSetAttribute(k_mask_rows<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    k_mask_rows<false><<<G, dim3(32, 8), smem, st>>>(p);
  }
  if (colsum) {
    k_colsum_reduce<<<(p.C + 127) / 128, 128, 0, st>>>(part, G, p.C, colsum);
    cudaFreeAsync(part, st);
  }
  PASCO_CHECK_LAUNCH(name);
  return 0;
}

extern "C" int pasco_mask_rows_sigmoid(const float* logits, const int32_t* rows, int64_t n, int32_t Q, float* out,
                                       void* hi, void* lo, int32_t Qp, float* colsum, uint8_t* nonzero,
                                       pasco_stream_t s) {
  MaskRowsParams p = {};
  p.a = logits;
  p.rows = rows;
  p.n = n;
  p.C = Q;
  p.Cp = hi ? Qp : Q;
  p.out = out;
  p.hi = (__nv_bfloat16*)hi;
  p.lo = (__nv_bfloat16*)lo;
  p.nz = nonzero;
  return mask_rows_launch("pasco_mask_rows_sigmoid", p, false, colsum, (cudaStream_t)s);
}

extern "C" int pasco_mask_merge(const float* a, const int32_t* cell_a, int32_t qa, const float* b, const int32_t* cell_b,
                                int32_t qb, const int32_t* lin, int64_t n, const int32_t* a_col, const int32_t* b_col,
                                int32_t q_out, int32_t weight, const uint8_t* gate, float* out, void* hi, void* lo,
                                int32_t Qp, float* colsum, uint8_t* nonzero, pasco_stream_t s) {
  PASCO_CHECK_ARG(b_col == nullptr || cell_b, "pasco_mask_merge: a subnet's columns need its cell map");
  MaskRowsParams p = {};
  p.a = a;
  p.cell_a = cell_a;
  p.qa = qa;
  p.b = b;
  p.cell_b = cell_b;
  p.qb = qb;
  p.lin = lin;
  p.a_col = a_col;
  p.b_col = b_col;
  p.gate = gate;
  p.w = (float)weight;
  p.w1 = (float)(weight + 1);
  p.n = n;
  p.C = q_out;
  p.Cp = hi ? Qp : q_out;
  p.out = out;
  p.hi = (__nv_bfloat16*)hi;
  p.lo = (__nv_bfloat16*)lo;
  p.nz = nonzero;
  return mask_rows_launch("pasco_mask_merge", p, true, colsum, (cudaStream_t)s);
}

extern "C" int pasco_softmax_rows(const float* logits, const int32_t* rows, int64_t n, int32_t K, float* out,
                                  pasco_stream_t s) {
  if (n == 0) return 0;
  k_softmax_rows<<<grid_for(n * 32, 256), 256, 0, (cudaStream_t)s>>>(logits, rows, n, K, out);
  PASCO_CHECK_LAUNCH("pasco_softmax_rows");
  return 0;
}

extern "C" int pasco_soft_iou(const float* inter, int32_t Q, int64_t pitch, const float* sum_a, const float* sum_b,
                              float threshold, float* gated, pasco_stream_t s) {
  if (Q == 0) return 0;
  k_soft_iou<<<grid_for((int64_t)Q * Q, 256), 256, 0, (cudaStream_t)s>>>(inter, Q, pitch, sum_a, sum_b, threshold, gated);
  PASCO_CHECK_LAUNCH("pasco_soft_iou");
  return 0;
}

extern "C" int pasco_sem_ensemble(int32_t M, const float* const probs[], const int32_t* const cell_rows[],
                                  const int32_t* lin, int64_t n, int32_t K, int32_t* pred, float* conf, uint8_t* gate,
                                  pasco_stream_t s) {
  PASCO_CHECK_ARG(M >= 1 && M <= kMaxSubnets, "pasco_sem_ensemble: 1 <= M <= %d subnets (got %d)", kMaxSubnets, M);
  if (n == 0) return 0;
  SemParams p = {};
  p.M = M;
  for (int m = 0; m < M; ++m) {
    p.prob[m] = probs[m];
    p.cell_row[m] = cell_rows[m];
  }
  k_sem_ensemble<<<grid_for(n, 256), 256, 0, (cudaStream_t)s>>>(p, lin, n, K, pred, conf, gate);
  PASCO_CHECK_LAUNCH("pasco_sem_ensemble");
  return 0;
}

extern "C" int pasco_panoptic_pass1(const float* probs, int64_t n, int32_t Q, const float* query_probs, int32_t K1,
                                    float object_mask_threshold, float vox_occ_threshold, int32_t* win, float* m_win,
                                    float* m_sum, float* c_sum, int32_t* areas, pasco_stream_t s) {
  PASCO_CHECK_ARG(Q >= 1 && Q <= 8192 && K1 >= 2, "pasco_panoptic_pass1: 1 <= Q <= 8192 queries, K1 >= 2 classes");
  if (n == 0) return 0;
  const size_t smem = sizeof(int) * 4 * Q;
  cudaFuncSetAttribute(k_panoptic_pass1, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  k_panoptic_pass1<<<grid_for(n * 32, 256, 2), 256, smem, (cudaStream_t)s>>>(probs, n, Q, query_probs, K1,
                                                                            object_mask_threshold, vox_occ_threshold, win,
                                                                            m_win, m_sum, c_sum, areas);
  PASCO_CHECK_LAUNCH("pasco_panoptic_pass1");
  return 0;
}

extern "C" int pasco_panoptic_segments(const float* query_probs, int32_t Q, int32_t K1, float object_mask_threshold,
                                       double overlap_threshold, uint64_t thing_mask, const int32_t* areas,
                                       int32_t* seg_of, int32_t* cls_of, int32_t* records, int32_t* kept,
                                       pasco_stream_t s) {
  PASCO_CHECK_ARG(K1 >= 2 && K1 <= 65, "pasco_panoptic_segments: 2 <= K1 <= 65 classes (got %d)", K1);
  k_panoptic_segments<<<1, 32, 0, (cudaStream_t)s>>>(query_probs, Q, K1, object_mask_threshold, overlap_threshold,
                                                     (unsigned long long)thing_mask, areas, seg_of, cls_of, records, kept);
  PASCO_CHECK_LAUNCH("pasco_panoptic_segments");
  return 0;
}

extern "C" int pasco_panoptic_pass2(const int32_t* win, const float* m_win, const float* m_sum, int64_t n,
                                    const int32_t* seg_of, const int32_t* cls_of, int32_t* panoptic, int32_t* semantic,
                                    float* confidence, pasco_stream_t s) {
  if (n == 0) return 0;
  k_panoptic_pass2<<<grid_for(n, 256), 256, 0, (cudaStream_t)s>>>(win, m_win, m_sum, n, seg_of, cls_of, panoptic, semantic,
                                                                  confidence);
  PASCO_CHECK_LAUNCH("pasco_panoptic_pass2");
  return 0;
}

extern "C" int pasco_panoptic_dense(const int32_t* coords, int64_t n, const int32_t min_c[3], int32_t X, int32_t Y,
                                    int32_t Z, const int32_t* panoptic_rows, const int32_t* semantic_rows,
                                    const float* confidence_rows, const int32_t* win, const float* m_win,
                                    const float* c_sum, const float* query_probs, int32_t K1, const float* probs,
                                    int32_t Q, const int32_t* kept, int32_t kq, int32_t* panoptic, int32_t* semantic,
                                    float* confidence, float* ins_uncertainty, float* vox_uncertainty,
                                    float* all_mask_probs, int32_t* err_flag, pasco_stream_t s) {
  PASCO_CHECK_ARG(X > 0 && Y > 0 && Z > 0, "pasco_panoptic_dense: empty grid");
  PASCO_CHECK_ARG(kq >= 0 && kq <= Q && (kq == 0 || (kept && all_mask_probs)),
                  "pasco_panoptic_dense: 0 <= kq <= Q kept queries with their list and volume");
  PASCO_CHECK_ARG(err_flag != nullptr, "pasco_panoptic_dense: the error flag is required");
  if (n == 0) return 0;
  PanopticDenseParams p = {};
  p.coords = coords;
  p.n = n;
  for (int d = 0; d < 3; ++d) p.min_c[d] = min_c[d];
  p.X = X;
  p.Y = Y;
  p.Z = Z;
  p.pan_row = panoptic_rows;
  p.sem_row = semantic_rows;
  p.conf_row = confidence_rows;
  p.win = win;
  p.m_win = m_win;
  p.c_sum = c_sum;
  p.qp = query_probs;
  p.K1 = K1;
  p.probs = probs;
  p.Q = Q;
  p.kept = kept;
  p.kq = kq;
  p.pan = panoptic;
  p.sem = semantic;
  p.conf = confidence;
  p.ins = ins_uncertainty;
  p.vox = vox_uncertainty;
  p.all = all_mask_probs;
  p.err = err_flag;
  k_panoptic_dense<<<grid_for(n, 256), 256, 0, (cudaStream_t)s>>>(p);
  PASCO_CHECK_LAUNCH("pasco_panoptic_dense");
  return 0;
}

extern "C" int pasco_sem_dense(int32_t M, const float* const probs[], const int32_t* const cell_rows[], int64_t cells,
                               int32_t K, float* const subnet_out[], float* ensemble_out, uint8_t* gate,
                               pasco_stream_t s) {
  PASCO_CHECK_ARG(M >= 1 && M <= kMaxSubnets, "pasco_sem_dense: 1 <= M <= %d subnets (got %d)", kMaxSubnets, M);
  PASCO_CHECK_ARG(K >= 1, "pasco_sem_dense: K >= 1 classes");
  if (cells == 0) return 0;
  SemParams p = {};
  SemDenseOut o = {};
  p.M = M;
  for (int m = 0; m < M; ++m) {
    p.prob[m] = probs[m];
    p.cell_row[m] = cell_rows[m];
    o.sub[m] = subnet_out ? subnet_out[m] : nullptr;
  }
  o.ens = ensemble_out;
  o.gate = gate;
  k_sem_dense<<<grid_for(cells, 256), 256, 0, (cudaStream_t)s>>>(p, o, cells, K);
  PASCO_CHECK_LAUNCH("pasco_sem_dense");
  return 0;
}

extern "C" int pasco_class_gate(const float* dense, int64_t cells, int32_t K, uint8_t* gate, pasco_stream_t s) {
  PASCO_CHECK_ARG(K >= 1, "pasco_class_gate: K >= 1 classes");
  if (cells == 0) return 0;
  k_class_gate<<<grid_for(cells, 256), 256, 0, (cudaStream_t)s>>>(dense, cells, K, gate);
  PASCO_CHECK_LAUNCH("pasco_class_gate");
  return 0;
}
