// The reference decoder's glue between its convolutions (pasco/models/decoder_v3.py) on the rows.
//
//   pasco_completion_rows   predict_completion_sem_logit's per-row work for the M subnets in one pass over their softmax
//                           rows: torch's argmax, the keep mask, the cap weight p_max · w[cls] and the per-row vote count,
//                           plus every count the caller's branches and log lines need, in one small buffer.
//   pasco_topk_mask         torch.multinomial(w, k, replacement=False) = topk(w / q, k) with q ~ Exp(1) drawn by the
//                           caller: a radix select of the k-th largest w / q on its fp32 bit pattern (w / q >= 0, so the
//                           bits order as the values), then the keep mask, ties at the threshold taken by lowest row.
//   pasco_panop_crop        predict_panop's two or three successive prunes of one subnet and scale as one mask:
//                           argmax != 0 AND the row inside [min_C, max_C], with the reference's keep[:1000] rule when no
//                           row has a non-empty argmax.
//   pasco_mimo_batch        batch_sparse_tensor (pasco/models/utils.py:659-670) for all M subnets, and keep_pad.
//
// Integer counts use integer atomics, so every output is exact and independent of the order the atomics land in.
#include "common.cuh"

using namespace pasco;

namespace {

constexpr int kMaxSubnets = 8;
constexpr int kMaxClasses = 64;

struct RowPtrs {
  const float* p[kMaxSubnets];
};

// torch's max(-1) index over one row: the first maximal value; a NaN wins at its first index.  Returns the value too.
__device__ __forceinline__ int row_argmax(const float* __restrict__ row, int K, float& best) {
  best = __ldg(row);
  int bi = 0;
  if (best != best) return 0;
  for (int k = 1; k < K; ++k) {
    const float v = __ldg(row + k);
    if (v != v) {
      best = v;
      return k;
    }
    if (v > best) {
      best = v;
      bi = k;
    }
  }
  return bi;
}

// sum v over the block into *dst with one atomic per block (blockDim.x a multiple of 32, <= 1024)
__device__ __forceinline__ void block_add(int v, int32_t* dst) {
  __shared__ int part[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = __reduce_add_sync(0xFFFFFFFFu, v);
  __syncthreads();                          // part[] may still be read by a previous call
  if (lane == 0) part[warp] = v;
  __syncthreads();
  if (warp == 0) {
    int s = lane < (int)(blockDim.x >> 5) ? part[lane] : 0;
    s = __reduce_add_sync(0xFFFFFFFFu, s);
    if (lane == 0 && s) atomicAdd(dst, s);
  }
}

// counts: [0, M) kept rows per subnet, [M, 2M) labelled cells per subnet (k_labelled), [2M, 3M) rows whose weight is
// not a finite value >= 0, [3M] rows with at least one vote
__global__ void k_completion_rows(RowPtrs probs, int M, int64_t n, int K, const float* __restrict__ w,
                                  int32_t* __restrict__ cls, uint8_t* __restrict__ keep, float* __restrict__ weight,
                                  int32_t* __restrict__ votes, int32_t* __restrict__ counts) {
  const int64_t n_pad = (n + blockDim.x - 1) / blockDim.x * blockDim.x;     // every thread reaches the block sums
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n_pad; i += (int64_t)gridDim.x * blockDim.x) {
    const bool live = i < n;
    int v = 0;
#pragma unroll
    for (int m = 0; m < kMaxSubnets; ++m) {
      if (m >= M) break;
      int kept = 0, bad = 0;
      if (live) {
        float best;
        const int c = row_argmax(probs.p[m] + i * K, K, best);
        kept = c != 0;
        cls[m * n + i] = c;
        keep[m * n + i] = (uint8_t)kept;
        if (w) {
          const float x = __fmul_rn(best, __ldg(w + c));
          weight[m * n + i] = x;
          bad = !(x >= 0.f && x <= 3.402823466e38f);
        }
      }
      v += kept;
      block_add(kept, counts + m);
      if (w) block_add(bad, counts + 2 * M + m);
    }
    if (live) votes[i] = v;
    block_add(v > 0, counts + 3 * M);
  }
}

// (label != 0) & (label != 255) over M label volumes of n_label signed integers of `bytes` bytes each
struct LabelPtrs {
  const void* p[kMaxSubnets];
};

__device__ __forceinline__ int64_t label_at(const void* base, int bytes, int64_t i) {
  if (bytes == 1) return ((const uint8_t*)base)[i];
  if (bytes == 2) return ((const int16_t*)base)[i];
  if (bytes == 4) return ((const int32_t*)base)[i];
  return ((const int64_t*)base)[i];
}

__global__ void k_labelled(LabelPtrs labels, int M, int64_t n_label, int bytes, int32_t* __restrict__ counts) {
  const int64_t n_pad = (n_label + blockDim.x - 1) / blockDim.x * blockDim.x;
#pragma unroll
  for (int m = 0; m < kMaxSubnets; ++m) {
    if (m >= M) break;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n_pad; i += (int64_t)gridDim.x * blockDim.x) {
      int c = 0;
      if (i < n_label) {
        const int64_t v = label_at(labels.p[m], bytes, i);
        c = v != 0 && v != 255;
      }
      block_add(c, counts + M + m);
    }
  }
}

// ---- the cap: radix select of the k-th largest w / q -------------------------------------------------------------
// state int32: [0] prefix bits, [1] prefix mask, [2] rows still to take at or below the prefix, [3..259) histogram
__device__ __forceinline__ uint32_t ratio_bits(const float* __restrict__ w, const float* __restrict__ q, int64_t i) {
  return __float_as_uint(__fdiv_rn(__ldg(w + i), __ldg(q + i)));
}

__global__ void k_sel_init(int32_t* state, int32_t k) {
  const int t = threadIdx.x;
  if (t < 3) state[t] = t == 2 ? k : 0;
  state[3 + t] = 0;
}

__global__ void k_sel_hist(const float* __restrict__ w, const float* __restrict__ q, int64_t n, int shift,
                           int32_t* state) {
  __shared__ int hist[256];
  hist[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t prefix = (uint32_t)state[0], mask = (uint32_t)state[1];
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t b = ratio_bits(w, q, i);
    if ((b & mask) == prefix) atomicAdd(hist + ((b >> shift) & 255u), 1);
  }
  __syncthreads();
  const int h = hist[threadIdx.x];
  if (h) atomicAdd(state + 3 + threadIdx.x, h);
}

// one block of 256: the digit at `shift` of the k-th largest among the rows matching the prefix
__global__ void k_sel_pick(int32_t* state, int shift) {
  __shared__ int cum[256];
  const int t = threadIdx.x;
  const int h = state[3 + 255 - t];                // descending digits
  cum[t] = h;
  __syncthreads();
  for (int off = 1; off < 256; off <<= 1) {
    const int add = t >= off ? cum[t - off] : 0;
    __syncthreads();
    cum[t] += add;
    __syncthreads();
  }
  const int need = state[2];
  const int before = cum[t] - h;
  __syncthreads();
  if (before < need && cum[t] >= need) {          // exactly one thread: the digit holding the k-th largest
    state[0] |= (int32_t)((uint32_t)(255 - t) << shift);
    state[1] |= (int32_t)(255u << shift);
    state[2] = need - before;
  }
  state[3 + t] = 0;
}

// ties at the threshold: per-1024-row block counts, their exclusive scan, then the mask
__global__ void k_tie_counts(const float* __restrict__ w, const float* __restrict__ q, int64_t n,
                             const int32_t* __restrict__ state, int32_t* __restrict__ block_counts) {
  const int64_t i = blockIdx.x * 1024ll + threadIdx.x;
  const int tie = i < n && ratio_bits(w, q, i) == (uint32_t)state[0];
  __shared__ int part[32];
  const int s = __reduce_add_sync(0xFFFFFFFFu, tie);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    const int v = __reduce_add_sync(0xFFFFFFFFu, part[threadIdx.x]);
    if (threadIdx.x == 0) block_counts[blockIdx.x] = v;
  }
}

__global__ void k_tie_scan(int32_t* counts, int64_t nb) {        // in place, exclusive; one block of 1024
  __shared__ int buf[1024];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int64_t base = 0; base < nb; base += 1024) {
    const int64_t i = base + threadIdx.x;
    const int v = i < nb ? counts[i] : 0;
    buf[threadIdx.x] = v;
    __syncthreads();
    for (int off = 1; off < 1024; off <<= 1) {
      const int add = threadIdx.x >= off ? buf[threadIdx.x - off] : 0;
      __syncthreads();
      buf[threadIdx.x] += add;
      __syncthreads();
    }
    if (i < nb) counts[i] = carry + buf[threadIdx.x] - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry += buf[1023];
    __syncthreads();
  }
}

__global__ void k_topk_write(const float* __restrict__ w, const float* __restrict__ q, int64_t n,
                             const int32_t* __restrict__ state, const int32_t* __restrict__ offsets,
                             uint8_t* __restrict__ keep) {
  const int64_t i = blockIdx.x * 1024ll + threadIdx.x;
  const uint32_t thr = (uint32_t)state[0];
  const int take = state[2];
  const uint32_t b = i < n ? ratio_bits(w, q, i) : 0u;
  const int tie = i < n && b == thr;
  __shared__ int part[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned ballot = __ballot_sync(0xFFFFFFFFu, tie);
  if (lane == 0) part[warp] = __popc(ballot);
  __syncthreads();
  int before = offsets[blockIdx.x] + __popc(ballot & ((1u << lane) - 1));
  for (int j = 0; j < warp; ++j) before += part[j];
  if (i < n) keep[i] = (uint8_t)(b > thr || (tie && before < take));
}

// ---- predict_panop's crop -------------------------------------------------------------------------------------------
__device__ __forceinline__ bool in_box(const int4 c, const int32_t* __restrict__ box) {
  return c.y >= box[0] && c.z >= box[1] && c.w >= box[2] && c.y <= box[3] && c.z <= box[4] && c.w <= box[5];
}

// counts int32 [2]: rows with argmax != 0, rows kept
__global__ void k_crop(const float* __restrict__ logits, int64_t n, int K, const int4* __restrict__ coords,
                       const int32_t* __restrict__ box, uint8_t* __restrict__ mask, int32_t* __restrict__ counts) {
  const int64_t n_pad = (n + blockDim.x - 1) / blockDim.x * blockDim.x;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n_pad; i += (int64_t)gridDim.x * blockDim.x) {
    int c = 0, k = 0;
    if (i < n) {
      float best;
      c = row_argmax(logits + i * K, K, best) != 0;
      k = c && in_box(__ldg(coords + i), box);
      mask[i] = (uint8_t)k;
    }
    block_add(c, counts);
    block_add(k, counts + 1);
  }
}

// decoder_v3.py:415-417 then the box test: no row with a non-empty argmax → the first 1000 rows inside the box.  One
// block of 1024; a no-op when counts[0] != 0.
__global__ void k_crop_empty(int64_t n, const int4* __restrict__ coords, const int32_t* __restrict__ box,
                             uint8_t* __restrict__ mask, int32_t* __restrict__ counts) {
  if (counts[0] != 0) return;
  const int64_t i = threadIdx.x;
  int k = 0;
  if (i < 1000 && i < n) {
    k = in_box(__ldg(coords + i), box);
    mask[i] = (uint8_t)k;
  }
  const int s = __syncthreads_count(k);
  if (threadIdx.x == 0) counts[1] = s;
}

// ---- batch_sparse_tensor ---------------------------------------------------------------------------------------------
struct BatchArgs {
  const float* f[kMaxSubnets];
  const int4* c[kMaxSubnets];
  int64_t len[kMaxSubnets];
};

// one warp per (subnet, row): out_F [M][L][C], out_C [M][L][4], zero past the subnet's rows; keep_pad[m][r] = any
// feature or coordinate != 0 (utils.py:659-670 and decoder_v3.py:443-446)
__global__ void k_mimo_batch(BatchArgs a, int M, int64_t L, int C, float* __restrict__ out_F,
                             int4* __restrict__ out_C, uint8_t* __restrict__ keep_pad) {
  const int lane = threadIdx.x & 31;
  const int64_t total = (int64_t)M * L;
  for (int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; r < total;
       r += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    const int m = (int)(r / L);
    const int64_t row = r - (int64_t)m * L;
    const float* f = nullptr;
    const int4* c = nullptr;
    int64_t len = 0;
#pragma unroll
    for (int j = 0; j < kMaxSubnets; ++j)
      if (j == m) {
        f = a.f[j];
        c = a.c[j];
        len = a.len[j];
      }
    const bool real = row < len;
    bool any = false;
    for (int k = lane; k < C; k += 32) {
      const float v = real ? __ldg(f + row * C + k) : 0.f;
      out_F[r * C + k] = v;
      any |= v != 0.f;
    }
    int4 cc = make_int4(0, 0, 0, 0);
    if (real) cc = __ldg(c + row);
    if (lane == 0) out_C[r] = cc;
    any |= cc.x != 0 || cc.y != 0 || cc.z != 0 || cc.w != 0;
    const bool keep = __any_sync(0xFFFFFFFFu, any);
    if (keep_pad && lane == 0) keep_pad[r] = (uint8_t)keep;
  }
}

}  // namespace

extern "C" int pasco_completion_rows(const float* const* probs, int32_t M, int64_t n, int32_t K, const float* w,
                                     const void* const* labels, int64_t n_label, int32_t label_bytes, int32_t* cls,
                                     uint8_t* keep, float* weight, int32_t* votes, int32_t* counts, pasco_stream_t s) {
  PASCO_CHECK_ARG(M >= 1 && M <= kMaxSubnets && K >= 1 && K <= kMaxClasses && n >= 0 && n_label >= 0,
                  "pasco_completion_rows: need 1 <= M <= %d and 1 <= K <= %d (M=%d, K=%d)", kMaxSubnets, kMaxClasses,
                  M, K);
  PASCO_CHECK_ARG(label_bytes == 1 || label_bytes == 2 || label_bytes == 4 || label_bytes == 8,
                  "pasco_completion_rows: label_bytes must be 1, 2, 4 or 8");
  PASCO_CHECK_ARG(!w || weight, "pasco_completion_rows: w needs the weight output");
  cudaStream_t st = (cudaStream_t)s;
  RowPtrs p = {};
  LabelPtrs lp = {};
  for (int m = 0; m < M; ++m) {
    p.p[m] = probs[m];
    lp.p[m] = labels ? labels[m] : nullptr;
  }
  if (n > 0)
    k_completion_rows<<<grid_for(n, 256), 256, 0, st>>>(p, M, n, K, w, cls, keep, weight, votes, counts);
  if (labels && n_label > 0) k_labelled<<<grid_for(n_label, 256), 256, 0, st>>>(lp, M, n_label, label_bytes, counts);
  PASCO_CHECK_LAUNCH("pasco_completion_rows");
  return 0;
}

extern "C" int pasco_topk_mask(const float* w, const float* q, int64_t n, int64_t k, uint8_t* keep, pasco_stream_t s) {
  PASCO_CHECK_ARG(n > 0 && k >= 1 && k <= n && n < (1ll << 31), "pasco_topk_mask: need 1 <= k <= n < 2^31");
  cudaStream_t st = (cudaStream_t)s;
  const int64_t nb = (n + 1023) / 1024;
  void* ws = nullptr;
  if (ws_alloc(&ws, (size_t)(260 + nb) * sizeof(int32_t), st) != cudaSuccess) {
    set_error("pasco_topk_mask: workspace allocation failed");
    return -1;
  }
  int32_t* state = (int32_t*)ws;
  int32_t* blocks = state + 260;
  k_sel_init<<<1, 256, 0, st>>>(state, (int32_t)k);
  for (int shift = 24; shift >= 0; shift -= 8) {
    k_sel_hist<<<grid_for(n, 256), 256, 0, st>>>(w, q, n, shift, state);
    k_sel_pick<<<1, 256, 0, st>>>(state, shift);
  }
  k_tie_counts<<<(unsigned)nb, 1024, 0, st>>>(w, q, n, state, blocks);
  k_tie_scan<<<1, 1024, 0, st>>>(blocks, nb);
  k_topk_write<<<(unsigned)nb, 1024, 0, st>>>(w, q, n, state, blocks, keep);
  cudaFreeAsync(ws, st);
  PASCO_CHECK_LAUNCH("pasco_topk_mask");
  return 0;
}

extern "C" int pasco_panop_crop(const float* logits, int64_t n, int32_t K, const int32_t* coords, const int32_t* box,
                                uint8_t* mask, int32_t* counts, pasco_stream_t s) {
  PASCO_CHECK_ARG(K >= 1 && K <= kMaxClasses && n >= 0, "pasco_panop_crop: need 1 <= K <= %d (K=%d)", kMaxClasses,
                  K);
  cudaStream_t st = (cudaStream_t)s;
  if (n > 0) {
    k_crop<<<grid_for(n, 256), 256, 0, st>>>(logits, n, K, (const int4*)coords, box, mask, counts);
    k_crop_empty<<<1, 1024, 0, st>>>(n, (const int4*)coords, box, mask, counts);
  }
  PASCO_CHECK_LAUNCH("pasco_panop_crop");
  return 0;
}

extern "C" int pasco_mimo_batch(const float* const* feats, const int32_t* const* coords, const int64_t* lengths,
                                int32_t M, int64_t L, int32_t C, float* out_F, int32_t* out_C, uint8_t* keep_pad,
                                pasco_stream_t s) {
  PASCO_CHECK_ARG(M >= 1 && M <= kMaxSubnets && L >= 0 && C >= 1, "pasco_mimo_batch: need 1 <= M <= %d, C >= 1",
                  kMaxSubnets);
  BatchArgs a = {};
  for (int m = 0; m < M; ++m) {
    PASCO_CHECK_ARG(lengths[m] >= 0 && lengths[m] <= L, "pasco_mimo_batch: subnet %d has %lld rows > L = %lld", m,
                    (long long)lengths[m], (long long)L);
    a.f[m] = feats[m];
    a.c[m] = (const int4*)coords[m];
    a.len[m] = lengths[m];
  }
  if (L == 0) return 0;
  cudaStream_t st = (cudaStream_t)s;
  k_mimo_batch<<<grid_for((int64_t)M * L * 32, 256), 256, 0, st>>>(a, M, L, C, out_F, (int4*)out_C, keep_pad);
  PASCO_CHECK_LAUNCH("pasco_mimo_batch");
  return 0;
}
