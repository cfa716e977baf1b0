// The cross-attention mask of transformer_predictor_v2.py:220-289 (and line 164) built directly as the bit rows that
// xattn.cu reads, sm_90a.
//
//   mask[q, v] = NOT OR_{u in block_s(v)} (logit[u, q] > 0)        (sigmoid(x) > 0.5 max-pooled to the key's scale)
//   a query with all P keys masked attends everywhere                (line 164)
//
// The reference builds a dense [Q, X/s, Y/s, Z/s] volume, a bool [B·heads, Q, P] mask and an int64 row sum of it; the
// attention only ever needs Q·P bits.  Three passes, each touching no more than the logits once and the bits once:
//   k_mask_pool  one warp per scale-1 voxel: the predicate of 32 queries → one ballot word, OR-ed into the voxel's
//                stride-s parent (integer atomicOr: exact and independent of the order voxels arrive in);
//   k_mask_keys  one warp per (32 output words, 32 queries): each lane reads its key's parent word, 32 ballots turn
//                the [key][query] bits into [query][key] words (through shared memory, so the stores are coalesced);
//                a query with any unmasked key is marked in `seen`;
//   k_mask_clear the rows of unseen queries get their P real-key bits cleared.
#include "common.cuh"

using namespace pasco;

namespace {

constexpr unsigned kFull = 0xFFFFFFFFu;
constexpr int kWarps = 8;

__global__ void k_mask_pool(const float* __restrict__ logits, int64_t ld, int Q, const int32_t* __restrict__ rows,
                            int64_t n_child, const int32_t* __restrict__ parent_of, uint32_t* __restrict__ pooled) {
  const int lane = threadIdx.x & 31;
  const int QW = (Q + 31) >> 5;
  const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t u = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5); u < n_child; u += nwarps) {
    const int64_t row = rows ? __ldg(rows + u) : u;
    const int64_t parent = parent_of ? __ldg(parent_of + u) : u;
    const float* src = logits + row * ld;
    for (int w = 0; w < QW; ++w) {
      const int q = (w << 5) + lane;
      const unsigned word = __ballot_sync(kFull, q < Q && __ldg(src + q) > 0.f);
      if (lane == 0 && parent >= 0 && word) {
        if (parent_of)
          atomicOr(pooled + parent * QW + w, word);
        else
          pooled[parent * QW + w] = word;
      }
    }
  }
}

__global__ void __launch_bounds__(kWarps * 32) k_mask_keys(const uint32_t* __restrict__ pooled, int Q,
                                                             const int32_t* __restrict__ key_parent, int64_t P,
                                                             int64_t W, int32_t* __restrict__ seen,
                                                             uint32_t* __restrict__ mask) {
  __shared__ uint32_t tile[kWarps][32][33];                 // [warp][query][word]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int QW = (Q + 31) >> 5;
  const int64_t groups = (W + 31) >> 5;
  const int64_t task = blockIdx.x * (int64_t)kWarps + warp;   // (word group, query word), query word fastest
  if (task >= groups * QW) return;
  const int qw = (int)(task % QW);
  const int64_t w0 = (task / QW) << 5;
  uint32_t(*t)[33] = tile[warp];
  unsigned any = 0;                                          // lane i: query qw·32 + i has an unmasked key
  for (int j = 0; j < 32; ++j) {
    const int64_t key = ((w0 + j) << 5) + lane;
    const int32_t parent = key < P ? __ldg(key_parent + key) : -1;
    const uint32_t bits = parent >= 0 ? __ldg(pooled + (int64_t)parent * QW + qw) : 0u;
    for (int i = 0; i < 32; ++i) {
      const unsigned kept = __ballot_sync(kFull, (bits >> i) & 1u);
      if (lane == i) {
        t[i][j] = ~kept;
        any |= kept;
      }
    }
  }
  const int q_me = (qw << 5) + lane;
  if (any && q_me < Q) seen[q_me] = 1;                      // every writer stores the same value
  __syncwarp();
  const int64_t w = w0 + lane;
  for (int i = 0; i < 32; ++i) {
    const int q = (qw << 5) + i;
    if (q < Q && w < W) mask[(int64_t)q * W + w] = t[i][lane];
  }
}

__global__ void k_mask_clear(const int32_t* __restrict__ seen, int Q, int64_t P, int64_t W, uint32_t* __restrict__ mask) {
  const int64_t total = (int64_t)Q * W;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t q = e / W;
    if (__ldg(seen + q)) continue;
    const int64_t lo = (e - q * W) << 5;
    if (lo >= P) continue;                                   // padding words stay masked
    mask[e] = lo + 32 <= P ? 0u : ~((1u << (P - lo)) - 1u);  // the word holding key P − 1 keeps its padding bits
  }
}

}  // namespace

extern "C" int pasco_attn_mask_bits(const float* logits, int64_t ld, int32_t Q, const int32_t* rows, int64_t n_child,
                                    const int32_t* parent_of, int64_t n_parent, const int32_t* key_parent, int64_t P,
                                    uint32_t* pooled, int32_t* seen, uint32_t* mask, pasco_stream_t s) {
  PASCO_CHECK_ARG(Q >= 1 && ld >= Q && n_child >= 0 && n_parent >= 0 && P >= 0,
                  "pasco_attn_mask_bits: bad shape (Q %d, ld %lld, n_child %lld, n_parent %lld, P %lld)", Q,
                  (long long)ld, (long long)n_child, (long long)n_parent, (long long)P);
  PASCO_CHECK_ARG(parent_of || n_parent == n_child, "pasco_attn_mask_bits: identity parents need n_parent == n_child");
  if (P == 0) return 0;
  const cudaStream_t st = (cudaStream_t)s;
  const int64_t W = 2 * ((P + 63) / 64);
  const int QW = (Q + 31) / 32;
  if (n_child > 0)
    k_mask_pool<<<grid_for(n_child * 32, 256), 256, 0, st>>>(logits, ld, Q, rows, n_child, parent_of, pooled);
  const int64_t tasks = ((W + 31) / 32) * QW;
  k_mask_keys<<<(unsigned)((tasks + kWarps - 1) / kWarps), kWarps * 32, 0, st>>>(pooled, Q, key_parent, P, W, seen,
                                                                                 mask);
  k_mask_clear<<<grid_for((int64_t)Q * W, 256), 256, 0, st>>>(seen, Q, P, W, mask);
  PASCO_CHECK_LAUNCH("pasco_attn_mask_bits");
  return 0;
}
