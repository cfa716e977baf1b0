// Evaluation of PascoNet.predict's outputs against a scene's ground truth (sm_90a): the counting passes behind the
// reference's Net.evaluate_all (net_panoptic_sparse.py:650-765) — panoptic quality (panoptic_quality.py:175-261),
// completion and semantic IoU and their calibration (metrics.py:450-691), and the voxel calibration of
// UncertaintyMetrics.compute_ece_panop (metrics.py:98-165).  The row-form passes read PascoNet.predict's sparse rows
// (pasco_b200/metrics.py); the dense forms read the volumes the unmodified reference hands its evaluate_all
// (pasco_b200/hooks.py): channel-major class planes and [X, Y, Z] id / confidence volumes, row i = cell i.  They produce
// small tables (integer histograms, 16-slot calibration bins) that the host finishes; the dense forms also write the
// two volumes evaluate_all returns (its argmax and the ground-truth ids).
//
// Counts are integer atomics, exact in any order.  Floating-point sums are accumulated in double by one thread per
// row position of a CTA, added over the CTA's threads in thread order and over the CTAs in CTA order (k_part_reduce):
// no floating-point atomics, so two calls give the same bits.
#include "common.cuh"
#include "semantic.cuh"

using namespace pasco;

namespace {

constexpr int kSlots = 16;             // torchmetrics' 15 bins plus the slot of a confidence of exactly 1.0
constexpr int kBlock = 256;
constexpr int kSmemCap = 200 * 1024;

struct Bounds {
  float b[kSlots];                     // torch.linspace(0, 1, 16) in fp32
};

// torch.bucketize(conf, bounds, right=True) − 1: the number of boundaries <= conf, minus one; a confidence below 0 (or
// NaN) would be an invalid index for torch's scatter_add and is put into slot 0
__device__ __forceinline__ int conf_slot(const Bounds& B, float c) {
  int k = 0;
#pragma unroll
  for (int i = 0; i < kSlots; ++i) k += B.b[i] <= c;
  return max(k - 1, 0);
}

// ------------------------------------------------------------------------------------------------
// ground truth, once per scene (convert_mask_label_to_panoptic_output, panoptic_quality.py:357-390, and the unknown
// zeroing of net_panoptic_sparse.py:719-726): one thread per cell walks the mask stack in order, the last mask with a
// segment id wins; one ballot per warp and mask counts mask.sum() before any overwrite or zeroing
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBlock) k_eval_gt(const uint8_t* __restrict__ masks, int n_masks,
                                                     const int32_t* __restrict__ seg_of_mask,
                                                     const uint8_t* __restrict__ label, int64_t cells, int G, int K,
                                                     int32_t* __restrict__ gt_id, int32_t* __restrict__ mask_count,
                                                     int32_t* __restrict__ gt_area, int32_t* __restrict__ hist) {
  extern __shared__ int s_gt[];
  int* s_cnt = s_gt;                         // [n_masks]
  int* s_area = s_cnt + n_masks;             // [G + 1]
  int* s_hist = s_area + G + 1;              // [K + 1]: known cells per class, then labels >= K other than 255
  const int tot = n_masks + G + 1 + K + 1;
  for (int i = threadIdx.x; i < tot; i += blockDim.x) s_gt[i] = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  for (int64_t i0 = blockIdx.x * (int64_t)blockDim.x; i0 < cells; i0 += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = i0 + threadIdx.x;                        // i0 is uniform over the CTA: full-warp ballots
    const bool in = i < cells;
    int id = 0;
    for (int m = 0; m < n_masks; ++m) {
      const bool v = in && __ldg(masks + (int64_t)m * cells + i) != 0;
      const unsigned bal = __ballot_sync(0xffffffffu, v);
      if (lane == 0 && bal) atomicAdd(s_cnt + m, __popc(bal));
      const int sg = __ldg(seg_of_mask + m);
      if (v && sg > 0) id = sg;
    }
    if (in) {
      const int lab = __ldg(label + i);
      if (lab == 255) {
        id = 0;
      } else {
        atomicAdd(s_hist + min(lab, K), 1);
      }
      gt_id[i] = id;
      atomicAdd(s_area + id, 1);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n_masks; i += blockDim.x)
    if (s_cnt[i]) atomicAdd(mask_count + i, s_cnt[i]);
  for (int i = threadIdx.x; i <= G; i += blockDim.x)
    if (s_area[i]) atomicAdd(gt_area + i, s_area[i]);
  for (int i = threadIdx.x; i <= K; i += blockDim.x)
    if (s_hist[i]) atomicAdd(hist + i, s_hist[i]);
}

// ------------------------------------------------------------------------------------------------
// panoptic pairs, per entry (pq_compute_single_core's np.unique over gt_id * OFFSET + pred_id): for every known row
// with a predicted id, the predicted area and the (gt id, pred id) intersection; the table [G1, S1] lives in shared
// memory when it fits (SHARED) and in global memory otherwise.  pred_area[0] counts the rows whose cell lies outside
// [0, cells) and the predicted ids outside [0, S1).
// ------------------------------------------------------------------------------------------------
template <bool SHARED>
__global__ void __launch_bounds__(kBlock) k_eval_pairs(const int64_t* __restrict__ lin, const int32_t* __restrict__ pan,
                                                        int64_t n, const int32_t* __restrict__ gt_id,
                                                        const uint8_t* __restrict__ label, int64_t cells, int G1, int S1,
                                                        int32_t* __restrict__ pairs, int32_t* __restrict__ pred_area) {
  extern __shared__ int s_pairs[];
  const int tot = G1 * S1 + S1;
  int* tab = SHARED ? s_pairs : pairs;
  int* area = SHARED ? s_pairs + G1 * S1 : pred_area;
  if (SHARED) {
    for (int i = threadIdx.x; i < tot; i += blockDim.x) s_pairs[i] = 0;
    __syncthreads();
  }
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    const int64_t cell = __ldg(lin + r);
    const int p = __ldg(pan + r);
    if (cell < 0 || cell >= cells) {
      atomicAdd(area, 1);
      continue;
    }
    if (p == 0) continue;
    if (__ldg(label + cell) == 255) continue;                  // pred_panoptic_seg[unknown_mask] = 0
    if (p < 0 || p >= S1) {
      atomicAdd(area, 1);
      continue;
    }
    atomicAdd(tab + (int64_t)__ldg(gt_id + cell) * S1 + p, 1);
    atomicAdd(area + p, 1);
  }
  if (SHARED) {
    __syncthreads();
    for (int i = threadIdx.x; i < tot; i += blockDim.x) {
      const int v = s_pairs[i];
      if (v) atomicAdd(i < G1 * S1 ? pairs + i : pred_area + (i - G1 * S1), v);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// calibration slots: per CTA thread, a double accumulator per float column in shared memory ([cols][kBlock], owned
// by the thread: no atomics), added over the threads in order into the CTA's partial row
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void flush_partials(const double* s_acc, int cols, double* part) {
  __syncthreads();
  for (int c = threadIdx.x; c < cols; c += blockDim.x) {
    double a = 0.0;
    for (int t = 0; t < kBlock; ++t) a += s_acc[c * kBlock + t];
    part[(int64_t)blockIdx.x * cols + c] = a;
  }
}

// SSC, per entry (SSCMetrics.add_batch / add_batch_ece): over the entry's semantic rows at known cells, the K x K
// confusion counts (gt row, predicted column); per partition (0: predicted empty, 1: non-empty) and slot the count and
// the number of correct predictions; float columns: 2 x 16 confidence sums, then per partition Σ −log(p[target] +
// 1e-12) when the semantic rows are given (sem.M > 0).  pred_bad counts the rows whose cell lies outside [0, cells)
// and the known rows whose prediction or label lies outside [0, K).
struct SscParams {
  SemParams sem;
  const int64_t* lin;
  const int32_t* pred;
  const float* conf;
  int64_t n, chunk;
  const uint8_t* label;
  int64_t cells;
  int K;
  Bounds B;
  int32_t* confmat;        // [K * K]
  int32_t* cal;            // [2][2][16]: partition, (count, correct), slot
  int32_t* pred_bad;
  double* part;            // [grid][34]
};
constexpr int kSscCols = 2 * kSlots + 2;

__global__ void __launch_bounds__(kBlock) k_eval_ssc(const __grid_constant__ SscParams p) {
  extern __shared__ double s_acc[];                            // [kSscCols][kBlock]
  int* s_conf = reinterpret_cast<int*>(s_acc + kSscCols * kBlock);    // [K * K]
  int* s_cal = s_conf + p.K * p.K;                             // [64]
  __shared__ int s_bad;
  for (int i = threadIdx.x; i < kSscCols * kBlock; i += blockDim.x) s_acc[i] = 0.0;
  for (int i = threadIdx.x; i < p.K * p.K + 4 * kSlots; i += blockDim.x) s_conf[i] = 0;
  if (threadIdx.x == 0) s_bad = 0;
  __syncthreads();
  const int64_t r0 = blockIdx.x * p.chunk, r1 = min(p.n, r0 + p.chunk);
  double* my = s_acc + threadIdx.x;
  for (int64_t r = r0 + threadIdx.x; r < r1; r += kBlock) {
    const int64_t cell = __ldg(p.lin + r);
    if (cell < 0 || cell >= p.cells) {
      atomicAdd(&s_bad, 1);
      continue;
    }
    const int lab = __ldg(p.label + cell);
    if (lab == 255) continue;                                  // keep = target != 255; counted as (0, 0) by the host
    const int pr = __ldg(p.pred + r);
    if (pr < 0 || pr >= p.K || lab >= p.K) {
      atomicAdd(&s_bad, 1);
      continue;
    }
    const float c = __ldg(p.conf + r);
    const int part = pr != 0, slot = conf_slot(p.B, c);
    atomicAdd(s_conf + lab * p.K + pr, 1);
    atomicAdd(s_cal + part * 2 * kSlots + slot, 1);
    if (pr == lab) atomicAdd(s_cal + part * 2 * kSlots + kSlots + slot, 1);
    my[(part * kSlots + slot) * kBlock] += (double)c;
    if (p.sem.M > 0) {
      int64_t rows[kMaxSubnets];
      sem_rows_at(p.sem, cell, rows);
      const float pt = sem_mean_prob(p.sem, rows, p.K, lab);
      my[(2 * kSlots + part) * kBlock] += (double)(-logf(__fadd_rn(pt, 1e-12f)));
    }
  }
  flush_partials(s_acc, kSscCols, p.part);
  for (int i = threadIdx.x; i < p.K * p.K + 4 * kSlots; i += blockDim.x) {
    const int v = s_conf[i];
    if (v) atomicAdd(i < p.K * p.K ? p.confmat + i : p.cal + (i - p.K * p.K), v);
  }
  if (threadIdx.x == 0 && s_bad) atomicAdd(p.pred_bad, s_bad);
}

// voxel calibration, per entry (compute_ece_panop): rows whose cell has a gt id (known, covered) and a non-zero
// vox_confidence; correct when the row's predicted segment is matched to exactly that gt id (match[pred id], 0 =
// unmatched).  cal [2][16] (count, correct) per slot, float columns: 16 confidence sums.  Rows whose cell lies outside
// [0, cells) are skipped (the pair pass over the same rows reports them).
struct VoxParams {
  const int64_t* lin;
  const int32_t* pan;
  const float* conf;
  int64_t n, chunk;
  const int32_t* gt_id;
  int64_t cells;
  const int32_t* match;    // [S1]
  int S1;
  Bounds B;
  int32_t* cal;
  double* part;            // [grid][16]
};

__global__ void __launch_bounds__(kBlock) k_eval_vox(const __grid_constant__ VoxParams p) {
  extern __shared__ double s_acc[];                            // [kSlots][kBlock]
  __shared__ int s_cal[2 * kSlots];
  for (int i = threadIdx.x; i < kSlots * kBlock; i += blockDim.x) s_acc[i] = 0.0;
  if (threadIdx.x < 2 * kSlots) s_cal[threadIdx.x] = 0;
  __syncthreads();
  const int64_t r0 = blockIdx.x * p.chunk, r1 = min(p.n, r0 + p.chunk);
  double* my = s_acc + threadIdx.x;
  for (int64_t r = r0 + threadIdx.x; r < r1; r += kBlock) {
    const float c = __ldg(p.conf + r);
    if (c == 0.f) continue;
    const int64_t cell = __ldg(p.lin + r);
    if (cell < 0 || cell >= p.cells) continue;
    const int g = __ldg(p.gt_id + cell);
    if (g == 0) continue;
    const int pid = __ldg(p.pan + r);
    const int mapped = pid > 0 && pid < p.S1 ? __ldg(p.match + pid) : 0;
    const int slot = conf_slot(p.B, c);
    atomicAdd(s_cal + slot, 1);
    if (mapped == g) atomicAdd(s_cal + kSlots + slot, 1);
    my[slot * kBlock] += (double)c;
  }
  flush_partials(s_acc, kSlots, p.part);
  if (threadIdx.x < 2 * kSlots && s_cal[threadIdx.x]) atomicAdd(p.cal + threadIdx.x, s_cal[threadIdx.x]);
}

__global__ void k_part_reduce(const double* __restrict__ part, int G, int C, double* __restrict__ out) {
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    double a = 0.0;
    for (int g = 0; g < G; ++g) a += part[(int64_t)g * C + c];
    out[c] = a;
  }
}

// CTA count of the calibration passes: a function of n alone on a given device, so the partial sums are too
int eval_grid(int64_t n, int64_t* chunk) {
  int64_t g = (n + 4 * kBlock - 1) / (4 * kBlock);
  const int64_t cap = 2 * (int64_t)num_sms();
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  *chunk = (n + g - 1) / g;
  return (int)g;
}

// launch a calibration pass with a partial-sum workspace, then reduce the partials into sums[cols]
template <typename Params, typename Kernel>
int cal_launch(const char* name, Kernel kernel, Params& p, int cols, size_t extra_smem, double* sums, cudaStream_t st) {
  const int G = eval_grid(p.n, &p.chunk);
  double* part = nullptr;
  cudaError_t e = ws_alloc((void**)&part, sizeof(double) * (size_t)G * cols, st);
  if (e != cudaSuccess) {
    set_error("%s: workspace allocation failed: %s", name, cudaGetErrorString(e));
    return -1;
  }
  p.part = part;
  const size_t smem = sizeof(double) * cols * kBlock + extra_smem;
  cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  kernel<<<G, kBlock, smem, st>>>(p);
  k_part_reduce<<<1, 64, 0, st>>>(part, G, cols, sums);
  cudaFreeAsync(part, st);
  PASCO_CHECK_LAUNCH(name);
  return 0;
}

Bounds to_bounds(const float b[kSlots]) {
  Bounds B;
  for (int i = 0; i < kSlots; ++i) B.b[i] = b[i];
  return B;
}

// ------------------------------------------------------------------------------------------------
// dense forms: the volumes the reference's evaluate_all is given (net_panoptic_sparse.py:650-695), row i = cell i
// ------------------------------------------------------------------------------------------------

// the gt_panoptic_seg volume convert_mask_label_to_panoptic_output returns (float32, torch.zeros(masks.shape[1:])),
// zeroed at unknown cells: k_eval_gt's ids as floats
__global__ void __launch_bounds__(kBlock) k_eval_gt_volume(const int32_t* __restrict__ gt_id, int64_t cells,
                                                            float* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < cells; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = (float)__ldg(gt_id + i);
}

// k_eval_pairs over a dense id volume: no cell array, every id outside [0, S1) counts in pred_area[0]
template <bool SHARED>
__global__ void __launch_bounds__(kBlock) k_eval_pairs_dense(const int32_t* __restrict__ pan,
                                                              const int32_t* __restrict__ gt_id,
                                                              const uint8_t* __restrict__ label, int64_t cells, int G1,
                                                              int S1, int32_t* __restrict__ pairs,
                                                              int32_t* __restrict__ pred_area) {
  extern __shared__ int s_pairs[];
  const int tot = G1 * S1 + S1;
  int* tab = SHARED ? s_pairs : pairs;
  int* area = SHARED ? s_pairs + G1 * S1 : pred_area;
  if (SHARED) {
    for (int i = threadIdx.x; i < tot; i += blockDim.x) s_pairs[i] = 0;
    __syncthreads();
  }
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < cells; r += (int64_t)gridDim.x * blockDim.x) {
    const int p = __ldg(pan + r);
    if (p == 0) continue;
    if (__ldg(label + r) == 255) continue;                     // pred_panoptic_seg[unknown_mask] = 0
    if (p < 0 || p >= S1) {
      atomicAdd(area, 1);
      continue;
    }
    atomicAdd(tab + (int64_t)__ldg(gt_id + r) * S1 + p, 1);
    atomicAdd(area + p, 1);
  }
  if (SHARED) {
    __syncthreads();
    for (int i = threadIdx.x; i < tot; i += blockDim.x) {
      const int v = s_pairs[i];
      if (v) atomicAdd(i < G1 * S1 ? pairs + i : pred_area + (i - G1 * S1), v);
    }
  }
}

// SSC over channel-major class planes prob [K][cells] (evaluate_all's argmax, add_batch, add_batch_ece): per cell the
// first-max argmax over K as torch.argmax takes it (a NaN wins, the first NaN), written as int64 pred; at known cells
// the K x K confusion counts; with ECE, for the given confidence, the 2 x 2 x 16 calibration counts, the 2 x 16
// confidence sums and per partition Σ −log(prob[label] + 1e-12) (float columns as k_eval_ssc's).  bad counts the known
// cells with a label >= K and, with ECE, those whose confidence lies outside [0, 1] (torchmetrics would take sigmoids).
struct SscPlaneParams {
  const float* prob;
  const float* conf;
  const uint8_t* label;
  int64_t n, chunk;        // n = cells
  int K;
  Bounds B;
  int64_t* pred;
  int32_t* confmat;
  int32_t* cal;
  int32_t* bad;
  double* part;
};

template <bool ECE>
__global__ void __launch_bounds__(kBlock) k_eval_ssc_planes(const __grid_constant__ SscPlaneParams p) {
  extern __shared__ double s_acc[];                            // ECE: [kSscCols][kBlock]
  int* s_conf = reinterpret_cast<int*>(s_acc + (ECE ? kSscCols * kBlock : 0));   // [K * K]
  int* s_cal = s_conf + p.K * p.K;                             // [64]
  __shared__ int s_bad;
  if (ECE)
    for (int i = threadIdx.x; i < kSscCols * kBlock; i += blockDim.x) s_acc[i] = 0.0;
  for (int i = threadIdx.x; i < p.K * p.K + 4 * kSlots; i += blockDim.x) s_conf[i] = 0;
  if (threadIdx.x == 0) s_bad = 0;
  __syncthreads();
  const int64_t r0 = blockIdx.x * p.chunk, r1 = min(p.n, r0 + p.chunk);
  double* my = s_acc + threadIdx.x;
  for (int64_t i = r0 + threadIdx.x; i < r1; i += kBlock) {
    float best = __ldg(p.prob + i);
    int arg = 0;
#pragma unroll 4
    for (int k = 1; k < p.K; ++k) {
      const float v = __ldg(p.prob + (int64_t)k * p.n + i);
      if (!isnan(best) && (isnan(v) || v > best)) {
        best = v;
        arg = k;
      }
    }
    p.pred[i] = arg;
    const int lab = __ldg(p.label + i);
    if (lab == 255) continue;                                  // keep = target != 255
    if (lab >= p.K) {
      atomicAdd(&s_bad, 1);
      continue;
    }
    atomicAdd(s_conf + lab * p.K + arg, 1);
    if (ECE) {
      const float c = __ldg(p.conf + i);
      if (!(c >= 0.f && c <= 1.f)) {
        atomicAdd(&s_bad, 1);
        continue;
      }
      const int part = arg != 0, slot = conf_slot(p.B, c);
      atomicAdd(s_cal + part * 2 * kSlots + slot, 1);
      if (arg == lab) atomicAdd(s_cal + part * 2 * kSlots + kSlots + slot, 1);
      my[(part * kSlots + slot) * kBlock] += (double)c;
      const float pt = __ldg(p.prob + (int64_t)lab * p.n + i);
      my[(2 * kSlots + part) * kBlock] += (double)(-logf(__fadd_rn(pt, 1e-12f)));
    }
  }
  if (ECE) flush_partials(s_acc, kSscCols, p.part);
  else __syncthreads();
  for (int i = threadIdx.x; i < p.K * p.K + 4 * kSlots; i += blockDim.x) {
    const int v = s_conf[i];
    if (v) atomicAdd(i < p.K * p.K ? p.confmat + i : p.cal + (i - p.K * p.K), v);
  }
  if (threadIdx.x == 0 && s_bad) atomicAdd(p.bad, s_bad);
}

// k_eval_vox over dense volumes (compute_ece_panop's nonempty_mask = gt id != 0 and confidence != 0); bad counts the
// confidences of those cells outside [0, 1]
struct VoxDenseParams {
  const int32_t* pan;
  const float* conf;
  int64_t n, chunk;        // n = cells
  const int32_t* gt_id;
  const int32_t* match;    // [S1]
  int S1;
  Bounds B;
  int32_t* cal;
  int32_t* bad;
  double* part;            // [grid][16]
};

__global__ void __launch_bounds__(kBlock) k_eval_vox_dense(const __grid_constant__ VoxDenseParams p) {
  extern __shared__ double s_acc[];                            // [kSlots][kBlock]
  __shared__ int s_cal[2 * kSlots + 1];
  for (int i = threadIdx.x; i < kSlots * kBlock; i += blockDim.x) s_acc[i] = 0.0;
  if (threadIdx.x <= 2 * kSlots) s_cal[threadIdx.x] = 0;
  __syncthreads();
  const int64_t r0 = blockIdx.x * p.chunk, r1 = min(p.n, r0 + p.chunk);
  double* my = s_acc + threadIdx.x;
  for (int64_t r = r0 + threadIdx.x; r < r1; r += kBlock) {
    const float c = __ldg(p.conf + r);
    if (c == 0.f) continue;
    const int g = __ldg(p.gt_id + r);
    if (g == 0) continue;
    if (!(c >= 0.f && c <= 1.f)) {
      atomicAdd(s_cal + 2 * kSlots, 1);
      continue;
    }
    const int pid = __ldg(p.pan + r);
    const int mapped = pid > 0 && pid < p.S1 ? __ldg(p.match + pid) : 0;
    const int slot = conf_slot(p.B, c);
    atomicAdd(s_cal + slot, 1);
    if (mapped == g) atomicAdd(s_cal + kSlots + slot, 1);
    my[slot * kBlock] += (double)c;
  }
  flush_partials(s_acc, kSlots, p.part);
  if (threadIdx.x < 2 * kSlots && s_cal[threadIdx.x]) atomicAdd(p.cal + threadIdx.x, s_cal[threadIdx.x]);
  if (threadIdx.x == 2 * kSlots && s_cal[threadIdx.x]) atomicAdd(p.bad, s_cal[threadIdx.x]);
}

}  // namespace

extern "C" int pasco_eval_gt(const uint8_t* masks, int32_t n_masks, const int32_t* seg_of_mask, const uint8_t* label,
                             int64_t cells, int32_t G, int32_t K, int32_t* gt_id, int32_t* mask_count, int32_t* gt_area,
                             int32_t* hist, pasco_stream_t s) {
  PASCO_CHECK_ARG(n_masks >= 0 && G >= 0 && G <= n_masks && K >= 1 && K <= 254 && cells > 0,
                  "pasco_eval_gt: bad sizes (masks %d, segments %d, classes %d)", n_masks, G, K);
  const size_t smem = sizeof(int) * ((size_t)n_masks + G + 1 + K + 1);
  PASCO_CHECK_ARG(smem <= kSmemCap, "pasco_eval_gt: %d masks exceed the shared-memory counters", n_masks);
  cudaFuncSetAttribute(k_eval_gt, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemCap);
  k_eval_gt<<<grid_for(cells, kBlock, 2), kBlock, smem, (cudaStream_t)s>>>(masks, n_masks, seg_of_mask, label, cells, G,
                                                                          K, gt_id, mask_count, gt_area, hist);
  PASCO_CHECK_LAUNCH("pasco_eval_gt");
  return 0;
}

extern "C" int pasco_eval_pairs(const int64_t* lin, const int32_t* panoptic, int64_t n, const int32_t* gt_id,
                                const uint8_t* label, int64_t cells, int32_t G, int32_t S, int32_t* pairs,
                                int32_t* pred_area, pasco_stream_t s) {
  PASCO_CHECK_ARG(G >= 0 && S >= 0 && cells > 0, "pasco_eval_pairs: bad segment or cell counts");
  if (n == 0) return 0;
  const int G1 = G + 1, S1 = S + 1;
  const size_t smem = sizeof(int) * ((size_t)G1 * S1 + S1);
  const int grid = grid_for(n, kBlock, 2);
  if (smem <= kSmemCap) {
    cudaFuncSetAttribute(k_eval_pairs<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemCap);
    k_eval_pairs<true><<<grid, kBlock, smem, (cudaStream_t)s>>>(lin, panoptic, n, gt_id, label, cells, G1, S1, pairs,
                                                                pred_area);
  } else {
    k_eval_pairs<false><<<grid, kBlock, 0, (cudaStream_t)s>>>(lin, panoptic, n, gt_id, label, cells, G1, S1, pairs,
                                                              pred_area);
  }
  PASCO_CHECK_LAUNCH("pasco_eval_pairs");
  return 0;
}

extern "C" int pasco_eval_ssc(const int64_t* lin, const int32_t* pred, const float* conf, int64_t n,
                              const uint8_t* label, int64_t cells, int32_t K, const float bounds[16], int32_t M,
                              const float* const probs[], const int32_t* const cell_rows[], int32_t* confmat,
                              int32_t* cal, int32_t* pred_bad, double* sums, pasco_stream_t s) {
  PASCO_CHECK_ARG(K >= 1 && K <= 64, "pasco_eval_ssc: 1 <= K <= 64 classes (got %d)", K);
  PASCO_CHECK_ARG(M >= 0 && M <= kMaxSubnets, "pasco_eval_ssc: 0 <= M <= %d subnets (got %d)", kMaxSubnets, M);
  PASCO_CHECK_ARG(cells > 0, "pasco_eval_ssc: empty grid");
  SscParams p = {};
  p.sem.M = M;
  for (int m = 0; m < M; ++m) {
    p.sem.prob[m] = probs[m];
    p.sem.cell_row[m] = cell_rows[m];
  }
  p.lin = lin;
  p.pred = pred;
  p.conf = conf;
  p.n = n;
  p.label = label;
  p.cells = cells;
  p.K = K;
  p.B = to_bounds(bounds);
  p.confmat = confmat;
  p.cal = cal;
  p.pred_bad = pred_bad;
  return cal_launch("pasco_eval_ssc", k_eval_ssc, p, kSscCols, sizeof(int) * ((size_t)K * K + 4 * kSlots), sums,
                    (cudaStream_t)s);
}

extern "C" int pasco_eval_vox(const int64_t* lin, const int32_t* panoptic, const float* confidence, int64_t n,
                              const int32_t* gt_id, int64_t cells, const int32_t* match, int32_t S, const float bounds[16], int32_t* cal,
                              double* sums, pasco_stream_t s) {
  PASCO_CHECK_ARG(S >= 0 && cells > 0, "pasco_eval_vox: bad segment or cell count");
  VoxParams p = {};
  p.lin = lin;
  p.pan = panoptic;
  p.conf = confidence;
  p.n = n;
  p.gt_id = gt_id;
  p.cells = cells;
  p.match = match;
  p.S1 = S + 1;
  p.B = to_bounds(bounds);
  p.cal = cal;
  return cal_launch("pasco_eval_vox", k_eval_vox, p, kSlots, 0, sums, (cudaStream_t)s);
}

extern "C" int pasco_eval_gt_volume(const int32_t* gt_id, int64_t cells, float* out, pasco_stream_t s) {
  PASCO_CHECK_ARG(cells > 0, "pasco_eval_gt_volume: empty grid");
  k_eval_gt_volume<<<grid_for(cells, kBlock, 4), kBlock, 0, (cudaStream_t)s>>>(gt_id, cells, out);
  PASCO_CHECK_LAUNCH("pasco_eval_gt_volume");
  return 0;
}

extern "C" int pasco_eval_pairs_dense(const int32_t* panoptic, const int32_t* gt_id, const uint8_t* label,
                                      int64_t cells, int32_t G, int32_t S, int32_t* pairs, int32_t* pred_area,
                                      pasco_stream_t s) {
  PASCO_CHECK_ARG(G >= 0 && S >= 0 && cells > 0, "pasco_eval_pairs_dense: bad segment or cell counts");
  const int G1 = G + 1, S1 = S + 1;
  const size_t smem = sizeof(int) * ((size_t)G1 * S1 + S1);
  const int grid = grid_for(cells, kBlock, 2);
  if (smem <= kSmemCap) {
    cudaFuncSetAttribute(k_eval_pairs_dense<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemCap);
    k_eval_pairs_dense<true><<<grid, kBlock, smem, (cudaStream_t)s>>>(panoptic, gt_id, label, cells, G1, S1, pairs,
                                                                      pred_area);
  } else {
    k_eval_pairs_dense<false><<<grid, kBlock, 0, (cudaStream_t)s>>>(panoptic, gt_id, label, cells, G1, S1, pairs,
                                                                    pred_area);
  }
  PASCO_CHECK_LAUNCH("pasco_eval_pairs_dense");
  return 0;
}

extern "C" int pasco_eval_ssc_planes(const float* prob, int32_t K, int64_t cells, const uint8_t* label,
                                     const float* confidence, const float bounds[16], int64_t* pred, int32_t* confmat,
                                     int32_t* cal, int32_t* bad, double* sums, pasco_stream_t s) {
  PASCO_CHECK_ARG(K >= 1 && K <= 64, "pasco_eval_ssc_planes: 1 <= K <= 64 classes (got %d)", K);
  PASCO_CHECK_ARG(cells > 0, "pasco_eval_ssc_planes: empty grid");
  SscPlaneParams p = {};
  p.prob = prob;
  p.conf = confidence;
  p.label = label;
  p.n = cells;
  p.K = K;
  p.B = to_bounds(bounds);
  p.pred = pred;
  p.confmat = confmat;
  p.cal = cal;
  p.bad = bad;
  const size_t counters = sizeof(int) * ((size_t)K * K + 4 * kSlots);
  if (confidence != nullptr)
    return cal_launch("pasco_eval_ssc_planes", k_eval_ssc_planes<true>, p, kSscCols, counters, sums, (cudaStream_t)s);
  const int G = eval_grid(cells, &p.chunk);
  k_eval_ssc_planes<false><<<G, kBlock, counters, (cudaStream_t)s>>>(p);
  PASCO_CHECK_LAUNCH("pasco_eval_ssc_planes");
  return 0;
}

extern "C" int pasco_eval_vox_dense(const int32_t* panoptic, const float* confidence, const int32_t* gt_id,
                                    int64_t cells, const int32_t* match, int32_t S, const float bounds[16],
                                    int32_t* cal, int32_t* bad, double* sums, pasco_stream_t s) {
  PASCO_CHECK_ARG(S >= 0 && cells > 0, "pasco_eval_vox_dense: bad segment or cell count");
  VoxDenseParams p = {};
  p.pan = panoptic;
  p.conf = confidence;
  p.n = cells;
  p.gt_id = gt_id;
  p.match = match;
  p.S1 = S + 1;
  p.B = to_bounds(bounds);
  p.cal = cal;
  p.bad = bad;
  return cal_launch("pasco_eval_vox_dense", k_eval_vox_dense, p, kSlots, 0, sums, (cudaStream_t)s);
}
