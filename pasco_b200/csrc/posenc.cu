// The sine position encoding of the reference's mask transformer (csrc side of ops.sine_pos).
//
//   pasco_sine_pos   PositionEmbeddingSineSparse(n, normalize=True) (transformer/position_encoding.py:90-135) of integer
//                    coordinate rows, written to or added into fp32 rows [P][3n] with a row pitch.
//
// With normalize=True every axis is encoded on its own: x -> x / (x + 1e-6) * 2pi -> / dim_t[j] -> sin (even j) or cos
// (odd j), so a row's encoding is three rows of one per-coordinate table, and the kernel gathers them.  The table is
// the reference's torch expression evaluated over a span of coordinates (ops.sine_pos builds it), so every value has
// torch's own bits; computing sinf here instead would pull in its slow-path argument reduction, which lives in local
// memory.  For |x| >= 32, x + 1e-6f rounds to x in fp32 and x / x is exactly 1, so every coordinate beyond the span's
// ends encodes as the end row: the kernel clamps to the span, and no coordinate falls outside it.
#include "common.cuh"

using namespace pasco;

namespace {

__device__ __forceinline__ int span_row(int64_t v, int32_t lo, int32_t rows) {
  int64_t r = v - (int64_t)lo;
  r = r < 0 ? 0 : (r >= rows ? rows - 1 : r);
  return (int)r;
}

// one warp per coordinate row; lanes walk the 3n output columns (x block, y block, z block of n each)
template <typename T>
__global__ void __launch_bounds__(256) k_sine_pos(const T* __restrict__ coords, int64_t P, int64_t cpitch,
                                                  const float* __restrict__ table, int32_t lo, int32_t rows, int32_t n,
                                                  float* __restrict__ out, int64_t opitch, int add) {
  const int warps = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  for (int64_t r = (int64_t)blockIdx.x * warps + (threadIdx.x >> 5); r < P; r += (int64_t)gridDim.x * warps) {
    const T* c = coords + r * cpitch;
    const float* tx = table + (int64_t)span_row((int64_t)__ldg(c), lo, rows) * n;
    const float* ty = table + (int64_t)span_row((int64_t)__ldg(c + 1), lo, rows) * n;
    const float* tz = table + (int64_t)span_row((int64_t)__ldg(c + 2), lo, rows) * n;
    float* o = out + r * opitch;
    for (int k = lane; k < 3 * n; k += 32) {
      const float* t = k < n ? tx : (k < 2 * n ? ty : tz);
      const float v = __ldg(t + (k < n ? k : (k < 2 * n ? k - n : k - 2 * n)));
      o[k] = add ? o[k] + v : v;
    }
  }
}

}  // namespace

extern "C" int pasco_sine_pos(const void* coords, int32_t is_i64, int64_t P, int64_t coord_pitch, const float* table,
                              int32_t lo, int32_t rows, int32_t n, float* out, int64_t out_pitch, int32_t add,
                              pasco_stream_t s) {
  PASCO_CHECK_ARG(n >= 2 && n <= 256 && n % 2 == 0, "pasco_sine_pos: n must be even and in [2, 256] (n=%d)", n);
  PASCO_CHECK_ARG(P >= 0 && rows >= 1 && coord_pitch >= 3 && out_pitch >= 3 * (int64_t)n,
                  "pasco_sine_pos: need P >= 0, rows >= 1, coord_pitch >= 3 and out_pitch >= 3n");
  if (P == 0) return 0;
  cudaStream_t st = (cudaStream_t)s;
  const int grid = grid_for(P * 32, 256);
  if (is_i64)
    k_sine_pos<int64_t><<<grid, 256, 0, st>>>((const int64_t*)coords, P, coord_pitch, table, lo, rows, n, out,
                                              out_pitch, add);
  else
    k_sine_pos<int32_t><<<grid, 256, 0, st>>>((const int32_t*)coords, P, coord_pitch, table, lo, rows, n, out,
                                              out_pitch, add);
  PASCO_CHECK_LAUNCH("pasco_sine_pos");
  return 0;
}
