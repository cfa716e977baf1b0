// CUDA-core fp32 path of the sparse-conv contraction  out[o,:] = Σ_k in[nbr[k,o],:] @ W[k].
// Any Cin/Cout.  This is the in-library cross-check for the tensor-core path (conv_tc.cu) and serves the
// shapes the tensor-core kernels do not take (channel counts that are not multiples of 16, or more than 512 outputs).
#include "common.cuh"

using namespace pasco;

constexpr int TR = 16;  // output rows per block
struct KoffMap {
  int v[256];
};

// W layout: transposed==0 → W[k][ci][co] ; transposed==1 → W[k][co][ci] (used for dgrad: "Cin" here is the
// gradient's channel count = forward Cout)
__global__ void __launch_bounds__(256)
k_conv_simt(const float* __restrict__ in, const int32_t* __restrict__ nbr, int K, int64_t n_out, int Cin, int Cout,
            const float* __restrict__ W, int w_transposed, const __grid_constant__ KoffMap koff, const float* __restrict__ bias,
            float* __restrict__ out) {
  extern __shared__ float sA[];  // [TR][Cin]
  __shared__ int sIdx[TR];
  int64_t row0 = (int64_t)blockIdx.x * TR;
  // each thread owns output columns co = threadIdx.x + j*256, all TR rows
  constexpr int MAXJ = 2;  // Cout <= 512
  float acc[MAXJ][TR];
#pragma unroll
  for (int j = 0; j < MAXJ; ++j)
#pragma unroll
    for (int r = 0; r < TR; ++r) acc[j][r] = 0.f;

  for (int k = 0; k < K; ++k) {
    if (threadIdx.x < TR) {
      int64_t o = row0 + threadIdx.x;
      sIdx[threadIdx.x] = o < n_out ? __ldg(nbr + (int64_t)k * n_out + o) : -1;
    }
    __syncthreads();
    int any = 0;
#pragma unroll
    for (int r = 0; r < TR; ++r) any |= (sIdx[r] >= 0);
    if (any) {
      for (int t = threadIdx.x; t < TR * Cin; t += blockDim.x) {
        int r = t / Cin, c = t - r * Cin;
        int src = sIdx[r];
        sA[t] = src >= 0 ? __ldg(in + (int64_t)src * Cin + c) : 0.f;
      }
      __syncthreads();
      int kw = koff.v[k];
      const float* Wk = W + (int64_t)kw * Cin * Cout;
#pragma unroll
      for (int j = 0; j < MAXJ; ++j) {
        int co = threadIdx.x + j * 256;
        if (co < Cout) {
          for (int ci = 0; ci < Cin; ++ci) {
            float w = w_transposed ? __ldg(Wk + (int64_t)co * Cin + ci) : __ldg(Wk + (int64_t)ci * Cout + co);
#pragma unroll
            for (int r = 0; r < TR; ++r) acc[j][r] = fmaf(sA[r * Cin + ci], w, acc[j][r]);
          }
        }
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int j = 0; j < MAXJ; ++j) {
    int co = threadIdx.x + j * 256;
    if (co < Cout) {
      float b = bias ? __ldg(bias + co) : 0.f;
#pragma unroll
      for (int r = 0; r < TR; ++r) {
        int64_t o = row0 + r;
        if (o < n_out) out[o * Cout + co] = acc[j][r] + b;
      }
    }
  }
}

extern "C" int pasco_conv_forward_simt(const float* in, const int32_t* nbr, int32_t K, int64_t n_out, int32_t Cin,
                                       int32_t Cout, const float* W, int32_t w_transposed, const int32_t* koff_map,
                                       const float* bias, float* out, pasco_stream_t s) {
  PASCO_CHECK_ARG(Cout <= 512 && Cin <= 2048, "pasco_conv_forward_simt: channel count too large");
  PASCO_CHECK_ARG(K <= 256, "pasco_conv_forward_simt: K too large");
  if (n_out == 0) return 0;
  cudaStream_t st = (cudaStream_t)s;
  KoffMap km;
  for (int k = 0; k < K; ++k) km.v[k] = koff_map ? koff_map[k] : k;
  int64_t nb = (n_out + TR - 1) / TR;
  size_t smem = (size_t)TR * Cin * sizeof(float);
  if (smem > 48 * 1024) cudaFuncSetAttribute(k_conv_simt, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  k_conv_simt<<<(unsigned)nb, 256, smem, st>>>(in, nbr, K, n_out, Cin, Cout, W, w_transposed, km, bias, out);
  PASCO_CHECK_LAUNCH("pasco_conv_forward_simt");
  return 0;
}

// dW[k][ci][co] = Σ_o in[nbr[k,o]][ci] * gout[o][co];  grid = (row blocks, K); each block stores its partial sums
constexpr int WG_ROWS = 2048;  // minimum rows per block
constexpr int WG_TILE = 16;    // rows staged per iteration
constexpr int WG_MAX_BLOCKS = 128;
constexpr int64_t WG_MAX_WS_FLOATS = 16 << 20;   // workspace bound: 64 MB of per-block partials

__global__ void __launch_bounds__(256)
k_wgrad_simt(const float* __restrict__ in, const int32_t* __restrict__ nbr, int64_t n_out, int64_t rows, int Cin, int Cout,
             const float* __restrict__ gout, float* __restrict__ part) {
  extern __shared__ float sm[];  // sA[WG_TILE][Cin], sG[WG_TILE][Cout]
  float* sA = sm;
  float* sG = sm + WG_TILE * Cin;
  __shared__ int sIdx[WG_TILE];
  int k = blockIdx.y;
  int64_t r0 = (int64_t)blockIdx.x * rows;
  int64_t r1 = r0 + rows < n_out ? r0 + rows : n_out;
  int total = Cin * Cout;
  // each thread owns outputs e = threadIdx.x + j*256 (ci = e / Cout, co = e % Cout)
  constexpr int MAXE = 16;  // up to 4096 outputs per pass
  for (int e0 = 0; e0 < total; e0 += 256 * MAXE) {
    float acc[MAXE];
#pragma unroll
    for (int j = 0; j < MAXE; ++j) acc[j] = 0.f;
    for (int64_t rr = r0; rr < r1; rr += WG_TILE) {
      if (threadIdx.x < WG_TILE) {
        int64_t o = rr + threadIdx.x;
        sIdx[threadIdx.x] = o < r1 ? __ldg(nbr + (int64_t)k * n_out + o) : -1;
      }
      __syncthreads();
      int any = 0;
#pragma unroll
      for (int r = 0; r < WG_TILE; ++r) any |= (sIdx[r] >= 0);
      if (any) {
        for (int t = threadIdx.x; t < WG_TILE * Cin; t += 256) {
          int r = t / Cin, c = t - r * Cin;
          int src = sIdx[r];
          sA[t] = src >= 0 ? __ldg(in + (int64_t)src * Cin + c) : 0.f;
        }
        for (int t = threadIdx.x; t < WG_TILE * Cout; t += 256) {
          int r = t / Cout, c = t - r * Cout;
          sG[t] = (sIdx[r] >= 0) ? __ldg(gout + (rr + r) * Cout + c) : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < MAXE; ++j) {
          int e = e0 + threadIdx.x + j * 256;
          if (e < total) {
            int ci = e / Cout, co = e - ci * Cout;
#pragma unroll
            for (int r = 0; r < WG_TILE; ++r) acc[j] = fmaf(sA[r * Cin + ci], sG[r * Cout + co], acc[j]);
          }
        }
      }
      __syncthreads();
    }
#pragma unroll
    for (int j = 0; j < MAXE; ++j) {
      int e = e0 + threadIdx.x + j * 256;
      if (e < total) part[((int64_t)blockIdx.x * gridDim.y + k) * total + e] = acc[j];
    }
  }
}

// dW[i] += Σ_b part[b][i] in block order (deterministic, no atomics)
__global__ void k_wgrad_simt_sum(const float* __restrict__ part, int nb, int64_t n, float* __restrict__ dW) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float acc = 0.f;
    for (int b = 0; b < nb; ++b) acc += __ldg(part + b * n + i);
    dW[i] += acc;
  }
}

extern "C" int pasco_conv_wgrad_simt(const float* in, const int32_t* nbr, int32_t K, int64_t n_out, int32_t Cin,
                                     int32_t Cout, const float* gout, float* dW, pasco_stream_t s) {
  if (n_out == 0) return 0;
  size_t smem = (size_t)WG_TILE * (Cin + Cout) * sizeof(float);
  PASCO_CHECK_ARG(smem <= 200 * 1024, "pasco_conv_wgrad_simt: channels too large");
  if (smem > 48 * 1024) cudaFuncSetAttribute(k_wgrad_simt, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  // at most WG_MAX_BLOCKS row blocks (fewer when K*Cin*Cout is large, so that the workspace stays within 64 MB), whose
  // partials go to a stream-ordered workspace and are summed in block order
  const int64_t n = (int64_t)K * Cin * Cout;
  int64_t max_blocks = WG_MAX_WS_FLOATS / n;
  if (max_blocks > WG_MAX_BLOCKS) max_blocks = WG_MAX_BLOCKS;
  if (max_blocks < 1) max_blocks = 1;
  int64_t rows = (n_out + max_blocks - 1) / max_blocks;
  if (rows < WG_ROWS) rows = WG_ROWS;
  rows = (rows + WG_TILE - 1) / WG_TILE * WG_TILE;
  const int nb = (int)((n_out + rows - 1) / rows);
  cudaStream_t st = (cudaStream_t)s;
  float* part = nullptr;
  cudaError_t e = ws_alloc((void**)&part, (size_t)nb * n * sizeof(float), st);
  if (e != cudaSuccess) {
    ::pasco::set_error("pasco_conv_wgrad_simt: workspace of %lld bytes: %s", (long long)nb * n * 4, cudaGetErrorString(e));
    return -1;
  }
  k_wgrad_simt<<<dim3((unsigned)nb, K), 256, smem, st>>>(in, nbr, n_out, rows, Cin, Cout, gout, part);
  k_wgrad_simt_sum<<<grid_for(n, 256), 256, 0, st>>>(part, nb, n, dW);
  cudaFreeAsync(part, st);
  PASCO_CHECK_LAUNCH("pasco_conv_wgrad_simt");
  return 0;
}
