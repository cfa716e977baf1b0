// Column statistics / fused affine+activation (BatchNorm over rows), max-pool, scatter-max.
// All HBM-bound: one coalesced pass over [N, C] float32 per call.
#include <math_constants.h>
#include "common.cuh"

using namespace pasco;

// ------------------------------------------------------------------------------------------------
// activation helpers: 0 none, 1 ReLU, 2 LeakyReLU(0.01) (act_fwd: common.cuh)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float act_grad(float z, int act) {
  if (act == 1) return z > 0.f ? 1.f : 0.f;
  if (act == 2) return z > 0.f ? 1.f : 0.01f;
  return 1.f;
}

// ------------------------------------------------------------------------------------------------
// column sums.  Vector path (C % 4 == 0): a thread owns 4 consecutive channels (one float4 per row), a block of
// 256 threads covers G = 256 / (C/4) rows per step and walks its row chunk with 4 independent loads in flight per
// thread (the first version issued one dependent 4-byte load per iteration and ran at ~0.9 TB/s).
// ------------------------------------------------------------------------------------------------
constexpr int kRowLanes = 8;
constexpr int kRowsPerBlock = 512;
constexpr int kVecRowsPerBlock = 2048;

__device__ __forceinline__ void col_acc(float4& s0, float4& s1, const float4& v, const float4& d, int mode, const float4& sc,
                                        const float4& sh, int act) {
  if (mode == 0) {
    s0.x += v.x; s0.y += v.y; s0.z += v.z; s0.w += v.w;
    s1.x += v.x * v.x; s1.y += v.y * v.y; s1.z += v.z * v.z; s1.w += v.w * v.w;
  } else {
    const float zx = d.x * act_grad(fmaf(v.x, sc.x, sh.x), act), zy = d.y * act_grad(fmaf(v.y, sc.y, sh.y), act);
    const float zz = d.z * act_grad(fmaf(v.z, sc.z, sh.z), act), zw = d.w * act_grad(fmaf(v.w, sc.w, sh.w), act);
    s0.x += zx; s0.y += zy; s0.z += zz; s0.w += zw;
    s1.x += zx * v.x; s1.y += zy * v.y; s1.z += zz * v.z; s1.w += zw * v.w;
  }
}

template <int MODE>
__global__ void __launch_bounds__(256) k_col_sums_vec(const float* __restrict__ x, const float* __restrict__ dy, int64_t n, int C,
                                                      const float* __restrict__ scale, const float* __restrict__ shift,
                                                      int act, double* __restrict__ sums) {
  extern __shared__ float red[];              // [2][256][4]
  const int cv = C >> 2;                      // float4 columns (<= 256)
  const int G = 256 / cv;                     // rows per step
  const int cg = threadIdx.x % cv, rl = threadIdx.x / cv;
  const int64_t row0 = (int64_t)blockIdx.x * kVecRowsPerBlock;
  const int64_t row1 = row0 + kVecRowsPerBlock < n ? row0 + kVecRowsPerBlock : n;
  float4 s0 = make_float4(0.f, 0.f, 0.f, 0.f), s1 = s0;
  float4 sc = make_float4(1.f, 1.f, 1.f, 1.f), sh = make_float4(0.f, 0.f, 0.f, 0.f);
  if (MODE == 1 && scale) {
    sc = __ldg(reinterpret_cast<const float4*>(scale) + cg);
    sh = __ldg(reinterpret_cast<const float4*>(shift) + cg);
  }
  if (rl < G) {
    const float4* xv = reinterpret_cast<const float4*>(x);
    const float4* dv = reinterpret_cast<const float4*>(dy);
    int64_t r = row0 + rl;
    for (; r + 3 * G < row1; r += 4 * G) {
      float4 v[4], d[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        v[u] = __ldg(xv + (r + u * G) * cv + cg);
        if (MODE == 1) d[u] = __ldg(dv + (r + u * G) * cv + cg);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) col_acc(s0, s1, v[u], d[u], MODE, sc, sh, act);
    }
    for (; r < row1; r += G) {
      float4 v = __ldg(xv + r * cv + cg), d = make_float4(0.f, 0.f, 0.f, 0.f);
      if (MODE == 1) d = __ldg(dv + r * cv + cg);
      col_acc(s0, s1, v, d, MODE, sc, sh, act);
    }
  }
  float4* r0 = reinterpret_cast<float4*>(red);
  float4* r1 = r0 + 256;
  r0[threadIdx.x] = s0;
  r1[threadIdx.x] = s1;
  __syncthreads();
  if (threadIdx.x < cv) {
    double a0[4] = {0, 0, 0, 0}, a1[4] = {0, 0, 0, 0};
    for (int l = 0; l < G; ++l) {
      const float4 p0 = r0[l * cv + threadIdx.x], p1 = r1[l * cv + threadIdx.x];
      a0[0] += p0.x; a0[1] += p0.y; a0[2] += p0.z; a0[3] += p0.w;
      a1[0] += p1.x; a1[1] += p1.y; a1[2] += p1.z; a1[3] += p1.w;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      atomicAdd(sums + threadIdx.x * 4 + j, a0[j]);
      atomicAdd(sums + C + threadIdx.x * 4 + j, a1[j]);
    }
  }
}

// scalar fallback (any C): block = 32 (channels) x 8 (row lanes)
// MODE 0: (Σx, Σx²)   MODE 1: (Σdz, Σdz·x) with dz = dy·act'(x·scale+shift)
template <int MODE>
__global__ void k_col_sums(const float* __restrict__ x, const float* __restrict__ dy, int64_t n, int C,
                           const float* __restrict__ scale, const float* __restrict__ shift, int act,
                           double* __restrict__ sums) {
  __shared__ float red[2][kRowLanes][32];
  int64_t row0 = (int64_t)blockIdx.x * kRowsPerBlock;
  int64_t row1 = row0 + kRowsPerBlock < n ? row0 + kRowsPerBlock : n;
  for (int c0 = 0; c0 < C; c0 += 32) {
    int c = c0 + threadIdx.x;
    float s0 = 0.f, s1 = 0.f;
    if (c < C) {
      float sc = 1.f, sh = 0.f;
      if (MODE == 1 && scale) {
        sc = __ldg(scale + c);
        sh = __ldg(shift + c);
      }
      for (int64_t r = row0 + threadIdx.y; r < row1; r += kRowLanes) {
        float v = __ldg(x + r * C + c);
        if (MODE == 0) {
          s0 += v;
          s1 += v * v;
        } else {
          float dz = __ldg(dy + r * C + c) * act_grad(v * sc + sh, act);
          s0 += dz;
          s1 += dz * v;
        }
      }
    }
    red[0][threadIdx.y][threadIdx.x] = s0;
    red[1][threadIdx.y][threadIdx.x] = s1;
    __syncthreads();
    if (threadIdx.y < 2 && c < C) {
      double acc = 0.0;
#pragma unroll
      for (int l = 0; l < kRowLanes; ++l) acc += (double)red[threadIdx.y][l][threadIdx.x];
      atomicAdd(sums + (int64_t)threadIdx.y * C + c, acc);
    }
    __syncthreads();
  }
}

template <int MODE>
static int launch_col_sums(const float* x, const float* dy, int64_t n, int C, const float* scale, const float* shift, int act,
                           double* sums, cudaStream_t st) {
  const bool vec = (C % 4 == 0) && (C / 4 <= 256) &&
                   ((((uintptr_t)x | (uintptr_t)dy | (uintptr_t)scale | (uintptr_t)shift) & 15) == 0);
  if (vec && 256 / (C / 4) >= 1) {
    int64_t nb = (n + kVecRowsPerBlock - 1) / kVecRowsPerBlock;
    k_col_sums_vec<MODE><<<(unsigned)nb, 256, 2 * 256 * 16, st>>>(x, dy, n, C, scale, shift, act, sums);
  } else {
    int64_t nb = (n + kRowsPerBlock - 1) / kRowsPerBlock;
    k_col_sums<MODE><<<(unsigned)nb, dim3(32, kRowLanes), 0, st>>>(x, dy, n, C, scale, shift, act, sums);
  }
  return 0;
}

extern "C" int pasco_bn_stats(const float* x, int64_t n, int32_t C, double* stats, pasco_stream_t s) {
  if (n == 0 || C == 0) return 0;
  launch_col_sums<0>(x, nullptr, n, C, nullptr, nullptr, 0, stats, (cudaStream_t)s);
  PASCO_CHECK_LAUNCH("pasco_bn_stats");
  return 0;
}

// ------------------------------------------------------------------------------------------------
// per-channel coefficient kernels: everything between the column sums and the apply pass in ONE launch (was ~15 tiny
// fp64 torch kernels per layer and the host-side bottleneck of the backward pass)
// ------------------------------------------------------------------------------------------------
__global__ void k_bn_finalize(const double* __restrict__ stats, const double* __restrict__ count_dev, double count, int C,
                              const float* __restrict__ gamma, const float* __restrict__ beta, float eps, float momentum,
                              float* __restrict__ scale, float* __restrict__ shift, float* __restrict__ mean_out,
                              float* __restrict__ rstd_out, float* __restrict__ run_mean, float* __restrict__ run_var) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double n = count_dev ? *count_dev : count;
  const double mean = stats[c] / n;
  double var = stats[C + c] / n - mean * mean;
  if (var < 0) var = 0;
  const double rstd = rsqrt(var + (double)eps);
  const double g = gamma ? (double)gamma[c] : 1.0, b = beta ? (double)beta[c] : 0.0;
  scale[c] = (float)(g * rstd);
  shift[c] = (float)(b - mean * g * rstd);
  mean_out[c] = (float)mean;
  rstd_out[c] = (float)rstd;
  if (run_mean) {
    const double unbias = n / (n > 1.0 ? n - 1.0 : 1.0);
    run_mean[c] = (1.f - momentum) * run_mean[c] + momentum * (float)mean;
    run_var[c] = (1.f - momentum) * run_var[c] + momentum * (float)(var * unbias);
  }
}

extern "C" int pasco_bn_finalize(const double* stats, const double* count_dev, double count, int32_t C, const float* gamma,
                                 const float* beta, float eps, float momentum, float* scale, float* shift, float* mean,
                                 float* rstd, float* running_mean, float* running_var, pasco_stream_t s) {
  if (C == 0) return 0;
  k_bn_finalize<<<(C + 127) / 128, 128, 0, (cudaStream_t)s>>>(stats, count_dev, count, C, gamma, beta, eps, momentum, scale,
                                                            shift, mean, rstd, running_mean, running_var);
  PASCO_CHECK_LAUNCH("pasco_bn_finalize");
  return 0;
}

// sums = (Σdz, Σdz·x) → dx = ca·dz + cb·x + cc coefficients and the parameter gradients
__global__ void k_bn_bwd_coefs(const double* __restrict__ sums, const double* __restrict__ count_dev, double count, int C,
                               const float* __restrict__ gamma, const float* __restrict__ mean, const float* __restrict__ rstd,
                               float grad_div, float* __restrict__ ca, float* __restrict__ cb, float* __restrict__ cc,
                               float* __restrict__ ggamma, float* __restrict__ gbeta) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double n = count_dev ? *count_dev : count;
  const double s_dz = sums[c], s_dzx = sums[C + c];
  const double m = mean[c], r = rstd[c], g = gamma ? (double)gamma[c] : 1.0;
  const double s_dzxhat = r * (s_dzx - m * s_dz);
  const double m1 = s_dz / n, m2 = s_dzxhat / n;
  ca[c] = (float)(g * r);
  cb[c] = (float)(-g * r * r * m2);
  cc[c] = (float)(g * r * (m * r * m2 - m1));
  ggamma[c] = (float)(s_dzxhat / grad_div);
  gbeta[c] = (float)(s_dz / grad_div);
}

extern "C" int pasco_bn_bwd_coefs(const double* sums, const double* count_dev, double count, int32_t C, const float* gamma,
                                  const float* mean, const float* rstd, float grad_div, float* ca, float* cb, float* cc,
                                  float* ggamma, float* gbeta, pasco_stream_t s) {
  if (C == 0) return 0;
  k_bn_bwd_coefs<<<(C + 127) / 128, 128, 0, (cudaStream_t)s>>>(sums, count_dev, count, C, gamma, mean, rstd, grad_div, ca, cb,
                                                             cc, ggamma, gbeta);
  PASCO_CHECK_LAUNCH("pasco_bn_bwd_coefs");
  return 0;
}

extern "C" int pasco_bn_bwd_reduce(const float* dy, const float* x, int64_t n, int32_t C, const float* scale,
                                   const float* shift, int32_t act, double* sums, pasco_stream_t s) {
  if (n == 0 || C == 0) return 0;
  launch_col_sums<1>(x, dy, n, C, scale, shift, act, sums, (cudaStream_t)s);
  PASCO_CHECK_LAUNCH("pasco_bn_bwd_reduce");
  return 0;
}

// ------------------------------------------------------------------------------------------------
// y = act(x*scale[c] + shift[c] + residual)
// ------------------------------------------------------------------------------------------------
template <bool VEC>
__global__ void k_affine_act(const float* __restrict__ x, int64_t n, int C, const float* __restrict__ scale,
                             const float* __restrict__ shift, int act, const float* __restrict__ residual,
                             float* __restrict__ y) {
  if (VEC) {
    int cv = C >> 2;
    int64_t total = n * cv;
    for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
      int c = (int)(t % cv) << 2;
      float4 v = __ldg((const float4*)x + t);
      float4 sc = scale ? __ldg((const float4*)(scale + c)) : make_float4(1.f, 1.f, 1.f, 1.f);
      float4 sh = shift ? __ldg((const float4*)(shift + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
      float4 r = residual ? __ldg((const float4*)residual + t) : make_float4(0.f, 0.f, 0.f, 0.f);
      float4 o;
      o.x = act_fwd(fmaf(v.x, sc.x, sh.x) + r.x, act);
      o.y = act_fwd(fmaf(v.y, sc.y, sh.y) + r.y, act);
      o.z = act_fwd(fmaf(v.z, sc.z, sh.z) + r.z, act);
      o.w = act_fwd(fmaf(v.w, sc.w, sh.w) + r.w, act);
      ((float4*)y)[t] = o;
    }
  } else {
    int64_t total = n * C;
    for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
      int c = (int)(t % C);
      float z = fmaf(__ldg(x + t), scale ? __ldg(scale + c) : 1.f, shift ? __ldg(shift + c) : 0.f);
      if (residual) z += __ldg(residual + t);
      y[t] = act_fwd(z, act);
    }
  }
}

extern "C" int pasco_affine_act(const float* x, int64_t n, int32_t C, const float* scale, const float* shift,
                                int32_t act, const float* residual, float* y, pasco_stream_t s) {
  if (n == 0 || C == 0) return 0;
  cudaStream_t st = (cudaStream_t)s;
  bool vec = (C % 4 == 0) && ((((uintptr_t)x | (uintptr_t)y | (uintptr_t)residual | (uintptr_t)scale | (uintptr_t)shift) % 16) == 0);
  if (vec)
    k_affine_act<true><<<grid_for(n * (C / 4), 256), 256, 0, st>>>(x, n, C, scale, shift, act, residual, y);
  else
    k_affine_act<false><<<grid_for(n * C, 256), 256, 0, st>>>(x, n, C, scale, shift, act, residual, y);
  PASCO_CHECK_LAUNCH("pasco_affine_act");
  return 0;
}

// dx = a[c]*dz + b[c]*x + c0[c],  dz = dy * act'(x*scale+shift)
__global__ void k_bn_bwd_apply_vec(const float4* __restrict__ dy, const float4* __restrict__ x, int64_t n, int cv,
                                   const float4* __restrict__ scale, const float4* __restrict__ shift, int act,
                                   const float4* __restrict__ ca, const float4* __restrict__ cb, const float4* __restrict__ cc,
                                   float4* __restrict__ dx) {
  const int64_t total = n * cv;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(t % cv);
    const float4 v = __ldg(x + t), g = __ldg(dy + t);
    const float4 sc = scale ? __ldg(scale + c) : make_float4(1.f, 1.f, 1.f, 1.f);
    const float4 sh = shift ? __ldg(shift + c) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 a = __ldg(ca + c), b = __ldg(cb + c), k = __ldg(cc + c);
    float4 o;
    o.x = fmaf(a.x, g.x * act_grad(fmaf(v.x, sc.x, sh.x), act), fmaf(b.x, v.x, k.x));
    o.y = fmaf(a.y, g.y * act_grad(fmaf(v.y, sc.y, sh.y), act), fmaf(b.y, v.y, k.y));
    o.z = fmaf(a.z, g.z * act_grad(fmaf(v.z, sc.z, sh.z), act), fmaf(b.z, v.z, k.z));
    o.w = fmaf(a.w, g.w * act_grad(fmaf(v.w, sc.w, sh.w), act), fmaf(b.w, v.w, k.w));
    dx[t] = o;
  }
}

__global__ void k_bn_bwd_apply(const float* __restrict__ dy, const float* __restrict__ x, int64_t n, int C,
                               const float* __restrict__ scale, const float* __restrict__ shift, int act,
                               const float* __restrict__ ca, const float* __restrict__ cb,
                               const float* __restrict__ cc, float* __restrict__ dx) {
  int64_t total = n * C;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    int c = (int)(t % C);
    float v = __ldg(x + t);
    float z = fmaf(v, scale ? __ldg(scale + c) : 1.f, shift ? __ldg(shift + c) : 0.f);
    float dz = __ldg(dy + t) * act_grad(z, act);
    dx[t] = fmaf(__ldg(ca + c), dz, fmaf(__ldg(cb + c), v, __ldg(cc + c)));
  }
}

extern "C" int pasco_bn_bwd_apply(const float* dy, const float* x, int64_t n, int32_t C, const float* scale,
                                  const float* shift, int32_t act, const float* coef_a, const float* coef_b,
                                  const float* coef_c, float* dx, pasco_stream_t s) {
  if (n == 0 || C == 0) return 0;
  const bool vec = (C % 4 == 0) && ((((uintptr_t)dy | (uintptr_t)x | (uintptr_t)dx | (uintptr_t)scale | (uintptr_t)shift |
                                       (uintptr_t)coef_a | (uintptr_t)coef_b | (uintptr_t)coef_c) & 15) == 0);
  if (vec)
    k_bn_bwd_apply_vec<<<grid_for(n * (C / 4), 256), 256, 0, (cudaStream_t)s>>>(
        (const float4*)dy, (const float4*)x, n, C / 4, (const float4*)scale, (const float4*)shift, act, (const float4*)coef_a,
        (const float4*)coef_b, (const float4*)coef_c, (float4*)dx);
  else
    k_bn_bwd_apply<<<grid_for(n * C, 256), 256, 0, (cudaStream_t)s>>>(dy, x, n, C, scale, shift, act, coef_a, coef_b,
                                                                      coef_c, dx);
  PASCO_CHECK_LAUNCH("pasco_bn_bwd_apply");
  return 0;
}

// ------------------------------------------------------------------------------------------------
// atomic float max (works with a -inf initial value)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void atomic_max_float(float* addr, float v) {
  if (v >= 0.f)
    atomicMax((int*)addr, __float_as_int(v));
  else
    atomicMin((unsigned int*)addr, __float_as_uint(v));
}

__global__ void k_maxpool(const float* __restrict__ in, const int32_t* __restrict__ parent, int64_t n, int C,
                          float* __restrict__ out) {
  int64_t total = n * C;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    int64_t i = t / C;
    int c = (int)(t - i * C);
    int p = __ldg(parent + i);
    if (p >= 0) atomic_max_float(out + (int64_t)p * C + c, __ldg(in + t));
  }
}

extern "C" int pasco_maxpool_forward(const float* in, const int32_t* parent_of, int64_t n_in, int32_t C, float* out,
                                     pasco_stream_t s) {
  if (n_in == 0 || C == 0) return 0;
  k_maxpool<<<grid_for(n_in * C, 256), 256, 0, (cudaStream_t)s>>>(in, parent_of, n_in, C, out);
  PASCO_CHECK_LAUNCH("pasco_maxpool_forward");
  return 0;
}

__global__ void k_scatter_max(const float* __restrict__ src, const int64_t* __restrict__ index, int64_t n, int C,
                              float* __restrict__ out) {
  int64_t total = n * C;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    int64_t i = t / C;
    int c = (int)(t - i * C);
    atomic_max_float(out + __ldg(index + i) * C + c, __ldg(src + t));
  }
}

__global__ void k_scatter_argmax(const float* __restrict__ src, const int64_t* __restrict__ index, int64_t n, int C,
                                 const float* __restrict__ out, unsigned long long* __restrict__ arg) {
  int64_t total = n * C;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    int64_t i = t / C;
    int c = (int)(t - i * C);
    int64_t o = __ldg(index + i) * C + c;
    if (__ldg(src + t) == out[o]) atomicMin(arg + o, (unsigned long long)i);
  }
}

__global__ void k_fill_empty(float* __restrict__ out, int64_t total) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x)
    if (out[t] == -CUDART_INF_F) out[t] = 0.f;
}

extern "C" int pasco_scatter_max(const float* src, const int64_t* index, int64_t n, int32_t C, float* out,
                                 int64_t n_seg, int64_t* argmax, pasco_stream_t s) {
  cudaStream_t st = (cudaStream_t)s;
  if (n > 0 && C > 0) {
    k_scatter_max<<<grid_for(n * C, 256), 256, 0, st>>>(src, index, n, C, out);
    if (argmax) k_scatter_argmax<<<grid_for(n * C, 256), 256, 0, st>>>(src, index, n, C, out, (unsigned long long*)argmax);
  }
  if (n_seg * C > 0) k_fill_empty<<<grid_for(n_seg * C, 256), 256, 0, st>>>(out, n_seg * C);
  PASCO_CHECK_LAUNCH("pasco_scatter_max");
  return 0;
}
