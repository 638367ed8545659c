// Spectral normalisation (torch.nn.utils.spectral_norm, as build_norm_layer applies it for norm_type='snorm':
// segan/models/modules.py:12-14, discriminator.py:118-121) on the PACKED fp32 master of a tap-GEMM layer.
//
// torch keeps weight_orig W (reshaped to [height = dim 0][rest]), buffers u [height], v [rest]; every training
// forward runs ONE power iteration  v = normalize(W^T u), u = normalize(W v)  (no grad), then uses W / sigma with
// sigma = u^T W v, differentiated through sigma with u, v constant.  The structural zeros of the packed layout
// M[T][nc][kc] contribute nothing to either product, so the iteration runs on the master as it lies: u has one entry
// per n (the layer's output channel), v one per (t, k) slot.  The two small vectors are converted to the reference
// layout only for state_dict().
#include "common.cuh"

namespace sg {

// vraw[t][k] = sum_n M[t][n][k] * u[n] ;  n2 += sum vraw^2            (thread = one (t, k) column)
__global__ void __launch_bounds__(256)
snorm_wt_u_kernel(const float* __restrict__ m, int nc, int kc, const float* __restrict__ u, float* __restrict__ vraw,
                  float* __restrict__ n2) {
  const int t = blockIdx.y;
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  float acc = 0.f;
  if (k < kc) {
    const float* p = m + (int64_t)t * nc * kc + k;
    for (int n = 0; n < nc; ++n) acc = fmaf(p[(int64_t)n * kc], __ldg(u + n), acc);
    vraw[(int64_t)t * kc + k] = acc;
  }
  float s = warp_sum(acc * acc);
  if ((threadIdx.x & 31) == 0 && s != 0.f) atomicAdd(n2, s);
}

// uraw[n] = sum_{t,k} M[t][n][k] * vraw[t][k] / max(sqrt(*n2v), eps) ;  n2u += uraw^2    (block = one row n)
__global__ void __launch_bounds__(256)
snorm_w_v_kernel(const float* __restrict__ m, int T, int nc, int kc, const float* __restrict__ vraw,
                 const float* __restrict__ n2v, float* __restrict__ uraw, float* __restrict__ n2u) {
  __shared__ float red[8];
  const int n = blockIdx.x;
  float acc = 0.f;
  for (int t = 0; t < T; ++t) {
    const float* p = m + ((int64_t)t * nc + n) * kc;
    const float* v = vraw + (int64_t)t * kc;
    for (int k = threadIdx.x; k < kc; k += 256) acc = fmaf(p[k], v[k], acc);
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < 8; ++i) s += red[i];
    const float inv = n2v ? 1.f / fmaxf(sqrtf(*n2v), 1e-12f) : 1.f;
    s *= inv;
    uraw[n] = s;
    atomicAdd(n2u, s * s);
  }
}

// normalise in place, publish sigma = ||uraw|| (= u^T W v for the freshly iterated u, v) and 1 / sigma
//   scal[0] = ||vraw||^2 (in), scal[1] = ||uraw||^2 (in), scal[2] = sigma (out), scal[3] = 1/sigma (out)
__global__ void snorm_finish_kernel(float* __restrict__ u, int nu, float* __restrict__ v, int nv,
                                    float* __restrict__ scal, int update_vectors) {
  const float nvn = fmaxf(sqrtf(scal[0]), 1e-12f);
  const float nun = fmaxf(sqrtf(scal[1]), 1e-12f);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (update_vectors) {
    if (i < nv) v[i] = v[i] / nvn;
    if (i < nu) u[i] = u[i] / nun;
  }
  if (i == 0) {
    // training: sigma = u^T W v = ||W v|| ; eval (update_vectors == 0): scal[1] holds u^T (W v) directly
    const float sigma = update_vectors ? sqrtf(scal[1]) : scal[1];
    scal[2] = sigma;
    scal[3] = 1.f / sigma;
  }
}

// eval mode: scal[1] = sum_n u[n] * (W v)[n]   with the STORED (already normalised) u, v
__global__ void snorm_dot_kernel(const float* __restrict__ a, const float* __restrict__ b, int64_t n,
                                 float* __restrict__ out) {
  float s = 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    s = fmaf(a[i], b[i], s);
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0 && s != 0.f) atomicAdd(out, s);
}

// gradient through W / sigma (u, v constant):  dW = G / sigma - (<G, W~> / sigma) u v^T,  <G, W~> = <G, W> / sigma
//   dwp[t][n][k] = dwp * inv_sigma - (dot * inv_sigma^2) * u[n] * v[t][k]      (dot = <dwp, M> = <G, W>)
__global__ void __launch_bounds__(256)
snorm_grad_apply_kernel(float* __restrict__ dwp, int T, int nc, int kc, const float* __restrict__ u,
                        const float* __restrict__ v, const float* __restrict__ scal, const float* __restrict__ dot) {
  const float is = scal[3];
  const float c = (*dot) * is * is;
  const int64_t total = (int64_t)T * nc * kc;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int k = (int)(i % kc);
    const int64_t r = i / kc;
    const int n = (int)(r % nc), t = (int)(r / nc);
    dwp[i] = dwp[i] * is - c * u[n] * v[(int64_t)t * kc + k];
  }
}

// coef = scal[3] * sum_c ( sum_slices red[.][2][c] - bias[c] * sum_slices red[.][1][c] )
// red = the activation-backward statistics of the layer's output ([SG_STAT_SLICES][3][C] doubles: [1] = sum g_pre,
// [2] = sum g_pre * x with x the stored pre-activation = W~ * h + bias).  Because the layer output is linear in the
// normalised weight, <dL/dW~, W~> = <g_pre, x - bias>: the scalar of the sigma term needs no second pass over dW.
__global__ void snorm_coef_kernel(const double* __restrict__ red, const float* __restrict__ bias, int C,
                                  const float* __restrict__ scal, float* __restrict__ coef) {
  __shared__ double sh[256];
  double acc = 0;
  for (int c = threadIdx.x; c < C; c += 256) {
    double s1 = 0, s2 = 0;
    for (int i = 0; i < SG_STAT_SLICES; ++i) {
      s1 += red[((int64_t)i * 3 + 1) * C + c];
      s2 += red[((int64_t)i * 3 + 2) * C + c];
    }
    acc += s2 - (bias ? (double)bias[c] : 0.0) * s1;
  }
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) *coef = (float)(sh[0] * (double)scal[3]);
}

// dwp[t][n][c * kc + k] -= sum_p coef[p] * u[p][n] * v[p][t][k]  for every copy c < n_copies, rows of ld floats
// (the sigma terms of P passes, one sweep; ld = kc and one copy: the plain packed layout)
__global__ void __launch_bounds__(256)
snorm_rank1_kernel(float* __restrict__ dwp, int T, int nc, int kc, int ld, int n_copies, int P,
                   const float* __restrict__ u, const float* __restrict__ v, const float* __restrict__ coef) {
  const int64_t total = (int64_t)T * nc * kc;
  const int64_t vstride = (int64_t)T * kc;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int k = (int)(i % kc);
    const int64_t r = i / kc;
    const int n = (int)(r % nc), t = (int)(r / nc);
    float corr = 0.f;
    for (int p = 0; p < P; ++p) corr = fmaf(coef[p] * u[(int64_t)p * nc + n], v[p * vstride + (int64_t)t * kc + k], corr);
    float* row = dwp + r * ld + k;
    for (int c = 0; c < n_copies; ++c) row[(int64_t)c * kc] -= corr;
  }
}

// ---- row-strided power iteration with fixed-order sums (sg_snorm_sigma_ld) ------------------------------------
// The matrix is M[t][n][k], k < kc, rows ld floats apart (ld > kc: one half of a tied [W | W] master).  No float
// atomics: every sum is reduced in an order fixed by the launch geometry, so sigma, u and v have the same bits on
// every run and every data-parallel rank that holds the same master.

// every thread of a 256-thread block returns the block's sum (fixed order: warp trees, then warps 0..7)
__device__ __forceinline__ float block_sum_256(float x, float* sh) {
  x = warp_sum(x);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = x;
  __syncthreads();
  float s = 0.f;
  for (int i = 0; i < 8; ++i) s += sh[i];
  __syncthreads();
  return s;
}

// vraw[t][k] = sum_n M[t][n][k] * u[n] ;  part[block] = sum over the block's columns of vraw^2
__global__ void __launch_bounds__(256)
snorm_ld_wt_u_kernel(const float* __restrict__ m, int nc, int kc, int ld, const float* __restrict__ u,
                     float* __restrict__ vraw, float* __restrict__ part) {
  __shared__ float sh[8];
  const int t = blockIdx.y;
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  float acc = 0.f;
  if (k < kc) {
    const float* p = m + (int64_t)t * nc * ld + k;
    for (int n = 0; n < nc; ++n) acc = fmaf(p[(int64_t)n * ld], __ldg(u + n), acc);
    vraw[(int64_t)t * kc + k] = acc;
  }
  const float s = block_sum_256(acc * acc, sh);
  if (threadIdx.x == 0) part[(int64_t)blockIdx.y * gridDim.x + blockIdx.x] = s;
}

// uraw[n] = sum_{t,k} M[t][n][k] * vraw[t][k] / max(sqrt(*n2v), eps)   (block = one row n; n2v may be NULL)
__global__ void __launch_bounds__(256)
snorm_ld_w_v_kernel(const float* __restrict__ m, int T, int nc, int kc, int ld, const float* __restrict__ vraw,
                    const float* __restrict__ n2v, float* __restrict__ uraw) {
  __shared__ float sh[8];
  const int n = blockIdx.x;
  float acc = 0.f;
  for (int t = 0; t < T; ++t) {
    const float* p = m + ((int64_t)t * nc + n) * ld;
    const float* v = vraw + (int64_t)t * kc;
    for (int k = threadIdx.x; k < kc; k += 256) acc = fmaf(p[k], v[k], acc);
  }
  const float s = block_sum_256(acc, sh);
  if (threadIdx.x == 0) uraw[n] = n2v ? s / fmaxf(sqrtf(*n2v), 1e-12f) : s;
}

// *out = sum_i a[i] * b[i]  (b NULL: sum_i a[i]); one 256-thread block
__global__ void __launch_bounds__(256)
snorm_ld_dot_kernel(const float* __restrict__ a, const float* __restrict__ b, int n, float* __restrict__ out) {
  __shared__ float sh[8];
  float acc = 0.f;
  for (int i = threadIdx.x; i < n; i += 256) acc = b ? fmaf(a[i], b[i], acc) : acc + a[i];
  const float s = block_sum_256(acc, sh);
  if (threadIdx.x == 0) *out = s;
}

}  // namespace sg

using namespace sg;
#define ST ((cudaStream_t)stream)

extern "C" int sg_snorm_coef(const double* red, const float* bias, int C, const float* scal, float* coef_out,
                             void* stream) {
  SG_CHECK_ARG(red && scal && coef_out && C > 0);
  snorm_coef_kernel<<<1, 256, 0, ST>>>(red, bias, C, scal, coef_out);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_snorm_rank1(float* dwp, int n_taps, int nc, int kc, int n_pass, const float* u, const float* v,
                              const float* coef, void* stream) {
  SG_CHECK_ARG(dwp && u && v && coef && n_pass >= 1);
  snorm_rank1_kernel<<<4 * NUM_SMS, 256, 0, ST>>>(dwp, n_taps, nc, kc, kc, 1, n_pass, u, v, coef);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_snorm_rank1_ld(float* dwp, int n_taps, int nc, int kc, int ld, int n_copies, int n_pass,
                                 const float* u, const float* v, const float* coef, void* stream) {
  SG_CHECK_ARG(dwp && u && v && coef && n_pass >= 1 && n_copies >= 1 && ld >= n_copies * kc);
  snorm_rank1_kernel<<<4 * NUM_SMS, 256, 0, ST>>>(dwp, n_taps, nc, kc, ld, n_copies, n_pass, u, v, coef);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

// sg_snorm_sigma on the row-strided matrix M[t][n][k < kc] (rows ld floats apart), with fixed-order sums.
// work: nc + n_taps * ceil(kc / 256) floats.
extern "C" int sg_snorm_sigma_ld(const float* m, int n_taps, int nc, int kc, int ld, float* u, float* v, float* scal,
                                 float* work, int training, void* stream) {
  SG_CHECK_ARG(m && u && v && scal && work && n_taps >= 1 && nc > 0 && kc > 0 && ld >= kc);
  const int nv = n_taps * kc;
  if (training) {
    dim3 g1((kc + 255) / 256, n_taps);
    float* part = work + nc;
    snorm_ld_wt_u_kernel<<<g1, 256, 0, ST>>>(m, nc, kc, ld, u, v, part);            // v <- W^T u (raw)
    SG_CHECK_LAUNCH();
    snorm_ld_dot_kernel<<<1, 256, 0, ST>>>(part, nullptr, (int)(g1.x * g1.y), scal + 0);
    SG_CHECK_LAUNCH();
    snorm_ld_w_v_kernel<<<nc, 256, 0, ST>>>(m, n_taps, nc, kc, ld, v, scal + 0, u);  // u <- W v / ||v|| (raw)
    SG_CHECK_LAUNCH();
    snorm_ld_dot_kernel<<<1, 256, 0, ST>>>(u, u, nc, scal + 1);
    SG_CHECK_LAUNCH();
    snorm_finish_kernel<<<((nv > nc ? nv : nc) + 255) / 256, 256, 0, ST>>>(u, nc, v, nv, scal, 1);
  } else {
    snorm_ld_w_v_kernel<<<nc, 256, 0, ST>>>(m, n_taps, nc, kc, ld, v, nullptr, work);
    SG_CHECK_LAUNCH();
    snorm_ld_dot_kernel<<<1, 256, 0, ST>>>(u, work, nc, scal + 1);
    SG_CHECK_LAUNCH();
    snorm_finish_kernel<<<1, 32, 0, ST>>>(u, nc, v, nv, scal, 0);
  }
  SG_CHECK_LAUNCH();
  return SG_OK;
}

// One power iteration (training != 0) or sigma from the stored vectors (training == 0) on M[T][nc][kc].
// u [nc], v [T*kc] (packed slots) are updated in place when training; scal: 4 floats of scratch + results
// (scal[2] = sigma, scal[3] = 1/sigma); work: nc + T*kc floats.
extern "C" int sg_snorm_sigma(const float* m, int n_taps, int nc, int kc, float* u, float* v, float* scal, float* work,
                              int training, void* stream) {
  SG_CHECK_ARG(m && u && v && scal && work && n_taps >= 1 && nc > 0 && kc > 0);
  const int nv = n_taps * kc;
  SG_CHECK_CUDA(cudaMemsetAsync(scal, 0, 4 * sizeof(float), ST));
  float* uraw = work;
  if (training) {
    float* vraw = v;                 // v is overwritten by W^T u, then normalised in place
    dim3 g1((kc + 255) / 256, n_taps);
    snorm_wt_u_kernel<<<g1, 256, 0, ST>>>(m, nc, kc, u, vraw, scal + 0);
    SG_CHECK_LAUNCH();
    snorm_w_v_kernel<<<nc, 256, 0, ST>>>(m, n_taps, nc, kc, vraw, scal + 0, u, scal + 1);
    SG_CHECK_LAUNCH();
    snorm_finish_kernel<<<((nv > nc ? nv : nc) + 255) / 256, 256, 0, ST>>>(u, nc, v, nv, scal, 1);
  } else {
    snorm_w_v_kernel<<<nc, 256, 0, ST>>>(m, n_taps, nc, kc, v, nullptr, uraw, scal + 0);   // scal[0] unused afterwards
    SG_CHECK_LAUNCH();
    SG_CHECK_CUDA(cudaMemsetAsync(scal, 0, 2 * sizeof(float), ST));
    snorm_dot_kernel<<<8, 256, 0, ST>>>(u, uraw, nc, scal + 1);
    SG_CHECK_LAUNCH();
    snorm_finish_kernel<<<1, 32, 0, ST>>>(u, nc, v, nv, scal, 0);
  }
  SG_CHECK_LAUNCH();
  return SG_OK;
}

// dWp (gradient w.r.t. the NORMALISED weight, packed) -> gradient w.r.t. weight_orig, in place.
// dot_ws: one float of scratch.
extern "C" int sg_snorm_grad(float* dwp, const float* m, int n_taps, int nc, int kc, const float* u, const float* v,
                             const float* scal, float* dot_ws, void* stream) {
  SG_CHECK_ARG(dwp && m && u && v && scal && dot_ws);
  const int64_t total = (int64_t)n_taps * nc * kc;
  SG_CHECK_CUDA(cudaMemsetAsync(dot_ws, 0, sizeof(float), ST));
  snorm_dot_kernel<<<4 * NUM_SMS, 256, 0, ST>>>(dwp, m, total, dot_ws);
  SG_CHECK_LAUNCH();
  snorm_grad_apply_kernel<<<4 * NUM_SMS, 256, 0, ST>>>(dwp, n_taps, nc, kc, u, v, scal, dot_ws);
  SG_CHECK_LAUNCH();
  return SG_OK;
}
