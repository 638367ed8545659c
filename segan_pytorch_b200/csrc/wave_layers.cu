// Waveform-end layers: the first encoder conv (Cin = 1 | 2) and the last decoder deconv
// (Cout = 1) and all of their gradients.  These are the HBM-bound ends of the U-Net
// (SURVEY.md App. A: G.enc0, D.enc0, G.dec4): K = Cin*31 <= 62 is far too thin for a
// 128-wide UMMA, so they run on CUDA cores as three generic stride-4 / 31-tap primitives:
//
//   analysis   out[b][t][c]  = bias[c] + sum_i sum_k W[c][i][k] * pad(v_i)[b][4t + k - off]
//   synthesis  out[b][4m+r]  = sum_c sum_d T[b][m+d][c] * W[c][-4d + r + off]
//   correlate  out[c][i][k] += sum_{b,t} T[b][t][c] * pad(v_i)[b][4t + k - off]
//
// v_i are fp32 waveforms [B][L]; T are 16-bit NLC tensors [B][L/4][C] (optionally the channel
// concatenation of two tensors).  pad() is either zero padding (transposed conv) or the
// reference's reflect padding preceded by the discriminator's circular phase shift.
#include "common.cuh"

namespace sg {

enum { PAD_ZERO = 0, PAD_REFLECT = 1 };

__device__ __forceinline__ float wave_at(const float* v, int64_t boff, int pos, int L, int mode, int roll) {
  if (mode == PAD_ZERO) return (pos < 0 || pos >= L) ? 0.f : v[boff + pos];
  if (pos < -(L - 1) || pos > 2 * (L - 1)) return 0.f;
  const int i = reflect_idx(pos, L);
  return v[boff + unroll_idx(i, roll, L)];
}

// ------------------------------------------------------------------------------------------
// analysis: 256 threads = C channels x (256/C) groups of 16 output positions
// ------------------------------------------------------------------------------------------
template <int C>
__global__ void __launch_bounds__(256)
wave_analysis_kernel(const float* __restrict__ v0, const float* __restrict__ v1, int cin, int L, int roll,
                     int mode, int off, const float* __restrict__ W, const float* __restrict__ bias,
                     void* __restrict__ a_out, int a_dtype, const float* __restrict__ prelu,
                     void* __restrict__ h_out) {
  constexpr int G = 256 / C;      // position groups
  constexpr int TT = G * 16;      // output positions per block
  __shared__ float xs[2][4 * TT + 32];
  __shared__ float ws[2 * KW][C];
  const int Lq = L / 4;
  const int b = blockIdx.y;
  const int t0 = blockIdx.x * TT;
  const int tid = threadIdx.x;
  for (int i = tid; i < cin * (4 * TT + 32); i += 256) {
    const int ci = i / (4 * TT + 32), q = i % (4 * TT + 32);
    const float* v = ci == 0 ? v0 : v1;
    xs[ci][q] = wave_at(v, (int64_t)b * L, 4 * t0 + q - off, L, mode, roll);
  }
  for (int i = tid; i < cin * KW * C; i += 256) {
    const int c = i / (cin * KW), r = i % (cin * KW);   // W[c][ci][k]
    ws[r][c] = W[i];
  }
  __syncthreads();
  const int c = tid % C, tg = tid / C;
  float acc[16];
  const float bv = bias ? bias[c] : 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) acc[i] = bv;
  for (int ci = 0; ci < cin; ++ci) {
    float xr[4 * 15 + KW + 1];
#pragma unroll
    for (int j = 0; j < 4 * 15 + KW; ++j) xr[j] = xs[ci][4 * tg * 16 + j];
#pragma unroll
    for (int k = 0; k < KW; ++k) {
      const float w = ws[ci * KW + k][c];
#pragma unroll
      for (int i = 0; i < 16; ++i) acc[i] = fmaf(w, xr[4 * i + k], acc[i]);
    }
  }
  const float slope = prelu ? prelu[c] : 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const int t = t0 + tg * 16 + i;
    if (t >= Lq) continue;
    st16(a_out, ((int64_t)b * Lq + t) * C + c, acc[i], a_dtype);
    if (h_out) {
      // consumer-ready view of the next conv: 16 halo positions each side, reflect-mirrored
      const float h = acc[i] > 0.f ? acc[i] : slope * acc[i];
      const int64_t hb = (int64_t)b * (Lq + 32) + 16;
      st16(h_out, (hb + t) * C + c, h, a_dtype);
      if (t >= 1 && t <= 16) st16(h_out, (hb - t) * C + c, h, a_dtype);
      if (t >= Lq - 17 && t <= Lq - 2) st16(h_out, (hb + 2 * (Lq - 1) - t) * C + c, h, a_dtype);
    }
  }
}

// ------------------------------------------------------------------------------------------
// synthesis: block = 32 rows m (128 outputs); thread = (m, channel slice of C/8, interleaved)
// ------------------------------------------------------------------------------------------
template <int C>
__global__ void __launch_bounds__(256)
wave_synthesis_kernel(const void* __restrict__ T0, int c0, const void* __restrict__ T1, int t_dtype, int Lq,
                      const float* __restrict__ W, int w_stride, int off, const float* __restrict__ bias,
                      int m_lo, int m_hi, int mode /*0: tanh -> y ; 1: fold/unroll atomics*/, int roll,
                      float* __restrict__ out, int L) {
  constexpr int CP = C + 8;
  __shared__ float ts[40][CP];
  __shared__ __align__(16) float w2[C][36];   // w2[c][j] = W[c][j + off - 16], zero outside [0,30]
  const int b = blockIdx.y;
  const int m0 = m_lo + blockIdx.x * 32;
  const int tid = threadIdx.x;
  for (int i = tid; i < 40 * C; i += 256) {
    const int r = i / C, c = i % C;
    const int m = m0 - 4 + r;
    float v = 0.f;
    if (m >= 0 && m < Lq) {
      if (c < c0) v = ld16(T0, ((int64_t)b * Lq + m) * c0 + c, t_dtype);
      else v = ld16(T1, ((int64_t)b * Lq + m) * (C - c0) + (c - c0), t_dtype);
    }
    ts[r][c] = v;
  }
  for (int i = tid; i < C * 36; i += 256) {
    const int c = i / 36, j = i % 36;
    const int k = j + off - 16;
    w2[c][j] = (k >= 0 && k < KW) ? W[(int64_t)c * w_stride + k] : 0.f;
  }
  __syncthreads();
  const int slice = tid % 8, ml = tid / 8;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  // out[4m + r] = sum_d sum_c T[m+d][c] * W[c][-4d + r + off];  j = -4d + r + 16 in [0, 36)
#pragma unroll
  for (int d = -4; d <= 4; ++d) {
    const float* trow = ts[ml + 4 + d];
    const int j0 = -4 * d + 16;
#pragma unroll 4
    for (int cc = 0; cc < C / 8; ++cc) {
      const int c = cc * 8 + slice;
      const float t = trow[c];
      const float4 w = *reinterpret_cast<const float4*>(&w2[c][j0]);
      acc[0] = fmaf(t, w.x, acc[0]);
      acc[1] = fmaf(t, w.y, acc[1]);
      acc[2] = fmaf(t, w.z, acc[2]);
      acc[3] = fmaf(t, w.w, acc[3]);
    }
  }
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], 1);
    acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], 2);
    acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], 4);
  }
  const int m = m0 + ml;
  if (slice < 4 && m < m_hi) {
    const int r = slice;
    float v = acc[0];
    if (r == 1) v = acc[1];
    if (r == 2) v = acc[2];
    if (r == 3) v = acc[3];
    const int q = 4 * m + r;
    if (mode == 0) {
      if (bias) v += bias[0];
      out[(int64_t)b * L + q] = tanhf(v);
    } else {
      if (q >= -14 && q <= L + 15) {
        const int i = reflect_idx(q, L);
        atomicAdd(out + (int64_t)b * L + unroll_idx(i, roll, L), v);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// correlate: persistent blocks, register accumulators, one atomic flush per block
// ------------------------------------------------------------------------------------------
template <int C>
__global__ void __launch_bounds__(256)
wave_correlate_kernel(const void* __restrict__ T0, int c0, const void* __restrict__ T1, int t_dtype,
                      const float* __restrict__ v0, const float* __restrict__ v1, int cin, int batch, int L,
                      int roll, int mode, int off, float* __restrict__ out /*[C][cin][31]*/,
                      float* __restrict__ colsum /*[C] or null*/) {
  constexpr int G = 256 / C;       // tap groups
  constexpr int KG = 32 / G;       // taps per group (8 or 16)
  constexpr int TT = 64;
  __shared__ float ts[TT][C];
  __shared__ __align__(16) float xs[2][4 * TT + 32];
  const int Lq = L / 4;
  const int tiles_per_b = (Lq + TT - 1) / TT;
  const int total = batch * tiles_per_b;
  const int tid = threadIdx.x;
  const int c = tid % C, kg = tid / C;
  float acc[2][KG];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < KG; ++j) acc[i][j] = 0.f;
  float csum = 0.f;
  for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
    const int b = tile / tiles_per_b, t0 = (tile % tiles_per_b) * TT;
    __syncthreads();
    for (int i = tid; i < TT * C; i += 256) {
      const int r = i / C, cc = i % C;
      const int t = t0 + r;
      float v = 0.f;
      if (t < Lq) {
        if (cc < c0) v = ld16(T0, ((int64_t)b * Lq + t) * c0 + cc, t_dtype);
        else v = ld16(T1, ((int64_t)b * Lq + t) * (C - c0) + (cc - c0), t_dtype);
      }
      ts[r][cc] = v;
    }
    for (int i = tid; i < cin * (4 * TT + 32); i += 256) {
      const int ci = i / (4 * TT + 32), q = i % (4 * TT + 32);
      xs[ci][q] = wave_at(ci == 0 ? v0 : v1, (int64_t)b * L, 4 * t0 + q - off, L, mode, roll);
    }
    __syncthreads();
#pragma unroll
    for (int ci = 0; ci < 2; ++ci) {
      if (ci >= cin) break;
#pragma unroll 4
      for (int t = 0; t < TT; ++t) {
        const float g = ts[t][c];
        if (ci == 0 && kg == 0) csum += g;
        const float4* xp = reinterpret_cast<const float4*>(&xs[ci][4 * t + kg * KG]);
#pragma unroll
        for (int j = 0; j < KG / 4; ++j) {
          const float4 x = xp[j];
          acc[ci][4 * j + 0] = fmaf(g, x.x, acc[ci][4 * j + 0]);
          acc[ci][4 * j + 1] = fmaf(g, x.y, acc[ci][4 * j + 1]);
          acc[ci][4 * j + 2] = fmaf(g, x.z, acc[ci][4 * j + 2]);
          acc[ci][4 * j + 3] = fmaf(g, x.w, acc[ci][4 * j + 3]);
        }
      }
    }
  }
#pragma unroll
  for (int ci = 0; ci < 2; ++ci) {
    if (ci >= cin) break;
#pragma unroll
    for (int j = 0; j < KG; ++j) {
      const int k = kg * KG + j;
      if (k < KW) atomicAdd(out + ((int64_t)c * cin + ci) * KW + k, acc[ci][j]);
    }
  }
  if (colsum && kg == 0) atomicAdd(colsum + c, csum);
}

static int grid_persistent() { return 2 * NUM_SMS; }

}  // namespace sg

using namespace sg;

extern "C" int sg_wave_conv_fwd(const float* x0, const float* x1, int cin, int batch, int L, int roll,
                                const float* w, const float* bias, int cout, void* a_out, const float* prelu,
                                void* h_out, void* stream) {
  SG_CHECK_ARG(cout == 64 && (cin == 1 || cin == 2) && L % 64 == 0 && L >= 64);
  SG_CHECK_ARG(x0 && (cin == 1 || x1) && w && a_out);
  dim3 grid((unsigned)cdiv(L / 4, 64), batch);
  wave_analysis_kernel<64><<<grid, 256, 0, (cudaStream_t)stream>>>(x0, x1, cin, L, roll, PAD_REFLECT, 14, w, bias,
                                                                   a_out, SG_F16, prelu, h_out);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_wave_conv_wgrad(const float* x0, const float* x1, int cin, int batch, int L, int roll,
                                  const void* g_a, int cout, float* dw, float* dbias, void* stream) {
  SG_CHECK_ARG(cout == 64 && (cin == 1 || cin == 2) && L % 64 == 0);
  wave_correlate_kernel<64><<<grid_persistent(), 256, 0, (cudaStream_t)stream>>>(
      g_a, 64, nullptr, g_grad_dtype, x0, x1, cin, batch, L, roll, PAD_REFLECT, 14, dw, dbias);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_wave_conv_dgrad(const void* g_a, int batch, int L, int roll, const float* w, int cin, int cout,
                                  float* gx0, int accumulate, void* stream) {
  SG_CHECK_ARG(cout == 64 && L % 64 == 0);
  cudaStream_t st = (cudaStream_t)stream;
  if (!accumulate) SG_CHECK_CUDA(cudaMemsetAsync(gx0, 0, sizeof(float) * (size_t)batch * L, st));
  const int Lq = L / 4;
  dim3 grid((unsigned)cdiv(Lq + 8, 32), batch);
  wave_synthesis_kernel<64><<<grid, 256, 0, st>>>(g_a, 64, nullptr, g_grad_dtype, Lq, w, cin * KW, 14, nullptr, -4,
                                                  Lq + 4, 1, roll, gx0, L);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_wave_deconv_fwd(const void* x0, int c0, const void* x1, int c1, int batch, int Lin,
                                  const float* w_eff, const float* bias, float* y, void* stream) {
  SG_CHECK_ARG(c0 + c1 == 128 && Lin % 32 == 0);
  dim3 grid((unsigned)cdiv(Lin, 32), batch);
  wave_synthesis_kernel<128><<<grid, 256, 0, (cudaStream_t)stream>>>(x0, c0, x1, SG_F16, Lin, w_eff, KW, 13, bias,
                                                                     0, Lin, 0, 0, y, 4 * Lin);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

namespace sg {
// gpre = gy * (1 - y^2)
__global__ void tanh_bwd_kernel(const float* __restrict__ gy, const float* __restrict__ y, float* __restrict__ gpre,
                                int64_t n, float* __restrict__ dbias) {
  float s = 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float yy = y[i];
    const float g = gy[i] * (1.f - yy * yy);
    gpre[i] = g;
    s += g;
  }
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0 && dbias) atomicAdd(dbias, s);
}
}  // namespace sg

// gpre_ws: caller-provided fp32 workspace [B][4*Lin] receiving gy * (1 - y^2)
extern "C" int sg_wave_deconv_bwd(const void* x0, int c0, const void* x1, int c1, int batch, int Lin,
                                     const float* w_eff, const float* gy, const float* y, float* gpre_ws,
                                     void* gx, float* dw_eff, float* dbias, void* stream) {
  SG_CHECK_ARG(c0 + c1 == 128 && Lin % 64 == 0 && gpre_ws);
  cudaStream_t st = (cudaStream_t)stream;
  const int L = 4 * Lin;
  const int64_t n = (int64_t)batch * L;
  tanh_bwd_kernel<<<2 * NUM_SMS, 256, 0, st>>>(gy, y, gpre_ws, n, dbias);
  SG_CHECK_LAUNCH();
  if (gx) {
    // gx[b][j][ci] = sum_k gpre[4j + k - 13] * w_eff[ci][k]   (zero padding)
    dim3 grid((unsigned)cdiv(Lin, 32), batch);
    wave_analysis_kernel<128><<<grid, 256, 0, st>>>(gpre_ws, nullptr, 1, L, 0, PAD_ZERO, 13, w_eff, nullptr, gx,
                                                    g_grad_dtype, nullptr, nullptr);
    SG_CHECK_LAUNCH();
  }
  if (dw_eff) {
    wave_correlate_kernel<128><<<grid_persistent(), 256, 0, st>>>(x0, c0, x1, SG_F16, gpre_ws, nullptr, 1, batch, L,
                                                                  0, PAD_ZERO, 13, dw_eff, nullptr);
    SG_CHECK_LAUNCH();
  }
  return SG_OK;
}

// ==========================================================================================
// Tensor-core route for the waveform-end layers: a 64-channel im2col of the waveform(s) turns
// the K = Cin*31 convs into single-tap tap-GEMMs (K = 64) on the wgmma kernels; the
// transposed forms are a GEMM followed by a shift-add ("col2im").  These three kernels are the
// HBM-bound glue around those GEMMs.
// ==========================================================================================
namespace sg {

// col[b][t][ci*32 + k] = pad(v_ci)[4t + k - off]   (k < kw <= 32; columns k >= kw and absent channels = 0)
__global__ void __launch_bounds__(256)
wave_im2col_kernel(const float* __restrict__ v0, const float* __restrict__ v1, int cin, int batch, int L, int roll,
                   const int* __restrict__ roll_dev,
                   int mode, int off, int kw, void* __restrict__ col_f16, void* __restrict__ col_bf16) {
  if (roll_dev) roll = *roll_dev;
  const int Lq = L / 4;
  const int64_t total = (int64_t)batch * Lq * 8;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int seg = (int)(i % 8);
    const int64_t row = i / 8;
    const int t = (int)(row % Lq), b = (int)(row / Lq);
    const int ci = seg / 4, k0 = (seg % 4) * 8;
    V8 o16, ob;
    const float* v = ci == 0 ? v0 : v1;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = k0 + j;
      float x = 0.f;
      if (ci < cin && k < kw) x = wave_at(v, (int64_t)b * L, 4 * t + k - off, L, mode, roll);
      o16.v[j] = cvt16(x, SG_F16);
      ob.v[j] = cvt16(x, SG_BF16);
    }
    if (col_f16) *reinterpret_cast<V8*>(reinterpret_cast<uint16_t*>(col_f16) + row * 64 + seg * 8) = o16;
    if (col_bf16) *reinterpret_cast<V8*>(reinterpret_cast<uint16_t*>(col_bf16) + row * 64 + seg * 8) = ob;
  }
}

// The same matrix, one block per IM2_T rows of one batch element: the waveform segment the rows cover is staged in
// shared memory once (reflect / zero padding and the circular phase shift resolved per INPUT sample: 8x fewer index
// computations than per output element, which made the kernel above instruction-bound at 1.5 TB/s), then every
// thread assembles 16-byte output vectors from shared memory.
constexpr int IM2_T = 256;
__global__ void __launch_bounds__(256)
wave_im2col_tiled_kernel(const float* __restrict__ v0, const float* __restrict__ v1, int cin, int L, int roll,
                         const int* __restrict__ roll_dev, int mode, int off, int kw, uint16_t* __restrict__ col_f16,
                         uint16_t* __restrict__ col_bf16) {
  constexpr int SEG = 4 * IM2_T + 32;            // input samples one tile touches (4 t + k, k < 32), padded
  __shared__ float xs[2][SEG + 4];
  if (roll_dev) roll = *roll_dev;
  const int Lq = L / 4;
  const int b = blockIdx.y;
  const int t0 = blockIdx.x * IM2_T;
  const int tid = threadIdx.x;
  for (int i = tid; i < cin * SEG; i += 256) {
    const int ci = i >= SEG ? 1 : 0, q = i - ci * SEG;
    xs[ci][q] = wave_at(ci == 0 ? v0 : v1, (int64_t)b * L, 4 * t0 + q - off, L, mode, roll);
  }
  __syncthreads();
  const int rows = min(IM2_T, Lq - t0);
  for (int i = tid; i < rows * 8; i += 256) {
    const int seg = i & 7, r = i >> 3;
    const int ci = seg >> 2, k0 = (seg & 3) * 8;
    float x[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) x[j] = (ci < cin && k0 + j < kw) ? xs[ci][4 * r + k0 + j] : 0.f;
    const int64_t o = ((int64_t)b * Lq + t0 + r) * 64 + seg * 8;
    if (col_f16) {
      uint32_t w[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        __half2 h2 = __floats2half2_rn(x[2 * j], x[2 * j + 1]);
        w[j] = *reinterpret_cast<uint32_t*>(&h2);
      }
      *reinterpret_cast<uint4*>(col_f16 + o) = make_uint4(w[0], w[1], w[2], w[3]);
    }
    if (col_bf16) {
      uint32_t w[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        __nv_bfloat162 h2 = __floats2bfloat162_rn(x[2 * j], x[2 * j + 1]);
        w[j] = *reinterpret_cast<uint32_t*>(&h2);
      }
      *reinterpret_cast<uint4*>(col_bf16 + o) = make_uint4(w[0], w[1], w[2], w[3]);
    }
  }
}

// y[b][4m + r] = tanh(bias + sum_d P[b][m + d][(d+4)*4 + r]),  P fp32 [B][Lin][64]
__global__ void __launch_bounds__(256)
wave_shiftadd_tanh_kernel(const float* __restrict__ P, int batch, int Lin, const float* __restrict__ bias,
                          float* __restrict__ y) {
  const int64_t total = (int64_t)batch * Lin * 4;
  const float bv = bias ? bias[0] : 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(i % 4);
    const int64_t mr = i / 4;
    const int m = (int)(mr % Lin), b = (int)(mr / Lin);
    float s = bv;
#pragma unroll
    for (int d = -4; d <= 4; ++d) {
      const int mm = m + d;
      if (mm >= 0 && mm < Lin) s += P[((int64_t)b * Lin + mm) * 64 + (d + 4) * 4 + r];
    }
    y[i] = tanhf(s);
  }
}

// gx[b][src(q)] += sum_{t,k < kw: 4t + k - off = q} P2[b][t][k]   (reflect fold + un-roll), P2 16-bit (gradient
// dtype) [B][Lq][64]; off = kw/2 - 1 is the left reflect pad, the right one is off + 1
__global__ void __launch_bounds__(256)
wave_col2im_fold_kernel(const void* __restrict__ P2, int gdt, int col0, int batch, int L, int roll,
                        const int* __restrict__ roll_dev, int off, int kw, float* __restrict__ gx) {
  if (roll_dev) roll = *roll_dev;
  const int Lq = L / 4;
  const int span = L + 2 * off + 2;                // q in [-off, L + off + 1]
  const int64_t total = (int64_t)batch * span;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int q = (int)(i % span) - off;
    const int b = (int)(i / span);
    const int e = q + off;                         // = 4t + k
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = (e & 3) + 4 * j;
      const int t = (e - k) / 4;
      if (k < kw && t >= 0 && t < Lq) s += ld16(P2, ((int64_t)b * Lq + t) * 64 + col0 + k, gdt);
    }
    const int src = unroll_idx(reflect_idx(q, L), roll, L);
    atomicAdd(gx + (int64_t)b * L + src, s);
  }
}

}  // namespace sg

extern "C" int sg_wave_im2col_kw(const float* v0, const float* v1, int cin, int batch, int L, int roll,
                                 const int32_t* roll_dev, int reflect, int off, int kw, void* col_f16, void* col_bf16,
                                 void* stream) {
  SG_CHECK_ARG(v0 && (cin == 1 || (cin == 2 && v1)) && L % 4 == 0 && (col_f16 || col_bf16) && kw_served(kw));
  if (batch <= 65535) {
    dim3 grid((unsigned)cdiv(L / 4, IM2_T), (unsigned)batch);
    wave_im2col_tiled_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(
        v0, v1, cin, L, roll, roll_dev, reflect ? PAD_REFLECT : PAD_ZERO, off, kw, reinterpret_cast<uint16_t*>(col_f16),
        reinterpret_cast<uint16_t*>(col_bf16));
    SG_CHECK_LAUNCH();
    return SG_OK;
  }
  const int64_t total = (int64_t)batch * (L / 4) * 8;
  int64_t g = cdiv(total, 256 * 4);
  if (g > 16 * NUM_SMS) g = 16 * NUM_SMS;
  wave_im2col_kernel<<<(int)g, 256, 0, (cudaStream_t)stream>>>(v0, v1, cin, batch, L, roll, roll_dev,
                                                              reflect ? PAD_REFLECT : PAD_ZERO, off, kw, col_f16,
                                                              col_bf16);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_wave_im2col(const float* v0, const float* v1, int cin, int batch, int L, int roll,
                              const int32_t* roll_dev, int reflect,
                              int off, void* col_f16, void* col_bf16, void* stream) {
  return sg_wave_im2col_kw(v0, v1, cin, batch, L, roll, roll_dev, reflect, off, KW, col_f16, col_bf16, stream);
}

extern "C" int sg_wave_shiftadd_tanh(const float* P, int batch, int Lin, const float* bias, float* y, void* stream) {
  const int64_t total = (int64_t)batch * Lin * 4;
  int64_t g = cdiv(total, 256 * 4);
  if (g > 16 * NUM_SMS) g = 16 * NUM_SMS;
  wave_shiftadd_tanh_kernel<<<(int)g, 256, 0, (cudaStream_t)stream>>>(P, batch, Lin, bias, y);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_wave_col2im_fold_kw(const void* P2, int col0, int batch, int L, int roll, const int32_t* roll_dev,
                                      int kw, float* gx, void* stream) {
  SG_CHECK_ARG(P2 && gx && kw_served(kw));
  const int off = kw / 2 - 1;
  const int64_t total = (int64_t)batch * (L + 2 * off + 2);
  int64_t g = cdiv(total, 256 * 4);
  if (g > 16 * NUM_SMS) g = 16 * NUM_SMS;
  wave_col2im_fold_kernel<<<(int)g, 256, 0, (cudaStream_t)stream>>>(P2, g_grad_dtype, col0, batch, L, roll, roll_dev,
                                                                    off, kw, gx);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_wave_col2im_fold(const void* P2, int col0, int batch, int L, int roll, const int32_t* roll_dev,
                                   float* gx, void* stream) {
  return sg_wave_col2im_fold_kw(P2, col0, batch, L, roll, roll_dev, KW, gx, stream);
}

// gpre = gy * (1 - y^2), dbias += sum gpre   (tanh backward of the last decoder block)
extern "C" int sg_tanh_bwd(const float* gy, const float* y, int64_t n, float* gpre, float* dbias, void* stream) {
  tanh_bwd_kernel<<<2 * NUM_SMS, 256, 0, (cudaStream_t)stream>>>(gy, y, gpre, n, dbias);
  SG_CHECK_LAUNCH();
  return SG_OK;
}
