// WSEGAN's spectral regression term (segan/models/model.py:638-653): pow_weight * L1 of the log-power spectrograms
// of the enhanced and the clean batch, torch.stft(n_fft 2048, hop 160, win_length 320 (rectangular, centred in the
// 2048 frame), center=True (reflect pad 1024), normalized) -> 10 log10(|X|^2 + 1e-19).
//
// With a rectangular 320-sample window only 320 of the 2048 frame samples are non-zero, so the transform of ALL
// frames is one dense GEMM on the tensor cores: frames [B*103][320] x DFT [320][re | im of 1025 bins] (fp16
// operands, fp32 out) -- the tap-GEMM with a single tap.  These kernels are the HBM-bound glue around the two
// GEMMs (forward, and the gradient back to the frames):
//   sg_stft_frames      waveform -> frames (the window's samples of every hop, reflect-padded ends), fp16
//   sg_logpow_l1        X_gen, X_clean (fp32 re | im) -> loss, dL/dX_gen (bf16: wide range, no loss scale needed)
//   sg_stft_frames_fold dL/dframes (fp32) -> += dL/dwaveform (overlap-add, reflect fold)
#include "common.cuh"

namespace sg {

constexpr int STFT_WIN = 320, STFT_HOP = 160, STFT_NFFT = 2048;
constexpr int STFT_OFF = (STFT_NFFT - STFT_WIN) / 2 - STFT_NFFT / 2;      // -160: window start relative to t * hop

__device__ __forceinline__ int stft_src(int t, int n, int L) {
  int s = t * STFT_HOP + n + STFT_OFF;
  if (s < 0) s = -s;
  if (s >= L) s = 2 * (L - 1) - s;
  return s;
}

__global__ void __launch_bounds__(256)
stft_frames_kernel(const float* __restrict__ x, int L, int frames, void* __restrict__ out, int dtype, int split) {
  const int b = blockIdx.y;
  const int64_t total = (int64_t)frames * STFT_WIN;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(i / STFT_WIN), n = (int)(i % STFT_WIN);
    const float v = x[(int64_t)b * L + stft_src(t, n, L)];
    if (!split) {
      st16(out, (int64_t)b * total + i, v, dtype);
    } else {
      // [hi | lo | hi]: v = hi + lo to ~22 bits; the K = 960 product against [Dhi ; Dhi ; Dlo] is hi Dhi + lo Dhi + hi Dlo
      const int64_t row = ((int64_t)b * frames + t) * (3 * STFT_WIN);
      const float hi = dtype == SG_F16 ? __half2float(__float2half_rn(v)) : __bfloat162float(__float2bfloat16_rn(v));
      st16(out, row + n, hi, dtype);
      st16(out, row + STFT_WIN + n, v - hi, dtype);
      st16(out, row + 2 * STFT_WIN + n, hi, dtype);
    }
  }
}

// X: [rows = B*frames][ld] fp32, re of bin f at column f, im at column half + f (f < bins)
__global__ void __launch_bounds__(256)
logpow_l1_kernel(const float* __restrict__ xg, const float* __restrict__ xc, int64_t rows, int bins, int half, int ld,
                 float weight, float* __restrict__ loss_out, void* __restrict__ gx, int gx_dtype, float gscale) {
  const int64_t total = rows * bins;
  const float wn = weight / (float)total;
  const float k10 = 4.342944819f;                    // 10 / ln(10)
  float acc = 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / bins;
    const int f = (int)(i % bins);
    const float re = xg[r * ld + f], im = xg[r * ld + half + f];
    const float rc = xc[r * ld + f], ic = xc[r * ld + half + f];
    const float pg = re * re + im * im + 1e-19f, pc = rc * rc + ic * ic + 1e-19f;
    // 10 log10(pg) - 10 log10(pc).  __fsub_rn keeps the subtraction out of an FMA with one logarithm's ln 2 scaling:
    // contracted, identical powers would leave that product's rounding error as d != 0 and a full-size gradient of
    // either sign where the reference's is 0
    const float d = k10 * __fsub_rn(__logf(pg), __logf(pc));
    acc += fabsf(d);
    if (gx) {
      // d/d re [10 log10(re^2 + im^2 + eps)] = (20 / ln 10) re / p
      const float s = (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f)) * wn * gscale * 2.f * k10 / pg;
      st16(gx, r * ld + f, s * re, gx_dtype);
      st16(gx, r * ld + half + f, s * im, gx_dtype);
    }
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0 && loss_out) atomicAdd(loss_out, acc * wn);
}

__global__ void __launch_bounds__(256)
stft_fold_kernel(const float* __restrict__ gf, int L, int frames, float scale, float* __restrict__ gy) {
  const int b = blockIdx.y;
  const int64_t total = (int64_t)frames * STFT_WIN;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(i / STFT_WIN), n = (int)(i % STFT_WIN);
    atomicAdd(gy + (int64_t)b * L + stft_src(t, n, L), scale * gf[(int64_t)b * total + i]);
  }
}

}  // namespace sg

using namespace sg;
#define ST ((cudaStream_t)stream)

// frames[b][t][n] = x[b][reflect(t*160 + n - 160)], t < 1 + L/160, n < 320 (16-bit); split: rows of 960 = hi | lo | hi
extern "C" int sg_stft_frames(const float* x, int batch, int L, void* frames, int dtype, int split, void* stream) {
  SG_CHECK_ARG(x && frames && batch > 0 && L > STFT_NFFT / 2 && (dtype == SG_F16 || dtype == SG_BF16));
  const int fr = 1 + L / STFT_HOP;
  dim3 grid((unsigned)cdiv((int64_t)fr * STFT_WIN, 256 * 4), batch);
  stft_frames_kernel<<<grid, 256, 0, ST>>>(x, L, fr, frames, dtype, split);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_logpow_l1(const float* x_gen, const float* x_clean, int64_t rows, int bins, int half, int ld,
                            float weight, float* loss_out, void* g_x, int g_dtype, float grad_scale, void* stream) {
  SG_CHECK_ARG(x_gen && x_clean && rows > 0 && bins > 0 && half >= bins && ld >= half + bins);
  SG_CHECK_ARG(!g_x || g_dtype == SG_F16 || g_dtype == SG_BF16);
  logpow_l1_kernel<<<4 * NUM_SMS, 256, 0, ST>>>(x_gen, x_clean, rows, bins, half, ld, weight, loss_out, g_x, g_dtype,
                                                grad_scale);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_stft_frames_fold(const float* g_frames, int batch, int L, float scale, float* g_wave, void* stream) {
  SG_CHECK_ARG(g_frames && g_wave && batch > 0 && L > STFT_NFFT / 2);
  const int fr = 1 + L / STFT_HOP;
  dim3 grid((unsigned)cdiv((int64_t)fr * STFT_WIN, 256 * 4), batch);
  stft_fold_kernel<<<grid, 256, 0, ST>>>(g_frames, L, fr, scale, g_wave);
  SG_CHECK_LAUNCH();
  return SG_OK;
}
