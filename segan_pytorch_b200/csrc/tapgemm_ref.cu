// CUDA-core (fp32 FFMA) implementation of the two tap-GEMM forms.  This is the validation /
// fallback back end (SG_BACKEND_FFMA): same operands, same HBM layouts and same semantics as
// the wgmma kernels in tapgemm_tc.cu, written the obvious way so that it can serve as an
// on-device cross-check for them.  It is NOT the performance path.
#include "common.cuh"

namespace sg {

struct TapRanges {
  int k_lo[NTAP], k_hi[NTAP], n_lo[NTAP], n_hi[NTAP];
};

struct FParams {
  const void* a0; const void* a1;
  int a0_c, a1_c, a_rows, a_halo, a_dtype;
  const void* w; int w_dtype, w_tap0;
  int kc, nc, d_lo, d_hi;
  TapRanges tr;
  void* out; int out_dtype, out_rows, out_halo, out_ld, out_col0;
  int m_lo, m_hi, n_lo, n_hi;
  const float* bias; int bias_mod;
  int batch, ksplit;
};

constexpr int TM = 64, TNn = 64, TK = 16;

// out[b,m,n] = bias + sum_d sum_kc A[b,m+d,kc] * Wp[d+4][n][kc]
__global__ void __launch_bounds__(256) tapgemm_f_ffma(FParams p) {
  __shared__ float As[TK][TM + 4];
  __shared__ float Ws[TK][TNn + 4];
  const int rows_m = p.m_hi - p.m_lo;
  const int mtiles = (rows_m + TM - 1) / TM;
  const int b = blockIdx.x / mtiles;
  const int m0 = p.m_lo + (blockIdx.x % mtiles) * TM;
  const int n0 = p.n_lo + blockIdx.y * TNn;
  const int ks = blockIdx.z;
  const int tid = threadIdx.x;
  const int tx = tid % 16, ty = tid / 16;   // tx -> n (4 each), ty -> m (4 each)
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  const int lrow = tid / 4, lk = (tid % 4) * 4;
  const int a_buf_rows = p.a_rows + 2 * p.a_halo;
  int step = 0;
  for (int d = p.d_lo; d <= p.d_hi; ++d) {
    const int ti = d + 4;
    if (n0 + TNn <= p.tr.n_lo[ti] || n0 >= p.tr.n_hi[ti]) continue;
    for (int k0 = p.tr.k_lo[ti]; k0 < p.tr.k_hi[ti]; k0 += TK, ++step) {
      if (step % p.ksplit != ks) continue;
      // A tile: rows m0+lrow+d, channels k0+lk..+3
      {
        const int m = m0 + lrow + d;
        const bool ok = (m >= -p.a_halo) && (m < p.a_rows + p.a_halo);
        const int kk = k0 + lk;
        const void* src = p.a0; int c = p.a0_c; int kc_local = kk;
        if (kk >= p.a0_c) { src = p.a1; c = p.a1_c; kc_local = kk - p.a0_c; }
        const int64_t base = ((int64_t)b * a_buf_rows + (m + p.a_halo)) * c + kc_local;
#pragma unroll
        for (int j = 0; j < 4; ++j) As[lk + j][lrow] = ok ? ld16(src, base + j, p.a_dtype) : 0.f;
      }
      {
        const int n = n0 + lrow;
        const int64_t base = ((int64_t)(ti - p.w_tap0) * p.nc + n) * p.kc + k0 + lk;
#pragma unroll
        for (int j = 0; j < 4; ++j) Ws[lk + j][lrow] = ld16(p.w, base + j, p.w_dtype);
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < TK; ++k) {
        float av[4], wv[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) av[i] = As[k][ty * 4 + i];
#pragma unroll
        for (int j = 0; j < 4; ++j) wv[j] = Ws[k][tx * 4 + j];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], wv[j], acc[i][j]);
      }
      __syncthreads();
    }
  }
  const int out_buf_rows = p.out_rows + 2 * p.out_halo;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= p.m_hi) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      float v = acc[i][j];
      if (p.bias && ks == 0) v += p.bias[n % p.bias_mod];
      const int64_t o = ((int64_t)b * out_buf_rows + (m + p.out_halo)) * p.out_ld + (n - p.n_lo + p.out_col0);
      // fp32: an interleaved k-split (ksplit > 1) accumulates into the caller's destination, ksplit = 1 overwrites
      // it (as the tensor-core epilogue does); fp16 saturates at +-65504 like the tensor-core stores
      if (p.out_dtype == SG_F32) {
        float* dst = reinterpret_cast<float*>(p.out) + o;
        if (p.ksplit > 1) atomicAdd(dst, v);
        else *dst = v;
      } else {
        st16(p.out, o, v, p.out_dtype);
      }
    }
  }
}

struct WParams {
  const void* g; int g_rows, g_dtype;
  const void* a0; const void* a1;
  int a0_c, a1_c, a_rows, a_halo, a_dtype;
  int kc, nc, d_lo, d_hi;
  TapRanges tr;
  float* dw; int dw_tap0;
  int batch, ksplit;
  const float* out_scale;
};

// dWp[d+4][n][kc] += sum_{b,m} G[b,m,n] * A[b,m+d,kc]
__global__ void __launch_bounds__(256) tapgemm_w_ffma(WParams p) {
  __shared__ float Gs[TK][TNn + 4];
  __shared__ float As[TK][TM + 4];
  const int kc0 = blockIdx.x * TM;          // kc tile (64)
  const int ntiles = p.nc / TNn;
  const int n0 = (blockIdx.y % ntiles) * TNn;
  const int d = p.d_lo + blockIdx.y / ntiles;
  const int ti = d + 4;
  if (n0 + TNn <= p.tr.n_lo[ti] || n0 >= p.tr.n_hi[ti]) return;
  if (kc0 + TM <= p.tr.k_lo[ti] || kc0 >= p.tr.k_hi[ti]) return;
  const int tid = threadIdx.x;
  const int tx = tid % 16, ty = tid / 16;   // tx -> kc (4), ty -> n (4)
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  const int64_t total = (int64_t)p.batch * p.g_rows;
  const int64_t per = cdiv(cdiv(total, p.ksplit), TK) * TK;
  const int64_t q_lo = per * blockIdx.z;
  const int64_t q_hi = (q_lo + per < total) ? q_lo + per : total;
  const int a_buf_rows = p.a_rows + 2 * p.a_halo;
  const int lp = tid / 16, lc = (tid % 16) * 4;   // position within chunk, channel offset
  const void* asrc = p.a0; int ac = p.a0_c; int akc = kc0;
  if (kc0 >= p.a0_c) { asrc = p.a1; ac = p.a1_c; akc = kc0 - p.a0_c; }
  for (int64_t q0 = q_lo; q0 < q_hi; q0 += TK) {
    const int64_t q = q0 + lp;
    const bool okq = q < q_hi;
    const int b = okq ? (int)(q / p.g_rows) : 0;
    const int m = okq ? (int)(q % p.g_rows) : 0;
    {
      const int64_t base = ((int64_t)b * p.g_rows + m) * p.nc + n0 + lc;
#pragma unroll
      for (int j = 0; j < 4; ++j) Gs[lp][lc + j] = okq ? ld16(p.g, base + j, p.g_dtype) : 0.f;
    }
    {
      const int ma = m + d;
      const bool ok = okq && (ma >= -p.a_halo) && (ma < p.a_rows + p.a_halo);
      const int64_t base = ((int64_t)b * a_buf_rows + (ma + p.a_halo)) * ac + akc + lc;
#pragma unroll
      for (int j = 0; j < 4; ++j) As[lp][lc + j] = ok ? ld16(asrc, base + j, p.a_dtype) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < TK; ++k) {
      float gv[4], av[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) gv[i] = Gs[k][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) av[j] = As[k][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(gv[i], av[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + ty * 4 + i, kc = kc0 + tx * 4 + j;
      atomicAdd(p.dw + ((int64_t)(ti - p.dw_tap0) * p.nc + n) * p.kc + kc,
                acc[i][j] * (p.out_scale ? *p.out_scale : 1.f));
    }
}

int tapgemm_f_ffma_launch(const sg_tapgemm_f* q, cudaStream_t st) {
  FParams p;
  p.a0 = q->a0; p.a1 = q->a1; p.a0_c = q->a0_c; p.a1_c = q->a1_c;
  p.a_rows = q->a_rows; p.a_halo = q->a_halo; p.a_dtype = q->a_dtype;
  p.w = q->w; p.w_dtype = q->w_dtype; p.w_tap0 = q->w_tap0; p.kc = q->kc; p.nc = q->nc;
  p.d_lo = q->d_lo; p.d_hi = q->d_hi;
  for (int i = 0; i < NTAP; ++i) {
    p.tr.k_lo[i] = q->tap_k_lo[i]; p.tr.k_hi[i] = q->tap_k_hi[i];
    p.tr.n_lo[i] = q->tap_n_lo[i]; p.tr.n_hi[i] = q->tap_n_hi[i];
  }
  p.out = q->out; p.out_dtype = q->out_dtype; p.out_rows = q->out_rows; p.out_halo = q->out_halo;
  p.out_ld = q->out_ld > 0 ? q->out_ld : q->nc;
  p.out_col0 = q->out_ld > 0 ? q->out_col0 : q->n_lo;
  p.m_lo = q->m_lo; p.m_hi = q->m_hi; p.n_lo = q->n_lo; p.n_hi = q->n_hi;
  p.bias = q->bias; p.bias_mod = q->bias_mod > 0 ? q->bias_mod : q->nc;
  p.batch = q->batch; p.ksplit = q->ksplit < 1 ? 1 : q->ksplit;
  const int mtiles = (q->m_hi - q->m_lo + TM - 1) / TM;
  dim3 grid(q->batch * mtiles, (q->n_hi - q->n_lo) / TNn, p.ksplit);
  tapgemm_f_ffma<<<grid, 256, 0, st>>>(p);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

int tapgemm_w_ffma_launch(const sg_tapgemm_w* q, cudaStream_t st) {
  WParams p;
  p.g = q->g; p.g_rows = q->g_rows; p.g_dtype = q->g_dtype;
  p.a0 = q->a0; p.a1 = q->a1; p.a0_c = q->a0_c; p.a1_c = q->a1_c;
  p.a_rows = q->a_rows; p.a_halo = q->a_halo; p.a_dtype = q->a_dtype;
  p.kc = q->kc; p.nc = q->nc; p.d_lo = q->d_lo; p.d_hi = q->d_hi;
  for (int i = 0; i < NTAP; ++i) {
    p.tr.k_lo[i] = q->tap_k_lo[i]; p.tr.k_hi[i] = q->tap_k_hi[i];
    p.tr.n_lo[i] = q->tap_n_lo[i]; p.tr.n_hi[i] = q->tap_n_hi[i];
  }
  p.dw = q->dw; p.dw_tap0 = q->dw_tap0; p.batch = q->batch; p.ksplit = q->ksplit < 1 ? 1 : q->ksplit;
  p.out_scale = q->out_scale;
  dim3 grid(q->kc / TM, (q->nc / TNn) * (q->d_hi - q->d_lo + 1), p.ksplit);
  tapgemm_w_ffma<<<grid, 256, 0, st>>>(p);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

}  // namespace sg
