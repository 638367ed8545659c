// Optimisers on flat fp32 parameter buffers, weight packing into the 16-bit tap-GEMM operand
// layouts, gradient unpacking, and the inference-side emphasis filters.
#include "common.cuh"

namespace sg {

// 16-bit or fp32 destination element (the packed fp32 MASTER is written with SG_F32)
__device__ __forceinline__ void st_any(void* p, int64_t i, float v, int dtype) {
  if (dtype == SG_F32) reinterpret_cast<float*>(p)[i] = v;
  else st16(p, i, v, dtype);
}

// ------------------------------------------------------------------------------------------
// torch.optim.RMSprop (centered=False, momentum=0, weight_decay=0):
//   sq = alpha*sq + (1-alpha)*g*g ; p -= lr * g / (sqrt(sq) + eps)
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
rmsprop_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ sq,
               int64_t n, float lr, float alpha, float eps, float gscale, int clear) {
  // two float4 per stream and thread in flight (6 x 16 B loads before the first use): the kernel is pure streaming,
  // 24 B per parameter with the clear-on-read store
  const int64_t n4 = n / 4;
  float4* p4 = reinterpret_cast<float4*>(p);
  float4* g4 = reinterpret_cast<float4*>(g);
  float4* s4 = reinterpret_cast<float4*>(sq);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += 2 * stride) {
    const int64_t i2 = i + stride;
    const bool two = i2 < n4;
    float4 pv[2], gv[2], sv[2];
    pv[0] = p4[i]; gv[0] = g4[i]; sv[0] = s4[i];
    if (two) { pv[1] = p4[i2]; gv[1] = g4[i2]; sv[1] = s4[i2]; }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      if (u == 1 && !two) break;
      float* pp = &pv[u].x; float* gp = &gv[u].x; float* sp = &sv[u].x;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float gi = gp[j] * gscale;
        const float s = alpha * sp[j] + (1.f - alpha) * gi * gi;
        sp[j] = s;
        pp[j] = pp[j] - lr * (gi / (sqrtf(s) + eps));
      }
      const int64_t k = u == 0 ? i : i2;
      p4[k] = pv[u];
      s4[k] = sv[u];
      if (clear) g4[k] = make_float4(0.f, 0.f, 0.f, 0.f);   // clear-on-read: the next backward accumulates from zero
    }
  }
  for (int64_t i = n4 * 4 + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) {
    const float gi = g[i] * gscale;
    if (clear) g[i] = 0.f;
    const float s = alpha * sq[i] + (1.f - alpha) * gi * gi;
    sq[i] = s;
    p[i] = p[i] - lr * (gi / (sqrtf(s) + eps));
  }
}
// torch.optim.Adam (amsgrad=False, weight_decay=0)
__global__ void __launch_bounds__(256)
adam_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, int64_t n,
            float lr, float b1, float b2, float eps, float bc1, float bc2_sqrt, float gscale, int clear) {
  const int64_t n4 = n / 4;
  float4* p4 = reinterpret_cast<float4*>(p);
  float4* g4 = reinterpret_cast<float4*>(g);
  float4* m4 = reinterpret_cast<float4*>(m);
  float4* v4 = reinterpret_cast<float4*>(v);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const float step = lr / bc1;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 pv = p4[i], gv = g4[i], mv = m4[i], vv = v4[i];
    float* pp = &pv.x; float* gp = &gv.x; float* mp = &mv.x; float* vp = &vv.x;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float gi = gp[j] * gscale;
      const float mi = b1 * mp[j] + (1.f - b1) * gi;
      const float vi = b2 * vp[j] + (1.f - b2) * gi * gi;
      mp[j] = mi;
      vp[j] = vi;
      pp[j] = pp[j] - step * (mi / (sqrtf(vi) / bc2_sqrt + eps));
    }
    p4[i] = pv; m4[i] = mv; v4[i] = vv;
    if (clear) g4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  for (int64_t i = n4 * 4 + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) {
    const float gi = g[i] * gscale;
    if (clear) g[i] = 0.f;
    const float mi = b1 * m[i] + (1.f - b1) * gi;
    const float vi = b2 * v[i] + (1.f - b2) * gi * gi;
    m[i] = mi;
    v[i] = vi;
    p[i] = p[i] - step * (mi / (sqrtf(vi) / bc2_sqrt + eps));
  }
}

// ------------------------------------------------------------------------------------------
// packing.  One block handles a 16 x 32 (outer x inner channel) tile of the fp32 master and all
// kw taps: coalesced reads, 32-byte segment writes into both packed layouts.
//
// kind 0 (Conv1d W[co][ci][k], reflect pad kw/2 - 1 on the left: o = kw/2 - 1, 14 for kw = 31):
//   Wf [d+4][co][p*Cin + ci] = W[co][ci][ 4d + p + o]         (fwd:   K = (p,ci), N = co)
//   Wdg[d+4][p*Cin + ci][co] = W[co][ci][-4d + p + o]         (dgrad: K = co, N = (p,ci))
// kind 1 (ConvTranspose1d W[ci][co][k], padding P = (kw - 4)/2, 13 for kw = 31; alpha folded for ci >= alpha_from):
//   Wt [d+4][r*Cout + co][ci] = a(ci) W[ci][co][-4d + r + P]  (fwd:   K = ci, N = (r,co))
//   Wtd[d+4][ci][r*Cout + co] = a(ci) W[ci][co][ 4d + r + P]  (dgrad: K = (r,co), N = ci)
// entries whose tap index falls outside [0, kw) are zero.  4 <= kw <= 32: with at most 32 taps every index
// 4d + p + o (|d| <= 4) of a stride-4 layer lies within the 9-tap table.
// ------------------------------------------------------------------------------------------
constexpr int PO = 16, PI = 32;              // tile: 16 outer x 32 inner channels x kw taps (3 CTAs/SM)
constexpr int PACK_THREADS = 512;
constexpr int PACK_SMEM = PO * PI * (KW_MAX + 1) * 4;   // last dim padded to 33 words: conflict-free transposes

__host__ __device__ __forceinline__ int tap_offset(int kind, int kw) { return kind == 0 ? kw / 2 - 1 : (kw - 4) / 2; }

__global__ void __launch_bounds__(PACK_THREADS)
pack_conv_kernel(int kind, int kw, const float* __restrict__ w, int c_outer, int c_inner, const float* __restrict__ alpha,
                 int alpha_from, void* __restrict__ w_fwd, void* __restrict__ w_dg, int dt_fwd, int dt_dg) {
  // master layout is [outer][inner][kw]; kind 0: outer = co, inner = ci ; kind 1: outer = ci, inner = co
  extern __shared__ float tile_raw[];
  float (*tile)[PI][KW_MAX + 1] = reinterpret_cast<float (*)[PI][KW_MAX + 1]>(tile_raw);
  const int o0 = blockIdx.y * PO, i0 = blockIdx.x * PI;
  const int tid = threadIdx.x;
  const int off = tap_offset(kind, kw);
  for (int idx = tid; idx < PO * PI * kw; idx += PACK_THREADS) {
    const int oo = idx / (PI * kw), rem = idx % (PI * kw);
    const int ii = rem / kw, k = rem % kw;
    float v = w[((int64_t)(o0 + oo) * c_inner + (i0 + ii)) * kw + k];
    if (kind == 1 && alpha && (o0 + oo) >= alpha_from) v *= alpha[o0 + oo - alpha_from];
    tile[oo][ii][k] = v;
  }
  __syncthreads();
  // destination A: contiguous along the INNER channel (32 wide); destination B: along the OUTER (16 wide)
  for (int idx = tid; idx < NTAP * 4 * PO * PI; idx += PACK_THREADS) {
    {  // A: lo = inner
      const int lo = idx % PI, hi = (idx / PI) % PO, ph = (idx / (PI * PO)) % 4, ti = idx / (4 * PI * PO);
      const int d = ti - 4;
      if (kind == 0) {   // Wf[ti][co = hi][ph*Cin + ci = lo],  k = 4d + ph + o
        const int k = 4 * d + ph + off;
        const float v = (k >= 0 && k < kw) ? tile[hi][lo][k] : 0.f;
        if (w_fwd) st_any(w_fwd, ((int64_t)ti * c_outer + (o0 + hi)) * (4 * c_inner) + ph * c_inner + (i0 + lo), v, dt_fwd);
      } else {           // Wtd[ti][ci = hi][ph*Cout + co = lo],  k = 4d + ph + P
        const int k = 4 * d + ph + off;
        const float v = (k >= 0 && k < kw) ? tile[hi][lo][k] : 0.f;
        if (w_dg) st_any(w_dg, ((int64_t)ti * c_outer + (o0 + hi)) * (4 * c_inner) + ph * c_inner + (i0 + lo), v, dt_dg);
      }
    }
    {  // B: lo = outer
      const int lo = idx % PO, hi = (idx / PO) % PI, ph = (idx / (PI * PO)) % 4, ti = idx / (4 * PI * PO);
      const int d = ti - 4;
      if (kind == 0) {   // Wdg[ti][ph*Cin + ci = hi][co = lo],  k = -4d + ph + o
        const int k = -4 * d + ph + off;
        const float v = (k >= 0 && k < kw) ? tile[lo][hi][k] : 0.f;
        if (w_dg) st_any(w_dg, ((int64_t)ti * (4 * c_inner) + ph * c_inner + (i0 + hi)) * c_outer + (o0 + lo), v, dt_dg);
      } else {           // Wt[ti][ph*Cout + co = hi][ci = lo],  k = -4d + ph + P
        const int k = -4 * d + ph + off;
        const float v = (k >= 0 && k < kw) ? tile[lo][hi][k] : 0.f;
        if (w_fwd) st_any(w_fwd, ((int64_t)ti * (4 * c_inner) + ph * c_inner + (i0 + hi)) * c_outer + (o0 + lo), v, dt_fwd);
      }
    }
  }
}

// kind 2 (Linear W[n][c*T + t]) -> W1p[n][t*C + c] ; W1dg[t*C + c][n]
__global__ void pack_fc_kernel(const float* __restrict__ w, int nout, int C, int T, void* __restrict__ w_fwd,
                               void* __restrict__ w_dg, int dt_fwd, int dt_dg) {
  const int64_t total = (int64_t)nout * C * T;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    // i indexes the destination W1p (coalesced writes)
    const int n = (int)(i / ((int64_t)C * T));
    const int kk = (int)(i % ((int64_t)C * T));
    const int t = kk / C, c = kk % C;
    const float v = w[(int64_t)n * C * T + (int64_t)c * T + t];
    if (w_fwd) st_any(w_fwd, i, v, dt_fwd);
    if (w_dg) st_any(w_dg, (int64_t)kk * nout + n, v, dt_dg);
  }
}

// ------------------------------------------------------------------------------------------
// unpack: packed fp32 dWp -> reference layout
// kind 0: dW[co][ci][k] = dWf[d+4][co][p*Cin+ci],  k = 4d + p + o
// kind 1: dWe[ci][co][k] = dWt[d+4][r*Cout+co][ci], k = -4d + r + P ; dW = a(ci) dWe ;
//         dalpha[ci-alpha_from] = sum_{co,k} dWe * W
// kind 2: dW[n][c*T+t] = dW1p[n][t*C+c]
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(PACK_THREADS)
unpack_conv_kernel(int kind, int kw, const float* __restrict__ dwp, int c_outer, int c_inner, const float* __restrict__ w,
                   const float* __restrict__ alpha, int alpha_from, float* __restrict__ dw,
                   float* __restrict__ dalpha, int accumulate) {
  extern __shared__ float tile_raw[];
  float (*tile)[PI][KW_MAX + 1] = reinterpret_cast<float (*)[PI][KW_MAX + 1]>(tile_raw);
  const int off = tap_offset(kind, kw);
  __shared__ float ared[PO];
  const int o0 = blockIdx.y * PO, i0 = blockIdx.x * PI;
  const int tid = threadIdx.x;
  if (tid < PO) ared[tid] = 0.f;
  for (int idx = tid; idx < NTAP * 4 * PO * PI; idx += PACK_THREADS) {
    if (kind == 0) {   // dWf[ti][co = hi][ph*Cin + ci = lo]: contiguous along the inner channel
      const int lo = idx % PI, hi = (idx / PI) % PO, ph = (idx / (PI * PO)) % 4, ti = idx / (4 * PI * PO);
      const int k = 4 * (ti - 4) + ph + off;
      if (k >= 0 && k < kw)
        tile[hi][lo][k] = dwp[((int64_t)ti * c_outer + (o0 + hi)) * (4 * c_inner) + ph * c_inner + (i0 + lo)];
    } else {           // dWt[ti][ph*Cout + co = hi][ci = lo]: contiguous along the outer channel
      const int lo = idx % PO, hi = (idx / PO) % PI, ph = (idx / (PI * PO)) % 4, ti = idx / (4 * PI * PO);
      const int k = -4 * (ti - 4) + ph + off;
      if (k >= 0 && k < kw)
        tile[lo][hi][k] = dwp[((int64_t)ti * (4 * c_inner) + ph * c_inner + (i0 + hi)) * c_outer + (o0 + lo)];
    }
  }
  __syncthreads();
  // PI*kw consecutive master elements share one outer channel `oo`
  for (int oo = 0; oo < PO; ++oo) {
    for (int e = tid; e < PI * kw; e += PACK_THREADS) {
      const int ii = e / kw, k = e % kw;
      const int64_t gi = ((int64_t)(o0 + oo) * c_inner + (i0 + ii)) * kw + k;
      float v = tile[oo][ii][k];
      float contrib = 0.f;
      const bool al = kind == 1 && alpha && (o0 + oo) >= alpha_from;
      if (al) {
        if (dalpha) contrib = v * w[gi];
        v *= alpha[o0 + oo - alpha_from];
      }
      dw[gi] = accumulate ? dw[gi] + v : v;
      if (al && dalpha) {
        contrib = warp_sum(contrib);
        if ((tid & 31) == 0) atomicAdd(&ared[oo], contrib);
      }
    }
  }
  __syncthreads();
  if (kind == 1 && alpha && dalpha && tid < PO && (o0 + tid) >= alpha_from)
    atomicAdd(dalpha + (o0 + tid - alpha_from), ared[tid]);
}

__global__ void unpack_fc_kernel(const float* __restrict__ dwp, int nout, int C, int T, float* __restrict__ dw,
                                 int accumulate) {
  const int64_t total = (int64_t)nout * C * T;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int n = (int)(i / ((int64_t)C * T));
    const int kk = (int)(i % ((int64_t)C * T));
    const int t = kk / C, c = kk % C;
    const int64_t o = (int64_t)n * C * T + (int64_t)c * T + t;
    dw[o] = accumulate ? dw[o] + dwp[i] : dwp[i];
  }
}

// ------------------------------------------------------------------------------------------
// Packed-master path.  The fp32 master weights, the optimiser state and the gradients of every tap-GEMM layer
// live in the layout of the layer's FORWARD operand, M[T][nc][kc] (T = 9 taps, or 1 for the Linear): the
// weight-gradient tap-GEMM already produces that layout, RMSprop / Adam are elementwise, and the two 16-bit
// operands are one elementwise copy and one per-tap transpose of it:
//     F [t][n][k]  = M[t][n][k] * colscale[k]                     (forward operand)
//     Dg[t][k][n]  = M[T-1-t][n][k] * colscale[k]                 (data-gradient operand: tap d <-> -d)
// colscale = the GSkip alpha of the decoder's skip half (generator.py:68-69), 1 elsewhere.
// One block = one 64 x 64 (n, k) tile of one tap.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
emit_operands_kernel(const float* __restrict__ m, int T, int nc, int kc, const float* __restrict__ alpha,
                     int alpha_from, void* __restrict__ f, void* __restrict__ dg, int dt_f, int dt_dg,
                     const float* __restrict__ scale_dev) {
  __shared__ float tile[64][65];
  const int t = blockIdx.z;
  const int n0 = blockIdx.y * 64, k0 = blockIdx.x * 64;
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;      // 64 x 4
  const float sc = ((alpha && k0 + tx >= alpha_from) ? alpha[k0 + tx - alpha_from] : 1.f) *
                   (scale_dev ? *scale_dev : 1.f);
  const int64_t mbase = ((int64_t)t * nc + n0) * kc + k0;
#pragma unroll 4
  for (int r = ty; r < 64; r += 4) {
    const float v = m[mbase + (int64_t)r * kc + tx] * sc;
    tile[r][tx] = v;
    if (f) st_any(f, mbase + (int64_t)r * kc + tx, v, dt_f);
  }
  if (!dg) return;
  __syncthreads();
  const int64_t dbase = ((int64_t)(T - 1 - t) * kc + k0) * nc + n0;
#pragma unroll 4
  for (int r = ty; r < 64; r += 4) st_any(dg, dbase + (int64_t)r * nc + tx, tile[tx][r], dt_dg);
}

// dWeff (packed, w.r.t. alpha-scaled weights) -> dW = alpha * dWeff in place and
// dalpha[k - alpha_from] += sum_{t, n} dWeff[t][n][k] * M[t][n][k]   for the columns k >= alpha_from.
// Block = 32 columns x (256/32 = 8) row lanes striding all T*nc rows.
__global__ void __launch_bounds__(256)
alpha_grad_kernel(float* __restrict__ dwp, const float* __restrict__ m, int64_t rows, int kc,
                  const float* __restrict__ alpha, int alpha_from, float* __restrict__ dalpha) {
  __shared__ float red[8][33];
  const int c = alpha_from + blockIdx.x * 32 + (threadIdx.x & 31);
  const int lane_r = threadIdx.x >> 5;
  const int64_t r_lo = (int64_t)blockIdx.y * 8 + lane_r;
  const float a = alpha[c - alpha_from];
  float acc = 0.f;
  for (int64_t r = r_lo; r < rows; r += (int64_t)gridDim.y * 8) {
    const int64_t i = r * kc + c;
    const float g = dwp[i];
    acc = fmaf(g, m[i], acc);
    dwp[i] = g * a;
  }
  red[lane_r][threadIdx.x & 31] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += red[i][threadIdx.x];
    if (dalpha) atomicAdd(dalpha + (c - alpha_from), s);
  }
}

// Waveform-end layer gradients out of their single-tap GEMM results (both tiny):
//   first conv (Cin = 1 | 2, width kw): dwq[2][64][2][64] (position-pair s x co x pair s' x (ci*32 + k)); the s == s'
//   blocks are the gradient:  dW[co][ci][k] += dwq[0][co][0][ci*32+k] + dwq[1][co][1][ci*32+k],  k < kw
//   (the blocks read are zeroed again: dwq needs no fill before the next weight-gradient GEMM accumulates into it;
//   the im2col columns k >= kw are zero, so the GEMM leaves the columns not read here at zero)
__global__ void wave_wgrad_fold_kernel(float* __restrict__ dwq, int cin, int kw, float* __restrict__ dw) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 64 * cin * kw) return;
  const int co = i / (cin * kw), rem = i % (cin * kw);
  const int ci = rem / kw, k = rem % kw;
  const int col = ci * 32 + k;
  float* p0 = dwq + ((0 * 64 + co) * 2 + 0) * 64 + col;
  float* p1 = dwq + ((1 * 64 + co) * 2 + 1) * 64 + col;
  const float v = *p0 + *p1;
  *p0 = 0.f;
  *p1 = 0.f;
  atomicAdd(dw + i, v);
}
//   last deconv (Cout = 1, width kw, alpha folded into its effective weight): dwq[2][64][NSRC][2][half] (s, k-slot,
//   source, s', c); dWeff[src*half + c][k] = dwq[0][k][src][0][c] + dwq[1][k][src][1][c], k < kw; dW += dWeff (* alpha for the skip
//   half), dalpha[c] += sum_k dWeff[half + c][k] * W[half + c][k].  NSRC = 2: cat(decoder, skip); NSRC = 1: the
//   decoder output alone (no skips: no alpha, w / alpha / dalpha unused)
template <int NSRC>
__global__ void last_deconv_wgrad_fold_kernel(float* __restrict__ dwq, int half, int kw, const float* __restrict__ w,
                                              const float* __restrict__ alpha, float* __restrict__ dw,
                                              float* __restrict__ dalpha) {
  const int ch = blockIdx.x * blockDim.x + threadIdx.x;       // channel of cat(decoder, skip): [0, NSRC*half)
  if (ch >= NSRC * half) return;
  const int src = ch / half, c = ch % half;
  float da = 0.f;
  for (int k = 0; k < kw; ++k) {
    float* p0 = dwq + ((((int64_t)0 * 64 + k) * NSRC + src) * 2 + 0) * half + c;
    float* p1 = dwq + ((((int64_t)1 * 64 + k) * NSRC + src) * 2 + 1) * half + c;
    const float v = *p0 + *p1;
    *p0 = 0.f;
    *p1 = 0.f;
    const int64_t wi = (int64_t)ch * kw + k;
    if (NSRC == 2 && src == 1) {
      da = fmaf(v, w[wi], da);
      atomicAdd(dw + wi, v * alpha[c]);
    } else {
      atomicAdd(dw + wi, v);
    }
  }
  if (NSRC == 2 && src == 1 && dalpha) atomicAdd(dalpha + c, da);
}

// ------------------------------------------------------------------------------------------
// emphasis filters (se_dataset.py:111-126).  De-emphasis x[n] = c x[n-1] + y[n] is a linear
// recurrence: single block, chunked scan over (a, b) pairs with the carry kept in a register.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) deemph_kernel(const float* __restrict__ y, int64_t n, float c,
                                                      float* __restrict__ x, const int64_t* __restrict__ seg) {
  constexpr int PER = 4;
  if (seg) {                       // segmented: block b filters [seg[2b], seg[2b] + seg[2b+1]) from a zero state
    y += seg[2 * blockIdx.x];
    x += seg[2 * blockIdx.x];
    n = seg[2 * blockIdx.x + 1];
  }
  __shared__ float sa[32], sb[32];
  __shared__ float carry_s;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) carry_s = 0.f;
  __syncthreads();
  const float c2 = c * c, c4 = c2 * c2;
  for (int64_t base = 0; base < n; base += 1024 * PER) {
    const int64_t i0 = base + (int64_t)tid * PER;
    float v[PER];
#pragma unroll
    for (int j = 0; j < PER; ++j) v[j] = (i0 + j < n) ? y[i0 + j] : 0.f;
    // local serial part: x_j = c x_{j-1} + v_j with x_{-1} = 0 ; thread transform is (A = c^4, B = local[3])
    float loc[PER];
    loc[0] = v[0];
#pragma unroll
    for (int j = 1; j < PER; ++j) loc[j] = fmaf(c, loc[j - 1], v[j]);
    float A = c4, Bv = loc[PER - 1];
    // inclusive scan of affine maps within the warp: (A2,B2) o (A1,B1) = (A1*A2, A2*B1 + B2)
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float Ap = __shfl_up_sync(0xffffffffu, A, o);
      const float Bp = __shfl_up_sync(0xffffffffu, Bv, o);
      if (lane >= o) { Bv = fmaf(A, Bp, Bv); A = A * Ap; }
    }
    if (lane == 31) { sa[warp] = A; sb[warp] = Bv; }
    __syncthreads();
    if (warp == 0) {
      float wa = sa[lane], wb = sb[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const float Ap = __shfl_up_sync(0xffffffffu, wa, o);
        const float Bp = __shfl_up_sync(0xffffffffu, wb, o);
        if (lane >= o) { wb = fmaf(wa, Bp, wb); wa = wa * Ap; }
      }
      sa[lane] = wa; sb[lane] = wb;
    }
    __syncthreads();
    const float carry = carry_s;
    // exclusive prefix for this thread: state before its first element
    float Aw = 1.f, Bw = 0.f;             // warps before
    if (warp > 0) { Aw = sa[warp - 1]; Bw = sb[warp - 1]; }
    float Al = __shfl_up_sync(0xffffffffu, A, 1), Bl = __shfl_up_sync(0xffffffffu, Bv, 1);
    if (lane == 0) { Al = 1.f; Bl = 0.f; }
    // state_in = Al*(Aw*carry + Bw) + Bl
    const float sin_ = fmaf(Al, fmaf(Aw, carry, Bw), Bl);
    float cp = c, xv = 0.f;
#pragma unroll
    for (int j = 0; j < PER; ++j) {
      xv = fmaf(cp, sin_, loc[j]);
      if (i0 + j < n) x[i0 + j] = xv;
      cp *= c;
    }
    __syncthreads();
    if (tid == 1023) carry_s = xv;      // filter state after this chunk
    __syncthreads();
  }
}

__global__ void preemph_kernel(const float* __restrict__ x, int64_t n, float c, float* __restrict__ y) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    y[i] = i == 0 ? x[0] : x[i] - c * x[i - 1];
}

}  // namespace sg

using namespace sg;
#define ST ((cudaStream_t)stream)

// the kernels stream every buffer as float4: each must be 16-byte aligned
static bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

extern "C" int sg_rmsprop_step(float* param, float* grad, float* square_avg, int64_t n, float lr, float alpha,
                               float eps, float grad_scale, int clear_grad, void* stream) {
  SG_CHECK_ARG(param && grad && square_avg && n >= 0);
  SG_CHECK_ARG(aligned16(param) && aligned16(grad) && aligned16(square_avg));
  rmsprop_kernel<<<8 * NUM_SMS, 256, 0, ST>>>(param, grad, square_avg, n, lr, alpha, eps, grad_scale, clear_grad);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_adam_step(float* param, float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, float lr,
                            float beta1, float beta2, float eps, int step, float grad_scale, int clear_grad,
                            void* stream) {
  SG_CHECK_ARG(param && grad && exp_avg && exp_avg_sq && n >= 0);
  SG_CHECK_ARG(aligned16(param) && aligned16(grad) && aligned16(exp_avg) && aligned16(exp_avg_sq));
  SG_CHECK_ARG(step >= 1);                      // the bias corrections divide by 1 - beta^step
  const float bc1 = 1.f - powf(beta1, (float)step);
  const float bc2 = 1.f - powf(beta2, (float)step);
  adam_kernel<<<8 * NUM_SMS, 256, 0, ST>>>(param, grad, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps, bc1,
                                           sqrtf(bc2), grad_scale, clear_grad);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_pack_weights_kw(int kind, const float* w, int c_out, int c_in, int t_len, int kw,
                                  const float* alpha, int alpha_from, void* w_fwd, void* w_dgrad, int dtype_fwd,
                                  int dtype_dgrad, void* stream) {
  SG_CHECK_ARG(w && (w_fwd || w_dgrad) && (kind == 2 || kw_served(kw)));
  static bool attr_set = false;
  if (!attr_set) {
    SG_CHECK_CUDA(cudaFuncSetAttribute(pack_conv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PACK_SMEM));
    SG_CHECK_CUDA(cudaFuncSetAttribute(unpack_conv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PACK_SMEM));
    attr_set = true;
  }
  if (kind == 0) {
    SG_CHECK_ARG(c_out % PO == 0 && c_in % PI == 0);
    dim3 grid(c_in / PI, c_out / PO);
    pack_conv_kernel<<<grid, PACK_THREADS, PACK_SMEM, ST>>>(0, kw, w, c_out, c_in, nullptr, 0, w_fwd, w_dgrad,
                                                            dtype_fwd, dtype_dgrad);
  } else if (kind == 1) {
    SG_CHECK_ARG(c_out % PI == 0 && c_in % PO == 0);
    dim3 grid(c_out / PI, c_in / PO);
    pack_conv_kernel<<<grid, PACK_THREADS, PACK_SMEM, ST>>>(1, kw, w, c_in, c_out, alpha, alpha_from, w_fwd, w_dgrad,
                                                            dtype_fwd, dtype_dgrad);
  } else if (kind == 2) {
    pack_fc_kernel<<<4 * NUM_SMS, 256, 0, ST>>>(w, c_out, c_in, t_len, w_fwd, w_dgrad, dtype_fwd, dtype_dgrad);
  } else {
    SG_CHECK_ARG(false);
  }
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_pack_weights(int kind, const float* w, int c_out, int c_in, int t_len, const float* alpha,
                               int alpha_from, void* w_fwd, void* w_dgrad, int dtype_fwd, int dtype_dgrad,
                               void* stream) {
  return sg_pack_weights_kw(kind, w, c_out, c_in, t_len, 31, alpha, alpha_from, w_fwd, w_dgrad, dtype_fwd, dtype_dgrad,
                            stream);
}

extern "C" int sg_unpack_wgrad_kw(int kind, const float* dwp, int c_out, int c_in, int t_len, int kw, const float* w,
                                  const float* alpha, int alpha_from, float* dw, float* dalpha, int accumulate,
                                  void* stream) {
  SG_CHECK_ARG(dwp && dw && (kind == 2 || kw_served(kw)));
  SG_CHECK_ARG(kind != 0 || (c_out % PO == 0 && c_in % PI == 0));     // the tile grid of sg_pack_weights
  SG_CHECK_ARG(kind != 1 || (c_out % PI == 0 && c_in % PO == 0));
  static bool attr_set = false;
  if (!attr_set) {
    SG_CHECK_CUDA(cudaFuncSetAttribute(pack_conv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PACK_SMEM));
    SG_CHECK_CUDA(cudaFuncSetAttribute(unpack_conv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PACK_SMEM));
    attr_set = true;
  }
  if (kind == 0) {
    dim3 grid(c_in / PI, c_out / PO);
    unpack_conv_kernel<<<grid, PACK_THREADS, PACK_SMEM, ST>>>(0, kw, dwp, c_out, c_in, nullptr, nullptr, 0, dw, nullptr,
                                                              accumulate);
  } else if (kind == 1) {
    dim3 grid(c_out / PI, c_in / PO);
    unpack_conv_kernel<<<grid, PACK_THREADS, PACK_SMEM, ST>>>(1, kw, dwp, c_in, c_out, w, alpha, alpha_from, dw, dalpha,
                                                              accumulate);
  } else if (kind == 2) {
    unpack_fc_kernel<<<4 * NUM_SMS, 256, 0, ST>>>(dwp, c_out, c_in, t_len, dw, accumulate);
  } else {
    SG_CHECK_ARG(false);
  }
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_unpack_wgrad(int kind, const float* dwp, int c_out, int c_in, int t_len, const float* w,
                               const float* alpha, int alpha_from, float* dw, float* dalpha, int accumulate,
                               void* stream) {
  return sg_unpack_wgrad_kw(kind, dwp, c_out, c_in, t_len, 31, w, alpha, alpha_from, dw, dalpha, accumulate, stream);
}

extern "C" int sg_emit_operands(const float* master, int n_taps, int nc, int kc, const float* alpha, int alpha_from,
                                void* w_fwd, void* w_dgrad, int dtype_fwd, int dtype_dgrad, const float* scale_dev,
                                void* stream) {
  SG_CHECK_ARG(master && (w_fwd || w_dgrad) && n_taps >= 1 && nc % 64 == 0 && kc % 64 == 0);
  SG_CHECK_ARG(!alpha || (alpha_from >= 0 && alpha_from < kc));
  dim3 grid(kc / 64, nc / 64, n_taps);
  emit_operands_kernel<<<grid, 256, 0, ST>>>(master, n_taps, nc, kc, alpha, alpha_from, w_fwd, w_dgrad, dtype_fwd,
                                             dtype_dgrad, scale_dev);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_alpha_grad(float* dwp, const float* master, int n_taps, int nc, int kc, const float* alpha,
                             int alpha_from, float* dalpha, void* stream) {
  SG_CHECK_ARG(dwp && master && alpha && alpha_from >= 0 && alpha_from < kc && (kc - alpha_from) % 32 == 0);
  const int64_t rows = (int64_t)n_taps * nc;
  int gy = (int)((rows + 8 * 64 - 1) / (8 * 64));
  if (gy < 1) gy = 1;
  if (gy > 64) gy = 64;
  dim3 grid((kc - alpha_from) / 32, gy);
  alpha_grad_kernel<<<grid, 256, 0, ST>>>(dwp, master, rows, kc, alpha, alpha_from, dalpha);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_wave_wgrad_fold_kw(float* dwq, int cin, int kw, float* dw, void* stream) {
  SG_CHECK_ARG(dwq && dw && (cin == 1 || cin == 2) && kw_served(kw));
  wave_wgrad_fold_kernel<<<(64 * cin * kw + 255) / 256, 256, 0, ST>>>(dwq, cin, kw, dw);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_wave_wgrad_fold(float* dwq, int cin, float* dw, void* stream) {
  return sg_wave_wgrad_fold_kw(dwq, cin, 31, dw, stream);
}

extern "C" int sg_last_deconv_wgrad_fold_kw(float* dwq, int half, int kw, const float* w, const float* alpha,
                                            float* dw, float* dalpha, void* stream) {
  SG_CHECK_ARG(dwq && w && alpha && dw && half > 0 && kw_served(kw));
  last_deconv_wgrad_fold_kernel<2><<<(2 * half + 127) / 128, 128, 0, ST>>>(dwq, half, kw, w, alpha, dw, dalpha);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_last_deconv_wgrad_fold(float* dwq, int half, const float* w, const float* alpha, float* dw,
                                         float* dalpha, void* stream) {
  return sg_last_deconv_wgrad_fold_kw(dwq, half, 31, w, alpha, dw, dalpha, stream);
}

extern "C" int sg_last_deconv_wgrad_fold_1src_kw(float* dwq, int cin, int kw, float* dw, void* stream) {
  SG_CHECK_ARG(dwq && dw && cin > 0 && kw_served(kw));
  last_deconv_wgrad_fold_kernel<1><<<(cin + 127) / 128, 128, 0, ST>>>(dwq, cin, kw, nullptr, nullptr, dw, nullptr);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_last_deconv_wgrad_fold_1src(float* dwq, int cin, float* dw, void* stream) {
  return sg_last_deconv_wgrad_fold_1src_kw(dwq, cin, 31, dw, stream);
}

extern "C" int sg_deemphasis(const float* y, int64_t n, float coef, float* x, void* stream) {
  deemph_kernel<<<1, 1024, 0, ST>>>(y, n, coef, x, nullptr);
  SG_CHECK_LAUNCH();
  return SG_OK;
}
extern "C" int sg_deemphasis_segments(const float* y, const int64_t* seg, int n_seg, float coef, float* x,
                                      void* stream) {
  SG_CHECK_ARG(y && x && seg && n_seg > 0);
  deemph_kernel<<<n_seg, 1024, 0, ST>>>(y, 0, coef, x, seg);
  SG_CHECK_LAUNCH();
  return SG_OK;
}
// int16 PCM windows -> network input: normalize_wave_minmax (se_dataset.py:108-109) then pre_emphasize
// (se_dataset.py:111-117): y[n] = x[n] - coef * x[n-1].  The reference pre-emphasises the WHOLE file before
// slicing (read_wav_file, se_dataset.py:191-199), so the sample before a window matters: prev[w] holds it (int32;
// SG_PCM_NO_PREV = the window starts the file, y[0] = x[0]); prev == NULL treats every window as a file start.
__global__ void pcm16_to_wave_kernel(const int16_t* __restrict__ pcm, const int32_t* __restrict__ prev, int64_t total,
                                     int L, float coef, float* __restrict__ out, const int32_t* __restrict__ valid) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    if (valid && (int)(i % L) >= valid[i / L]) {     // zero padding of a file's last window (model.py:122-131)
      out[i] = 0.f;
      continue;
    }
    const float x = (2.f / 65535.f) * ((float)pcm[i] - 32767.f) + 1.f;
    float y = x;
    if (coef > 0.f) {
      const int n = (int)(i % L);
      int p = SG_PCM_NO_PREV;
      if (n != 0) p = pcm[i - 1];
      else if (prev) p = prev[i / L];
      if (p != SG_PCM_NO_PREV) y = x - coef * ((2.f / 65535.f) * ((float)p - 32767.f) + 1.f);
    }
    out[i] = y;
  }
}

extern "C" int sg_pcm16_to_wave(const int16_t* pcm, const int32_t* prev, int64_t n_windows, int L, float coef,
                                float* out, const int32_t* valid_len, void* stream) {
  SG_CHECK_ARG(pcm && out && n_windows > 0 && L > 0);
  pcm16_to_wave_kernel<<<4 * NUM_SMS, 256, 0, ST>>>(pcm, prev, n_windows * L, L, coef, out, valid_len);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_preemphasis(const float* x, int64_t n, float coef, float* y, void* stream) {
  preemph_kernel<<<2 * NUM_SMS, 256, 0, ST>>>(x, n, coef, y);
  SG_CHECK_LAUNCH();
  return SG_OK;
}
