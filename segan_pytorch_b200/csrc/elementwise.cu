// HBM-bound glue between the tap-GEMMs: BatchNorm statistics / finalize, the fused
// "BN-apply + PReLU + circular phase shift + reflect halo" producer of conv inputs and its
// backward, layout converters, the discriminator FC tail, and the loss tails.
// All 16-bit tensors are NLC ([positions][C], C innermost); threads own 8 consecutive channels
// (one 16-byte vector) so every access is a coalesced 128-bit transaction.
#include "common.cuh"
#include <stdlib.h>
#include <string.h>

namespace sg {

// ------------------------------------------------------------------------------------------
// Streaming kernels.  Thread = VEC adjacent channels (one 8- or 16-byte load per stream) of a row,
// C/VEC threads per row, 256/(C/VEC) rows per CTA iteration, UNROLL rows in flight per thread.
// The per-thread bytes in flight (loads x VEC x 2 B x UNROLL) are what matters here: these
// kernels also run CONCURRENTLY with the persistent tap-GEMMs (engine.py side streams), where only
// 2-3 of their CTAs fit next to a GEMM CTA on an SM, so memory-level parallelism has to come from
// the thread, not from occupancy.  The variant (VEC, UNROLL, grid caps) is a runtime tuning knob
// (sg_set_ew_variant / SEGAN_B200_EW); every variant computes identical values.
// ------------------------------------------------------------------------------------------
// per-channel statistics are accumulated into SG_STAT_SLICES interleaved copies (slice = CTA % 8):
// ~450 CTAs hitting one fp64 address serialise at ~60 ns each (measured: ~30 us tail per launch);
// consumers add the slices up.
constexpr int SL = SG_STAT_SLICES;

template <int VEC> struct FV { float v[VEC]; };
// packed 16-bit vector as loaded (kept packed while in flight: VEC/2 registers instead of VEC)
template <int VEC> struct RV { uint32_t w[VEC / 2]; };

template <int VEC>
__device__ __forceinline__ RV<VEC> ldr(const void* p, int64_t elem) {
  RV<VEC> r;
  const uint16_t* q = reinterpret_cast<const uint16_t*>(p) + elem;
  if constexpr (VEC == 8) {
    const uint4 u = *reinterpret_cast<const uint4*>(q);
    r.w[0] = u.x; r.w[1] = u.y; r.w[2] = u.z; r.w[3] = u.w;
  } else {
    const uint2 u = *reinterpret_cast<const uint2*>(q);
    r.w[0] = u.x; r.w[1] = u.y;
  }
  return r;
}
template <int VEC>
__device__ __forceinline__ RV<VEC> zero_rv() {
  RV<VEC> r;
#pragma unroll
  for (int i = 0; i < VEC / 2; ++i) r.w[i] = 0u;
  return r;
}
template <int VEC>
__device__ __forceinline__ FV<VEC> up(const RV<VEC>& x, int dtype) {
  FV<VEC> r;
#pragma unroll
  for (int i = 0; i < VEC / 2; ++i) {
    float2 f;
    if (dtype == SG_F16) f = __half22float2(*reinterpret_cast<const __half2*>(&x.w[i]));
    else f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&x.w[i]));
    r.v[2 * i] = f.x; r.v[2 * i + 1] = f.y;
  }
  return r;
}
template <int VEC>
__device__ __forceinline__ FV<VEC> ldv(const void* p, int64_t elem, int dtype) {
  return up<VEC>(ldr<VEC>(p, elem), dtype);
}
template <int VEC>
__device__ __forceinline__ void stv(void* p, int64_t elem, const float (&x)[VEC], int dtype) {
  uint32_t w[VEC / 2];
#pragma unroll
  for (int i = 0; i < VEC / 2; ++i) {
    if (dtype == SG_F16) {
      w[i] = pack_half2_sat(x[2 * i], x[2 * i + 1]);
    } else {
      __nv_bfloat162 a = __floats2bfloat162_rn(x[2 * i], x[2 * i + 1]);
      w[i] = *reinterpret_cast<uint32_t*>(&a);
    }
  }
  uint16_t* q = reinterpret_cast<uint16_t*>(p) + elem;
  if constexpr (VEC == 8) *reinterpret_cast<uint4*>(q) = make_uint4(w[0], w[1], w[2], w[3]);
  else *reinterpret_cast<uint2*>(q) = make_uint2(w[0], w[1]);
}

// per-thread partial sums of NS statistics for VEC channels -> smem combine over the CTA's threads
// that own the same channels -> one double atomic per channel and CTA
template <int NS, int VEC>
__device__ __forceinline__ void block_stats_flush(float (&part)[NS][VEC], int cgs, int C, double* out,
                                                  float* smem /* [256][VEC] */) {
  const int tid = threadIdx.x;
  const int cg = tid % cgs;
  for (int s = 0; s < NS; ++s) {
    __syncthreads();
#pragma unroll
    for (int j = 0; j < VEC; ++j) smem[tid * VEC + j] = part[s][j];
    __syncthreads();
    if (tid < cgs) {
      double acc[VEC];
#pragma unroll
      for (int j = 0; j < VEC; ++j) acc[j] = 0;
      for (int t = tid; t < (int)blockDim.x; t += cgs)
#pragma unroll
        for (int j = 0; j < VEC; ++j) acc[j] += (double)smem[t * VEC + j];
#pragma unroll
      for (int j = 0; j < VEC; ++j)
        atomicAdd(out + ((int64_t)(blockIdx.x % SL) * NS + s) * C + cg * VEC + j, acc[j]);
    }
  }
}

template <int VEC, int UNROLL>
__global__ void __launch_bounds__(256, (VEC == 4 && UNROLL <= 4) ? 3 : 2)
bn_stats_kernel(const void* __restrict__ a, int dtype, int64_t rows64, int C, double* __restrict__ stats) {
  __shared__ float red[256 * VEC];
  const int cgs = C / VEC;
  const int tid = threadIdx.x;
  const int cg = tid % cgs;
  const int rpb = 256 / cgs;
  const int rows = (int)rows64;
  const int stride = gridDim.x * rpb;
  constexpr int U = 2 * UNROLL;            // a single input stream: twice the rows in flight
  float part[2][VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) { part[0][j] = 0.f; part[1][j] = 0.f; }
  for (int r0 = blockIdx.x * rpb + tid / cgs; r0 < rows; r0 += U * stride) {
    RV<VEC> raw[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int r = r0 + u * stride;
      raw[u] = (r < rows) ? ldr<VEC>(a, (int64_t)r * C + cg * VEC) : zero_rv<VEC>();
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const FV<VEC> v = up<VEC>(raw[u], dtype);
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        part[0][j] += v.v[j];
        part[1][j] = fmaf(v.v[j], v.v[j], part[1][j]);
      }
    }
  }
  block_stats_flush<2, VEC>(part, cgs, C, stats, red);
}

__global__ void bn_finalize_kernel(const double* __restrict__ stats, double count, int C,
                                   const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                   float momentum, float* __restrict__ rmean, float* __restrict__ rvar,
                                   float* __restrict__ scale_shift, float* __restrict__ mean_invstd) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double s0 = 0, s1 = 0;
  for (int i = 0; i < SL; ++i) { s0 += stats[(int64_t)i * 2 * C + c]; s1 += stats[(int64_t)i * 2 * C + C + c]; }
  const double mean = s0 / count;
  double var = s1 / count - mean * mean;
  if (var < 0) var = 0;
  const float invstd = (float)(1.0 / sqrt(var + (double)eps));
  const float sc = gamma[c] * invstd;
  scale_shift[c] = sc;
  scale_shift[C + c] = beta[c] - (float)mean * sc;
  mean_invstd[c] = (float)mean;
  mean_invstd[C + c] = invstd;
  if (rmean) {
    const double unbiased = count > 1 ? var * count / (count - 1.0) : var;
    rmean[c] = (1.f - momentum) * rmean[c] + momentum * (float)mean;
    rvar[c] = (1.f - momentum) * rvar[c] + momentum * (float)unbiased;
  }
}

// ------------------------------------------------------------------------------------------
// h[b][q + H][c] = act(a[b][src(q)][c] * scale + shift),  q in [-H, L + H),
// src(q) = unroll(reflect(q))
// ------------------------------------------------------------------------------------------
template <int VEC, int UNROLL>
__global__ void __launch_bounds__(256, (VEC == 4 && UNROLL <= 4) ? 3 : 2)
act_fwd_kernel(const void* __restrict__ a, int dtype, int batch, int L, int C,
               const float* __restrict__ scale_shift, const float* __restrict__ slope, int act, int roll,
               const int* __restrict__ roll_dev, int H,
               void* __restrict__ h, void* __restrict__ h_bf16, void* __restrict__ a_bf16) {
  if (roll_dev) roll = *roll_dev;
  constexpr int U = 2 * UNROLL;            // a single input stream: twice the rows in flight
  const int cgs = C / VEC;
  const int Lh = L + 2 * H;
  const int tid = threadIdx.x;
  const int cg = tid % cgs;
  const int rpb = 256 / cgs;
  const int rows = batch * Lh;           // output rows (incl. halo)
  const int stride = gridDim.x * rpb;
  float sc[VEC], sh[VEC], sl[VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    const int c = cg * VEC + j;
    sc[j] = scale_shift ? scale_shift[c] : 1.f;
    sh[j] = scale_shift ? scale_shift[C + c] : 0.f;
    sl[j] = (act == SG_ACT_PRELU) ? slope[c] : 1.f;
  }
  for (int r0 = blockIdx.x * rpb + tid / cgs; r0 < rows; r0 += U * stride) {
    RV<VEC> raw[U];
    int srcs[U];                 // source row, or -1 - source row for halo rows (no a_bf16 copy)
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int r = r0 + u * stride;
      srcs[u] = 0;
      raw[u] = zero_rv<VEC>();
      if (r < rows) {
        const int b = r / Lh;
        const int qh = r - b * Lh;
        const int src = b * L + unroll_idx(reflect_idx(qh - H, L), roll, L);
        srcs[u] = (qh >= H && qh < H + L) ? src : -1 - src;
        raw[u] = ldr<VEC>(a, (int64_t)src * C + cg * VEC);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int r = r0 + u * stride;
      if (r < rows) {
        const FV<VEC> v = up<VEC>(raw[u], dtype);
        float y[VEC];
#pragma unroll
        for (int j = 0; j < VEC; ++j) {
          y[j] = fmaf(v.v[j], sc[j], sh[j]);
          if (act == SG_ACT_PRELU) y[j] = y[j] > 0.f ? y[j] : sl[j] * y[j];
        }
        stv<VEC>(h, (int64_t)r * C + cg * VEC, y, dtype);
        // bf16 twins: operands of the weight-gradient tap-GEMM (wgmma cannot mix f16 x bf16 operands)
        if (h_bf16) stv<VEC>(h_bf16, (int64_t)r * C + cg * VEC, y, SG_BF16);
        if (a_bf16 && srcs[u] >= 0) stv<VEC>(a_bf16, (int64_t)srcs[u] * C + cg * VEC, v.v, SG_BF16);
      }
    }
  }
}

// gradient w.r.t. the activation output at exact position l: the consumer-view gradient at the
// rolled position plus its reflect-halo mirror (at most one of the two mirrors applies: the host
// checks L >= 2H + 3).  Returns the two packed vectors; `has_m` says whether the mirror is live.
template <int VEC>
__device__ __forceinline__ void gather_gy(const void* g_h, int ldh, int H, int roll, int b, int l, int L, int c,
                                          RV<VEC>& g, RV<VEC>& m, bool& has_m) {
  const int Lh = L + 2 * H;
  int q0 = l + roll;
  if (q0 >= L) q0 -= L;
  if (q0 < 0) q0 += L;
  const int64_t base = (int64_t)b * Lh + H;
  g = ldr<VEC>(g_h, (base + q0) * ldh + c);
  has_m = false;
  if (H > 0) {
    int64_t mrow = -1;
    if (q0 >= 1 && q0 <= H) mrow = base - q0;
    else if (q0 >= L - 1 - H && q0 <= L - 2) mrow = base + 2 * (L - 1) - q0;
    if (mrow >= 0) {
      m = ldr<VEC>(g_h, mrow * ldh + c);
      has_m = true;
    }
  }
}

// MODE 0: reductions (and, when g_a_out != null, g_pre written in the same pass: final without BN)
// MODE 1: apply (BN backward) using the reductions
// The skip-connection gradient g_add is w.r.t. the PRE-activation (generator.py:185,191) and joins
// after the activation derivative.
template <int MODE, int VEC, int UNROLL>
__global__ void __launch_bounds__(256, (VEC == 4 && UNROLL <= 4) ? 3 : 2)
act_bwd_kernel(const void* __restrict__ g_h, int ldh, int H, int roll, const int* __restrict__ roll_dev,
               const void* __restrict__ g_add, int lda,
               const void* __restrict__ a, int dtype, int batch, int L, int C,
               const float* __restrict__ scale_shift, const float* __restrict__ mean_invstd,
               const float* __restrict__ slope, int act, double* __restrict__ red, int use_bn,
               void* __restrict__ g_a_out, int gdt) {
  if (roll_dev) roll = *roll_dev;
  __shared__ float sred[MODE == 0 ? 256 * VEC : 1];
  const int cgs = C / VEC;
  const int tid = threadIdx.x;
  const int cg = tid % cgs;
  const int c0 = cg * VEC;
  const int rpb = 256 / cgs;
  const int rows = batch * L;
  const int stride = gridDim.x * rpb;
  // per-channel constants folded as far as possible:
  //   y = x*sc + sh (sign only) ; ahat = x*is - mi ; MODE 1: ga = sc*gpre + ka*x + kb
  float sc[VEC], sh[VEC], sl[VEC], p0[VEC], p1[VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    const int c = c0 + j;
    sc[j] = scale_shift ? scale_shift[c] : 1.f;
    sh[j] = scale_shift ? scale_shift[C + c] : 0.f;
    sl[j] = (act == SG_ACT_PRELU) ? slope[c] : 1.f;
    const float mu = mean_invstd ? mean_invstd[c] : 0.f;
    const float is = mean_invstd ? mean_invstd[C + c] : 1.f;
    if (MODE == 0) {
      p0[j] = is;
      p1[j] = mu * is;
    } else {
      // MODE 1 reads the SG_STAT_SLICES partial copies [SL][3][C] written by pass 1 and adds them up
      double d1 = 0, d2 = 0;
      if (use_bn) {
        for (int i = 0; i < SL; ++i) {
          d1 += red[((int64_t)i * 3 + 1) * C + c];
          d2 += red[((int64_t)i * 3 + 2) * C + c];
        }
      }
      const float r1 = (float)(d1 / (double)rows);
      const float r2 = (float)(d2 / (double)rows);
      p0[j] = use_bn ? -sc[j] * r2 * is : 0.f;                       // ka
      p1[j] = use_bn ? sc[j] * (r2 * is * mu - r1) : 0.f;           // kb
    }
  }
  float part[3][VEC];
#pragma unroll
  for (int s = 0; s < 3; ++s)
#pragma unroll
    for (int j = 0; j < VEC; ++j) part[s][j] = 0.f;
  for (int r0 = blockIdx.x * rpb + tid / cgs; r0 < rows; r0 += UNROLL * stride) {
    RV<VEC> gy[UNROLL], gm[UNROLL], gs[UNROLL], av[UNROLL];
    bool hm[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const int r = r0 + u * stride;
      gy[u] = zero_rv<VEC>(); gm[u] = zero_rv<VEC>(); gs[u] = zero_rv<VEC>(); av[u] = zero_rv<VEC>();
      hm[u] = false;
      if (r < rows) {
        const int b = r / L, l = r - b * L;
        if (g_h) gather_gy<VEC>(g_h, ldh, H, roll, b, l, L, c0, gy[u], gm[u], hm[u]);
        if (g_add) gs[u] = ldr<VEC>(g_add, (int64_t)r * lda + c0);
        av[u] = ldr<VEC>(a, (int64_t)r * C + c0);
      }
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const int r = r0 + u * stride;
      if (r < rows) {
        const FV<VEC> xa = up<VEC>(av[u], dtype);
        FV<VEC> gf = up<VEC>(gy[u], gdt);
        if (hm[u]) {
          const FV<VEC> mf = up<VEC>(gm[u], gdt);
#pragma unroll
          for (int j = 0; j < VEC; ++j) gf.v[j] += mf.v[j];
        }
        const FV<VEC> sf = up<VEC>(gs[u], gdt);     // zero bits -> 0.f when there is no skip gradient
        float out[VEC];
#pragma unroll
        for (int j = 0; j < VEC; ++j) {
          const float x = xa.v[j];
          const float y = fmaf(x, sc[j], sh[j]);
          const float g = gf.v[j];
          float gpre = g;
          if (act == SG_ACT_PRELU && y <= 0.f) {
            if (MODE == 0) part[0][j] = fmaf(g, y, part[0][j]);
            gpre = g * sl[j];
          }
          gpre += sf.v[j];
          if (MODE == 0) {
            part[1][j] += gpre;
            part[2][j] = fmaf(gpre, fmaf(x, p0[j], -p1[j]), part[2][j]);
            out[j] = gpre;
          } else {
            out[j] = use_bn ? fmaf(sc[j], gpre, fmaf(p0[j], x, p1[j])) : gpre;
          }
        }
        if (g_a_out) stv<VEC>(g_a_out, (int64_t)r * C + c0, out, gdt);
      }
    }
  }
  if (MODE == 0) block_stats_flush<3, VEC>(part, cgs, C, red, sred);
}

// ------------------------------------------------------------------------------------------
// Tiled activation backward (the default for sg_act_bwd_reduce / sg_act_bwd_apply).
// The generic kernel above spends ~50 instructions per element on index arithmetic (a division
// per row, 64-bit address chains, 4 channels per thread) and holds all per-channel constants in
// registers; measured 1.5-2.3 TB/s.  Here:
//   * a CTA walks a CONTIGUOUS range of tiles, a tile = U x RPB rows of ONE batch element, so
//     (batch, row) advance incrementally and row offsets are 32-bit relative to per-tile bases;
//   * threads own 8 channels (16-byte loads / stores), C/8 threads per row;
//   * per-channel constants live in shared memory (6 x LDS.128 per row instead of 40 registers),
//     which keeps the kernel at <= 128 registers so that two CTAs fit next to a tap-GEMM CTA;
//   * sum(g_pre * ahat) is accumulated as sum(g_pre * x) and centred in double at the flush.
// ------------------------------------------------------------------------------------------
struct RV8 { uint32_t w[4]; };
__device__ __forceinline__ RV8 ld8(const uint16_t* p) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  RV8 r; r.w[0] = u.x; r.w[1] = u.y; r.w[2] = u.z; r.w[3] = u.w;
  return r;
}
__device__ __forceinline__ void up8(const RV8& x, bool f16, float (&v)[8]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 f;
    if (f16) f = __half22float2(*reinterpret_cast<const __half2*>(&x.w[i]));
    else f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&x.w[i]));
    v[2 * i] = f.x; v[2 * i + 1] = f.y;
  }
}
__device__ __forceinline__ void ld_f8(const float* p, float (&v)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p);
  const float4 b = *reinterpret_cast<const float4*>(p + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

template <int MODE, int U>
__global__ void __launch_bounds__(256, 2)
act_bwd_tiled_kernel(const uint16_t* __restrict__ g_h, int ldh, int H, int roll, const int* __restrict__ roll_dev,
                     const uint16_t* __restrict__ g_add, int lda, const uint16_t* __restrict__ a, int a_f16,
                     int batch, int L, int C, int cgs_log2, const float* __restrict__ scale_shift,
                     const float* __restrict__ mean_invstd, const float* __restrict__ slope, int act,
                     const double* __restrict__ red_in, double* __restrict__ red_out, int use_bn,
                     uint16_t* __restrict__ g_a_out, int tiles_per_b, int tiles_per_cta, int g_f16) {
  extern __shared__ __align__(16) float smf[];
  if (roll_dev) roll = *roll_dev;
  float* s_sc = smf;                 // y = x*sc + sh (sign test, slope gradient)
  float* s_sh = smf + C;
  float* s_sl = smf + 2 * C;         // PReLU slope (1 when act == NONE)
  float* s_so = smf + 3 * C;         // MODE 1: out = so*gpre + ka*x + kb
  float* s_ka = smf + 4 * C;
  float* s_kb = smf + 5 * C;
  const int tid = threadIdx.x;
  const int rows_total = batch * L;
  for (int c = tid; c < C; c += 256) {
    const float sc = scale_shift ? scale_shift[c] : 1.f;
    s_sc[c] = sc;
    s_sh[c] = scale_shift ? scale_shift[C + c] : 0.f;
    s_sl[c] = (act == SG_ACT_PRELU) ? slope[c] : 1.f;
    if (MODE == 1) {
      float so = 1.f, ka = 0.f, kb = 0.f;
      if (use_bn) {
        double d1 = 0, d2 = 0;
        for (int i = 0; i < SL; ++i) {
          d1 += red_in[((int64_t)i * 3 + 1) * C + c];
          d2 += red_in[((int64_t)i * 3 + 2) * C + c];
        }
        const float r1 = (float)(d1 / (double)rows_total);
        const float r2 = (float)(d2 / (double)rows_total);
        const float mu = mean_invstd[c], is = mean_invstd[C + c];
        so = sc;
        ka = -sc * r2 * is;
        kb = sc * (r2 * is * mu - r1);
      }
      s_so[c] = so; s_ka[c] = ka; s_kb[c] = kb;
    }
  }
  __syncthreads();

  const int cgs = 1 << cgs_log2;
  const int cg = tid & (cgs - 1);
  const int rr = tid >> cgs_log2;
  const int c0 = cg * 8;
  const int RPB = 256 >> cgs_log2;
  const int TILE = RPB * U;
  const int Lh = L + 2 * H;
  const bool f16 = a_f16 != 0;
  const bool gf16 = g_f16 != 0;           // 16-bit format of the gradient tensors (sg_set_grad_dtype)
  const bool prelu = act == SG_ACT_PRELU;

  float part[3][8];
#pragma unroll
  for (int s = 0; s < 3; ++s)
#pragma unroll
    for (int j = 0; j < 8; ++j) part[s][j] = 0.f;

  int t = blockIdx.x * tiles_per_cta;
  const int t_end = min(t + tiles_per_cta, batch * tiles_per_b);
  int b = t / tiles_per_b;
  int lt = t - b * tiles_per_b;
  for (; t < t_end; ++t) {
    // 32-bit element offsets from the tensor bases (the host checks every tensor has < 2^31 elements)
    const int rb_a = b * L;                 // first row of this batch element in a / g_add / g_a
    const int rb_g = b * Lh + H;            // row of position 0 in the consumer-view gradient
    const int l0 = lt * TILE + rr;
    RV8 gy[U], gm[U], gs[U], av[U];
    unsigned hm = 0;
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int l = l0 + u * RPB;
      if (l < L) {
        int q0 = l + roll;
        q0 -= (q0 >= L) ? L : 0;
        q0 += (q0 < 0) ? L : 0;
        gy[u] = ld8(g_h + ((rb_g + q0) * ldh + c0));
        if (H > 0) {
          // reflect-halo mirror of position q0 (at most one applies: L >= 2H + 3)
          int m = 0;
          bool has = false;
          if ((unsigned)(q0 - 1) < (unsigned)H) { m = -q0; has = true; }
          else if ((unsigned)(L - 2 - q0) < (unsigned)H) { m = 2 * (L - 1) - q0; has = true; }
          if (has) { gm[u] = ld8(g_h + ((rb_g + m) * ldh + c0)); hm |= 1u << u; }
        }
        if (g_add) gs[u] = ld8(g_add + ((rb_a + l) * lda + c0));
        av[u] = ld8(a + ((rb_a + l) * C + c0));
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int l = l0 + u * RPB;
      if (l < L) {
        float x[8], g[8], sc[8], sh[8], sl[8], out[8];
        up8(av[u], f16, x);
        up8(gy[u], gf16, g);
        if (hm & (1u << u)) {
          float m[8];
          up8(gm[u], gf16, m);
#pragma unroll
          for (int j = 0; j < 8; ++j) g[j] += m[j];
        }
        ld_f8(s_sc + c0, sc); ld_f8(s_sh + c0, sh); ld_f8(s_sl + c0, sl);
        float gpre[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float y = fmaf(x[j], sc[j], sh[j]);
          const bool neg = prelu && y <= 0.f;
          if (MODE == 0 && neg) part[0][j] = fmaf(g[j], y, part[0][j]);
          gpre[j] = neg ? g[j] * sl[j] : g[j];
        }
        if (g_add) {
          float sk[8];
          up8(gs[u], gf16, sk);
#pragma unroll
          for (int j = 0; j < 8; ++j) gpre[j] += sk[j];
        }
        if (MODE == 0) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            part[1][j] += gpre[j];
            part[2][j] = fmaf(gpre[j], x[j], part[2][j]);
            out[j] = gpre[j];
          }
        } else {
          float so[8], ka[8], kb[8];
          ld_f8(s_so + c0, so); ld_f8(s_ka + c0, ka); ld_f8(s_kb + c0, kb);
#pragma unroll
          for (int j = 0; j < 8; ++j) out[j] = fmaf(so[j], gpre[j], fmaf(ka[j], x[j], kb[j]));
        }
        if (g_a_out) {
          uint32_t w[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            if (gf16) {
              w[i] = pack_half2_sat(out[2 * i], out[2 * i + 1]);
            } else {
              __nv_bfloat162 h2 = __floats2bfloat162_rn(out[2 * i], out[2 * i + 1]);
              w[i] = *reinterpret_cast<uint32_t*>(&h2);
            }
          }
          *reinterpret_cast<uint4*>(g_a_out + ((rb_a + l) * C + c0)) = make_uint4(w[0], w[1], w[2], w[3]);
        }
      }
    }
    if (++lt == tiles_per_b) { lt = 0; ++b; }
  }

  if (MODE == 0) {
    // block combine (threads with the same channel group), centre sum(g_pre*x) in double, one atomic
    // per channel, statistic and CTA into slice (CTA % SL)
    __syncthreads();                  // the constants in smf are dead from here on
    double tot[3][8];
    for (int s = 0; s < 3; ++s) {
      __syncthreads();
#pragma unroll
      for (int j = 0; j < 8; ++j) smf[tid * 8 + j] = part[s][j];
      __syncthreads();
      if (tid < cgs) {
#pragma unroll
        for (int j = 0; j < 8; ++j) tot[s][j] = 0;
        for (int q = tid; q < 256; q += cgs)
#pragma unroll
          for (int j = 0; j < 8; ++j) tot[s][j] += (double)smf[q * 8 + j];
      }
    }
    if (tid < cgs) {
      double* o = red_out + (int64_t)(blockIdx.x % SL) * 3 * C + c0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const double mu = mean_invstd ? (double)mean_invstd[c0 + j] : 0.0;
        const double is = mean_invstd ? (double)mean_invstd[C + c0 + j] : 1.0;
        atomicAdd(o + j, tot[0][j]);
        atomicAdd(o + C + j, tot[1][j]);
        atomicAdd(o + 2 * C + j, is * (tot[2][j] - mu * tot[1][j]));      // sum g_pre * ahat
      }
    }
  }
}

// g_s[c] += sum over slices of red[slice][s][c]  (PReLU slope / bias|beta / gamma gradients)
__global__ void stat_grads_kernel(const double* __restrict__ red, int C, int n_stats, float* __restrict__ g0,
                                  float* __restrict__ g1, float* __restrict__ g2) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float* outs[3] = {g0, g1, g2};
  for (int s = 0; s < n_stats && s < 3; ++s) {
    if (!outs[s]) continue;
    double acc = 0;
    for (int i = 0; i < SL; ++i) acc += red[((int64_t)i * n_stats + s) * C + c];
    atomicAdd(outs[s] + c, (float)acc);       // two passes of one network (D real / fake lanes) may run concurrently
  }
}

// ------------------------------------------------------------------------------------------
// layout converters (32 x 32 smem transpose tiles)
// ------------------------------------------------------------------------------------------
__global__ void ncl_to_nlc_kernel(const float* __restrict__ src, int C, int L, void* __restrict__ dst, int dtype) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int c0 = blockIdx.y * 32, l0 = blockIdx.x * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;      // 32 x 8
  for (int i = ty; i < 32; i += 8) {
    const int c = c0 + i, l = l0 + tx;
    tile[i][tx] = (c < C && l < L) ? src[((int64_t)b * C + c) * L + l] : 0.f;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int l = l0 + i, c = c0 + tx;
    if (c < C && l < L) st16(dst, ((int64_t)b * L + l) * C + c, tile[tx][i], dtype);
  }
}
__global__ void nlc_to_ncl_kernel(const void* __restrict__ src, int dtype, int C, int L, float* __restrict__ dst) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int c0 = blockIdx.y * 32, l0 = blockIdx.x * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;
  for (int i = ty; i < 32; i += 8) {
    const int l = l0 + i, c = c0 + tx;
    tile[i][tx] = (c < C && l < L) ? ld16(src, ((int64_t)b * L + l) * C + c, dtype) : 0.f;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int c = c0 + i, l = l0 + tx;
    if (c < C && l < L) dst[((int64_t)b * C + c) * L + l] = tile[tx][i];
  }
}

__global__ void __launch_bounds__(256)
colsum_kernel(const void* __restrict__ a, int dtype, int64_t rows64, int C, double* __restrict__ tmp) {
  constexpr int VEC = 4;
  __shared__ float red[256 * VEC];
  const int cgs = C / VEC;
  const int tid = threadIdx.x;
  const int cg = tid % cgs;
  const int rpb = 256 / cgs;
  const int rows = (int)rows64;
  const int stride = gridDim.x * rpb;
  float part[1][VEC] = {{0.f, 0.f, 0.f, 0.f}};
  for (int r = blockIdx.x * rpb + tid / cgs; r < rows; r += stride) {
    const FV<VEC> v = ldv<VEC>(a, (int64_t)r * C + cg * VEC, dtype);
#pragma unroll
    for (int j = 0; j < VEC; ++j) part[0][j] += v.v[j];
  }
  block_stats_flush<1, VEC>(part, cgs, C, tmp, red);
}
__global__ void colsum_fold_kernel(const double* __restrict__ tmp, int C, int mod, float* __restrict__ out,
                                   int accumulate) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= mod) return;
  double s = 0;
  for (int i = 0; i < SL; ++i)
    for (int c = m; c < C; c += mod) s += tmp[(int64_t)i * C + c];
  out[m] = (accumulate ? out[m] : 0.f) + (float)s;
}

// ------------------------------------------------------------------------------------------
// Discriminator head after fc.0 (discriminator.py:111-117)
// ------------------------------------------------------------------------------------------
constexpr int FC1 = 256, FC2 = 128;

__global__ void __launch_bounds__(256)
fc_tail_fwd_kernel(const float* __restrict__ fc0_acc, const float* __restrict__ b0, const float* __restrict__ s1,
                   const float* __restrict__ w2, const float* __restrict__ b2, const float* __restrict__ s3,
                   const float* __restrict__ w4, const float* __restrict__ b4, float* __restrict__ z1,
                   float* __restrict__ z2, float* __restrict__ logit) {
  __shared__ float h1[FC1];
  __shared__ float h2[FC2];
  __shared__ float wred[8];
  const int b = blockIdx.x, tid = threadIdx.x;
  {
    const float z = fc0_acc[(int64_t)b * FC1 + tid] + b0[tid];
    z1[(int64_t)b * FC1 + tid] = z;
    h1[tid] = z > 0.f ? z : s1[tid] * z;
  }
  __syncthreads();
  // z2[j] = b2[j] + sum_i w2[j][i] h1[i] : one warp per 16 outputs, lanes stride the 256 inputs
  const int warp = tid >> 5, lane = tid & 31;
  for (int j = warp * 16; j < warp * 16 + 16; ++j) {
    float s = 0.f;
    for (int i = lane; i < FC1; i += 32) s = fmaf(w2[j * FC1 + i], h1[i], s);
    s = warp_sum(s);
    if (lane == 0) {
      const float z = s + b2[j];
      z2[(int64_t)b * FC2 + j] = z;
      h2[j] = z > 0.f ? z : s3[j] * z;
    }
  }
  __syncthreads();
  float s = tid < FC2 ? w4[tid] * h2[tid] : 0.f;
  s = warp_sum(s);
  if (lane == 0) wred[warp] = s;
  __syncthreads();
  if (tid == 0) {
    float t = b4[0];
    for (int i = 0; i < 8; ++i) t += wred[i];
    logit[b] = t;
  }
}

// per-row backward: g_z2 [B][128], g_z1 [B][256], g_h1 [B][256] (fp32 workspaces) + bf16 copy of g_z1
__global__ void __launch_bounds__(256)
fc_tail_bwd_rows_kernel(const float* __restrict__ z1, const float* __restrict__ z2, const float* __restrict__ logit,
                        const float* __restrict__ g_logit_in, float target, float weight,
                        const float* __restrict__ s1, const float* __restrict__ w2,
                        const float* __restrict__ s3, const float* __restrict__ w4, int batch,
                        float* __restrict__ loss_out, float* __restrict__ g_logit_ws, float* __restrict__ g_z2_ws,
                        float* __restrict__ g_z1_ws, float* __restrict__ g_h1_ws, void* __restrict__ g_z1_bf16,
                        float gscale, int gdt) {
  __shared__ float gz2[FC2];
  const int b = blockIdx.x, tid = threadIdx.x;
  const float diff = logit[b] - target;
  // gscale: loss scale of the fp16 gradient tensors (every gradient downstream carries it; the loss does not)
  const float gl = g_logit_in ? g_logit_in[b] * gscale : 2.f * diff / (float)batch * weight * gscale;
  if (tid == 0) {
    g_logit_ws[b] = gl;
    if (loss_out) atomicAdd(loss_out, diff * diff / (float)batch * weight);
  }
  if (tid < FC2) {
    const float z = z2[(int64_t)b * FC2 + tid];
    const float gh2 = gl * w4[tid];
    const float g = z > 0.f ? gh2 : gh2 * s3[tid];
    gz2[tid] = g;
    g_z2_ws[(int64_t)b * FC2 + tid] = g;
  }
  __syncthreads();
  float gh1 = 0.f;
  for (int j = 0; j < FC2; ++j) gh1 = fmaf(gz2[j], w2[j * FC1 + tid], gh1);
  const float z = z1[(int64_t)b * FC1 + tid];
  const float g = z > 0.f ? gh1 : gh1 * s1[tid];
  g_z1_ws[(int64_t)b * FC1 + tid] = g;
  g_h1_ws[(int64_t)b * FC1 + tid] = gh1;
  st16(g_z1_bf16, (int64_t)b * FC1 + tid, g, gdt);
}

// parameter gradients of the head: blockIdx.y = chunk of 16 batch rows, one thread per output
// element, partial sums merged with one atomic per (element, chunk)
constexpr int FC_CHUNK = 16;
__global__ void __launch_bounds__(256)
fc_tail_bwd_params_kernel(const float* __restrict__ z1, const float* __restrict__ z2,
                          const float* __restrict__ g_logit, const float* __restrict__ g_z2,
                          const float* __restrict__ g_z1, const float* __restrict__ g_h1,
                          const float* __restrict__ s1, const float* __restrict__ s3,
                          const float* __restrict__ w4, int batch, float* __restrict__ g_b0, float* __restrict__ g_s1, float* __restrict__ g_w2,
                          float* __restrict__ g_b2, float* __restrict__ g_s3, float* __restrict__ g_w4,
                          float* __restrict__ g_b4) {
  __shared__ float h1s[FC_CHUNK][FC1];
  __shared__ float gz2s[FC_CHUNK][FC2];
  const int b0 = blockIdx.y * FC_CHUNK;
  const int nb = min(FC_CHUNK, batch - b0);
  const int tid = threadIdx.x;
  for (int i = tid; i < nb * FC1; i += 256) {
    const int r = i / FC1, c = i % FC1;
    const float z = z1[(int64_t)(b0 + r) * FC1 + c];
    h1s[r][c] = z > 0.f ? z : s1[c] * z;
  }
  for (int i = tid; i < nb * FC2; i += 256) gz2s[i / FC2][i % FC2] = g_z2[(int64_t)(b0 + i / FC2) * FC2 + i % FC2];
  __syncthreads();
  if (blockIdx.x < FC2) {                  // g_w2 row j = blockIdx.x, column i = tid
    const int j = blockIdx.x, i = tid;
    float s = 0.f;
    for (int r = 0; r < nb; ++r) s = fmaf(gz2s[r][j], h1s[r][i], s);
    atomicAdd(g_w2 + j * FC1 + i, s);
    return;
  }
  // last x-block: the vector gradients
  {
    const int i = tid;                     // FC1 outputs: g_b0, g_s1
    float sb = 0.f, ss = 0.f;
    for (int r = 0; r < nb; ++r) {
      const int64_t o = (int64_t)(b0 + r) * FC1 + i;
      sb += g_z1[o];
      const float z = z1[o];
      if (z <= 0.f) ss = fmaf(g_h1[o], z, ss);
    }
    atomicAdd(g_b0 + i, sb);
    atomicAdd(g_s1 + i, ss);
  }
  if (tid < FC2) {
    const int j = tid;
    float sb = 0.f, ss = 0.f, sw = 0.f;
    const float sl = s3[j];
    for (int r = 0; r < nb; ++r) {
      const float z = z2[(int64_t)(b0 + r) * FC2 + j];
      const float gl = g_logit[b0 + r];
      const float g = gz2s[r][j];
      sb += g;
      const float h = z > 0.f ? z : sl * z;
      sw = fmaf(gl, h, sw);
      if (z <= 0.f) ss = fmaf(gl * w4[j], z, ss);        // d s3 = sum g_h2 * z [z<=0], g_h2 = g_logit*w4
    }
    atomicAdd(g_b2 + j, sb);
    atomicAdd(g_s3 + j, ss);
    atomicAdd(g_w4 + j, sw);
  }
  if (tid == 0) {
    float s = 0.f;
    for (int r = 0; r < nb; ++r) s += g_logit[b0 + r];
    atomicAdd(g_b4, s);
  }
}

// G regression loss and its gradient, per element d = y - clean:  REG_L1: |d|, w/n sign(d)  |  REG_MSE: d^2, 2 w/n d.
// The loss is summed deterministically: every block stores its partial (fixed thread order), the last block to
// finish adds the partials up in block order.  The partials and the arrival counter are per device, so launches
// of this kernel must not overlap one another (they run on one stream; the counter is reset for the next launch).
enum { REG_L1 = 0, REG_MSE = 1 };
constexpr int REG_BLOCKS = 2 * NUM_SMS;
__device__ float g_reg_partial[REG_BLOCKS];
__device__ unsigned int g_reg_arrived;

template <int TERM>
__global__ void __launch_bounds__(256) reg_loss_bwd_kernel(const float* __restrict__ y,
                                                           const float* __restrict__ clean, int64_t n, float weight,
                                                           float* __restrict__ loss_out, float* __restrict__ gy,
                                                           int accumulate, float grad_scale) {
  __shared__ float warp_part[8];
  __shared__ bool last;
  float s = 0.f;
  const float lscale = weight / (float)n;
  const float gscale = lscale * grad_scale;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float d = y[i] - clean[i];
    float g;
    if (TERM == REG_L1) {
      s += fabsf(d);
      g = d > 0.f ? gscale : (d < 0.f ? -gscale : 0.f);
    } else {
      s = fmaf(d, d, s);
      g = 2.f * gscale * d;
    }
    if (gy) gy[i] = accumulate ? gy[i] + g : g;
  }
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) warp_part[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float b = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) b += warp_part[w];
    g_reg_partial[blockIdx.x] = b;
    __threadfence();
    last = atomicAdd(&g_reg_arrived, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (last && threadIdx.x < 32) {
    float t = 0.f;
    for (int b = threadIdx.x; b < (int)gridDim.x; b += 32) t += __ldcg(g_reg_partial + b);
    t = warp_sum(t);
    if (threadIdx.x == 0) {
      if (loss_out) *loss_out += t * lscale;
      g_reg_arrived = 0;
    }
  }
}

// ---- streaming-kernel variants (runtime tuning knobs, one per kernel family) -----------------
// vec: channels per thread (4 | 8); unroll: rows in flight per thread and input stream (2 | 4 | 8,
// vec*unroll <= 32); cap: CTAs per SM (the grid is persistent beyond that).  For the two activation-
// backward kernels vec == 8 selects the tiled kernel (unroll 2 | 4), vec == 4 the generic one.
// Kernels that end in a per-block reduction (smem + one double atomic per channel and block) keep
// the grid small so the same-address atomics stay in the hundreds, not thousands.
// TMA-staged versions (stream_ew.cu): variant vec == 16
bool stream_ew_ok(int C);
int launch_bn_stats_bulk(const void* a, int dtype, int64_t rows, int C, double* stats, cudaStream_t st);
int launch_act_fwd_bulk(const void* a, int dtype, int batch, int L, int C, const float* scale_shift, const float* slope,
                        int act, int roll, const int32_t* roll_dev, int H, void* h, cudaStream_t st);
template <int MODE>
int launch_act_bwd_bulk(const void* g_h, int H, int roll, const int32_t* roll_dev, const void* g_add, const void* a,
                        int dtype, int g_dtype, int batch, int L, int C, const float* scale_shift,
                        const float* mean_invstd, const float* slope, int act, const double* red_in, double* red_out,
                        int use_bn, void* g_a_out, cudaStream_t st);

// Defaults (tools/ew_sweep.py compares the variants): the TMA-staged kernels (vec 16) wherever
// they apply -- contiguous 16-bit tensors without twins -- else the register-staged (8, 4, 2); BatchNorm statistics
// (one read-only stream) gain nothing from staging and stay register-staged.
struct EwVariant { int vec, unroll, cap; };
enum { EW_ACT_FWD = 1, EW_BN_STATS = 2, EW_BWD_REDUCE = 3, EW_BWD_APPLY = 4, EW_KINDS = 5 };
static EwVariant g_ew[EW_KINDS] = {{0, 0, 0}, {16, 4, 2}, {4, 8, 3}, {16, 4, 2}, {16, 4, 2}};
static bool g_ew_env_read = false;
static bool ew_valid(int kind, int vec, int unroll, int cap) {
  if (kind < 1 || kind >= EW_KINDS) return false;
  if (vec == 16) return cap >= 1 && cap <= 32;          // TMA-staged kernels: unroll / cap are fixed by the kernel
  if (!((vec == 4 || vec == 8) && (unroll == 2 || unroll == 4 || unroll == 8) && vec * unroll <= 32)) return false;
  if ((kind == EW_BWD_REDUCE || kind == EW_BWD_APPLY) && vec == 8 && unroll > 4) return false;
  return cap >= 1 && cap <= 32;
}
static const EwVariant& ew(int kind) {
  if (!g_ew_env_read) {
    g_ew_env_read = true;
    // SEGAN_B200_EW="kind,vec,unroll,cap[;kind,vec,unroll,cap...]"
    const char* e = getenv("SEGAN_B200_EW");
    while (e && *e) {
      int k, v, u, c;
      if (sscanf(e, "%d,%d,%d,%d", &k, &v, &u, &c) == 4 && ew_valid(k, v, u, c)) g_ew[k] = {v, u, c};
      e = strchr(e, ';');
      if (e) ++e;
    }
  }
  return g_ew[kind];
}
// grid: enough CTAs to cover the rows once, capped at cap_per_sm CTAs per SM (persistent beyond that)
static inline int stream_grid(int64_t rows, int C, int vec, int rows_in_flight, int cap_per_sm) {
  const int rpb = 256 / (C / vec);
  int64_t g = cdiv(rows, (int64_t)rpb * rows_in_flight);
  const int64_t cap = (int64_t)cap_per_sm * NUM_SMS;
  if (g > cap) g = cap;
  return (int)(g < 1 ? 1 : g);
}
// C / vec threads share a row and 256 must be a multiple of that
static inline bool ew_shape_ok(int C) { return C >= 64 && C <= 1024 && (C & (C - 1)) == 0; }

template <int MODE>
static int launch_act_bwd_tiled(const void* g_h, int ldh, int H, int roll, const int32_t* roll_dev, const void* g_add,
                                int lda, const void* a,
                                int dtype, int batch, int L, int C, const float* scale_shift,
                                const float* mean_invstd, const float* slope, int act, const double* red_in,
                                double* red_out, int use_bn, void* g_a_out, int unroll, int cap_per_sm, cudaStream_t st) {
  // 32-bit element offsets inside the kernel
  SG_CHECK_ARG((int64_t)batch * (L + 2 * H) * (ldh > lda ? ldh : lda) < (1ll << 31) && (int64_t)batch * L * C < (1ll << 31));
  int cgs_log2 = 0;
  while ((8 << cgs_log2) < C) ++cgs_log2;               // C / 8 threads per row (C is a power of two >= 64)
  const int RPB = 256 >> cgs_log2;
  const int U = unroll >= 4 ? 4 : 2;
  const int TILE = RPB * U;
  const int tiles_per_b = (L + TILE - 1) / TILE;
  const int64_t total = (int64_t)batch * tiles_per_b;
  int64_t grid = (int64_t)cap_per_sm * NUM_SMS;
  if (grid > total) grid = total;
  const int tiles_per_cta = (int)((total + grid - 1) / grid);
  grid = (total + tiles_per_cta - 1) / tiles_per_cta;
  const size_t smem_const = (size_t)(MODE == 1 ? 6 : 3) * C * sizeof(float);
  const size_t smem_red = MODE == 0 ? 256 * 8 * sizeof(float) : 0;
  const size_t smem = smem_const > smem_red ? smem_const : smem_red;
#define SG_LAUNCH_TILED(UU)                                                                                   \
  act_bwd_tiled_kernel<MODE, UU><<<(int)grid, 256, smem, st>>>(                                                \
      (const uint16_t*)g_h, ldh, H, roll, roll_dev, (const uint16_t*)g_add, lda, (const uint16_t*)a,          \
      dtype == SG_F16,                                                                                       \
      batch, L, C, cgs_log2, scale_shift, mean_invstd, slope, act, red_in, red_out, use_bn, (uint16_t*)g_a_out, \
      tiles_per_b, tiles_per_cta, g_grad_dtype == SG_F16)
  if (U == 4) SG_LAUNCH_TILED(4); else SG_LAUNCH_TILED(2);
#undef SG_LAUNCH_TILED
  return SG_OK;
}

#define EW_DISPATCH(V, U, CALL)                                   \
  do {                                                            \
    if (V == 8 && U == 4) { constexpr int VEC = 8, UNR = 4; CALL; } \
    else if (V == 8 && U == 2) { constexpr int VEC = 8, UNR = 2; CALL; } \
    else if (V == 4 && U == 8) { constexpr int VEC = 4, UNR = 8; CALL; } \
    else if (V == 4 && U == 4) { constexpr int VEC = 4, UNR = 4; CALL; } \
    else { constexpr int VEC = 4, UNR = 2; CALL; }                \
  } while (0)

}  // namespace sg

using namespace sg;

#define ST ((cudaStream_t)stream)

extern "C" int sg_set_ew_variant(int kind, int vec, int unroll, int cap) {
  if (!ew_valid(kind, vec, unroll, cap)) {
    set_error("sg_set_ew_variant(%d,%d,%d,%d): unsupported variant", kind, vec, unroll, cap);
    return SG_ERR_INVALID;
  }
  ew(kind);                      // make sure the environment was read first (explicit calls win)
  g_ew[kind] = {vec, unroll, cap};
  return SG_OK;
}

extern "C" int sg_bn_stats(const void* a, int dtype, int64_t rows_total, int C, double* stats, void* stream) {
  SG_CHECK_ARG(ew_shape_ok(C) && a && stats && rows_total < (1ll << 31));
  const EwVariant v = ew(EW_BN_STATS);
  if (v.vec == 16 && (dtype == SG_F16 || dtype == SG_BF16) && stream_ew_ok(C)) {
    int rc = launch_bn_stats_bulk(a, dtype, rows_total, C, stats, ST);
    if (rc) return rc;
    SG_CHECK_LAUNCH();
    return SG_OK;
  }
  EW_DISPATCH(v.vec == 16 ? 4 : v.vec, v.vec == 16 ? 4 : v.unroll, (bn_stats_kernel<VEC, UNR><<<stream_grid(rows_total, C, VEC, 2 * UNR, v.cap), 256, 0, ST>>>(
      a, dtype, rows_total, C, stats)));
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_bn_finalize(const double* stats, int64_t count, int C, const float* gamma, const float* beta,
                              float eps, float momentum, float* running_mean, float* running_var,
                              float* scale_shift, float* mean_invstd, void* stream) {
  bn_finalize_kernel<<<(C + 127) / 128, 128, 0, ST>>>(stats, (double)count, C, gamma, beta, eps, momentum,
                                                      running_mean, running_var, scale_shift, mean_invstd);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_act_fwd(const void* a, int dtype, int batch, int L, int C, const float* scale_shift,
                          const float* slope, int act, int roll, const int32_t* roll_dev, int out_halo_pos, void* h,
                          void* h_bf16, void* a_bf16, void* stream) {
  SG_CHECK_ARG(ew_shape_ok(C) && (out_halo_pos == 0 || L > out_halo_pos));      // reflect padding needs pad < L
  SG_CHECK_ARG(act == SG_ACT_NONE || (act == SG_ACT_PRELU && slope));
  const EwVariant v = ew(EW_ACT_FWD);
  if (v.vec == 16 && (dtype == SG_F16 || dtype == SG_BF16) && stream_ew_ok(C) && !h_bf16 && !a_bf16 && h &&
      (out_halo_pos == 0 || L >= 2 * out_halo_pos + 3)) {
    int rc = launch_act_fwd_bulk(a, dtype, batch, L, C, scale_shift, slope, act, roll, roll_dev, out_halo_pos, h, ST);
    if (rc) return rc;
    SG_CHECK_LAUNCH();
    return SG_OK;
  }
  EW_DISPATCH(v.vec == 16 ? 8 : v.vec, v.vec == 16 ? 4 : v.unroll, (act_fwd_kernel<VEC, UNR><<<stream_grid((int64_t)batch * (L + 2 * out_halo_pos), C, VEC, 2 * UNR, v.cap), 256, 0, ST>>>(
      a, dtype, batch, L, C, scale_shift, slope, act, roll, roll_dev, out_halo_pos, h, h_bf16, a_bf16)));
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_act_bwd_reduce(const void* g_h, int g_h_ld, int in_halo_pos, int roll, const int32_t* roll_dev,
                                 const void* g_add, int g_add_ld, const void* a,
                                 int dtype, int batch, int L, int C, const float* scale_shift,
                                 const float* mean_invstd, const float* slope, int act, double* red,
                                 void* g_a_out, void* stream) {
  SG_CHECK_ARG(ew_shape_ok(C) && red && a && (in_halo_pos == 0 || L >= 2 * in_halo_pos + 3));
  SG_CHECK_ARG(dtype == SG_F16 || dtype == SG_BF16);
  const EwVariant v = ew(EW_BWD_REDUCE);
  const int ldh = g_h_ld > 0 ? g_h_ld : C, lda = g_add_ld > 0 ? g_add_ld : C;
  if (v.vec == 16 && g_h && ldh == C && (!g_add || lda == C) && stream_ew_ok(C)) {
    int rc = launch_act_bwd_bulk<0>(g_h, in_halo_pos, roll, roll_dev, g_add, a, dtype, g_grad_dtype, batch, L, C,
                                    scale_shift, mean_invstd, slope, act, nullptr, red, 0, g_a_out, ST);
    if (rc) return rc;
    SG_CHECK_LAUNCH();
    return SG_OK;
  }
  if (v.vec >= 8 && g_h && ldh % 8 == 0 && lda % 8 == 0) {
    int rc = launch_act_bwd_tiled<0>(g_h, ldh, in_halo_pos, roll, roll_dev, g_add, lda, a, dtype, batch, L, C, scale_shift,
                                     mean_invstd, slope, act, nullptr, red, 0, g_a_out, v.unroll, v.cap, ST);
    if (rc) return rc;
    SG_CHECK_LAUNCH();
    return SG_OK;
  }
  EW_DISPATCH(4, v.unroll, (act_bwd_kernel<0, VEC, UNR><<<stream_grid((int64_t)batch * L, C, VEC, UNR, v.cap), 256, 0, ST>>>(
      g_h, ldh, in_halo_pos, roll, roll_dev, g_add, lda, a, dtype, batch, L, C,
      scale_shift, mean_invstd, slope, act, red, 0, g_a_out, g_grad_dtype)));
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_act_bwd_apply(const void* g_h, int g_h_ld, int in_halo_pos, int roll, const int32_t* roll_dev,
                                const void* g_add, int g_add_ld, const void* a,
                                int dtype, int batch, int L, int C, const float* scale_shift,
                                const float* mean_invstd, const float* slope, int act, const double* red,
                                int use_bn, void* g_a, void* stream) {
  SG_CHECK_ARG(ew_shape_ok(C) && red && g_a && a && (in_halo_pos == 0 || L >= 2 * in_halo_pos + 3));
  SG_CHECK_ARG(dtype == SG_F16 || dtype == SG_BF16);
  SG_CHECK_ARG(!use_bn || (scale_shift && mean_invstd));
  const EwVariant v = ew(EW_BWD_APPLY);
  const int ldh = g_h_ld > 0 ? g_h_ld : C, lda = g_add_ld > 0 ? g_add_ld : C;
  if (v.vec == 16 && g_h && ldh == C && (!g_add || lda == C) && stream_ew_ok(C)) {
    int rc = launch_act_bwd_bulk<1>(g_h, in_halo_pos, roll, roll_dev, g_add, a, dtype, g_grad_dtype, batch, L, C,
                                    scale_shift, mean_invstd, slope, act, red, nullptr, use_bn, g_a, ST);
    if (rc) return rc;
    SG_CHECK_LAUNCH();
    return SG_OK;
  }
  if (v.vec >= 8 && g_h && ldh % 8 == 0 && lda % 8 == 0) {
    int rc = launch_act_bwd_tiled<1>(g_h, ldh, in_halo_pos, roll, roll_dev, g_add, lda, a, dtype, batch, L, C, scale_shift,
                                     mean_invstd, slope, act, red, nullptr, use_bn, g_a, v.unroll, v.cap, ST);
    if (rc) return rc;
    SG_CHECK_LAUNCH();
    return SG_OK;
  }
  EW_DISPATCH(4, v.unroll, (act_bwd_kernel<1, VEC, UNR><<<stream_grid((int64_t)batch * L, C, VEC, UNR, v.cap), 256, 0, ST>>>(
      g_h, ldh, in_halo_pos, roll, roll_dev, g_add, lda, a, dtype, batch, L, C,
      scale_shift, mean_invstd, slope, act, const_cast<double*>(red), use_bn, g_a, g_grad_dtype)));
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_stat_grads(const double* red, int C, int n_stats, float* g0, float* g1, float* g2, void* stream) {
  SG_CHECK_ARG(red && C > 0 && n_stats >= 1 && n_stats <= 3);
  stat_grads_kernel<<<(C + 127) / 128, 128, 0, ST>>>(red, C, n_stats, g0, g1, g2);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

// out[r][col0 + c] = (16-bit) ws[r][col0 + c]: final step of a split-K tail (fp32 partial sums -> the layer's tensor)
__global__ void convert_f32_rows_kernel(const float* __restrict__ ws, void* __restrict__ out, int dtype, int64_t rows,
                                        int ld, int col0, int ncols) {
  const int64_t total = rows * (ncols / 8);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / (ncols / 8);
    const int c = (int)(i % (ncols / 8)) * 8;
    const int64_t off = r * ld + col0 + c;
    const float4 a = *reinterpret_cast<const float4*>(ws + off);
    const float4 b = *reinterpret_cast<const float4*>(ws + off + 4);
    const float x[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    stv<8>(out, off, x, dtype);
  }
}

extern "C" int sg_convert_f32_rows(const float* ws, void* out, int dtype, int64_t rows, int ld, int col0, int ncols,
                                   void* stream) {
  SG_CHECK_ARG(ws && out && rows > 0 && ncols > 0 && ncols % 8 == 0 && col0 % 8 == 0 && ld % 8 == 0);
  SG_CHECK_ARG(dtype == SG_F16 || dtype == SG_BF16);
  const int64_t total = rows * (ncols / 8);
  int64_t g = (total + 255) / 256;
  if (g > 8 * NUM_SMS) g = 8 * NUM_SMS;
  convert_f32_rows_kernel<<<(int)g, 256, 0, ST>>>(ws, out, dtype, rows, ld, col0, ncols);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_ncl_to_nlc(const float* src, int batch, int C, int L, void* dst, int dtype, void* stream) {
  dim3 grid((L + 31) / 32, (C + 31) / 32, batch), block(32, 8);
  ncl_to_nlc_kernel<<<grid, block, 0, ST>>>(src, C, L, dst, dtype);
  SG_CHECK_LAUNCH();
  return SG_OK;
}
extern "C" int sg_nlc_to_ncl(const void* src, int dtype, int batch, int C, int L, float* dst, void* stream) {
  dim3 grid((L + 31) / 32, (C + 31) / 32, batch), block(32, 8);
  nlc_to_ncl_kernel<<<grid, block, 0, ST>>>(src, dtype, C, L, dst);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_colsum(const void* a, int dtype, int64_t rows, int C, int mod, float* out, int accumulate,
                         double* tmp, void* stream) {
  SG_CHECK_ARG(ew_shape_ok(C) && tmp && C % mod == 0);
  SG_CHECK_CUDA(cudaMemsetAsync(tmp, 0, sizeof(double) * C * SL, ST));
  colsum_kernel<<<stream_grid(rows, C, 4, 1, 3), 256, 0, ST>>>(a, dtype, rows, C, tmp);
  SG_CHECK_LAUNCH();
  colsum_fold_kernel<<<(mod + 127) / 128, 128, 0, ST>>>(tmp, C, mod, out, accumulate);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_fc_tail_fwd(const float* fc0_acc, const float* b0, const float* s1, const float* w2,
                              const float* b2, const float* s3, const float* w4, const float* b4, int batch,
                              float* z1, float* z2, float* logit, void* stream) {
  SG_CHECK_ARG(batch > 0 && fc0_acc && b0 && s1 && w2 && b2 && s3 && w4 && b4 && z1 && z2 && logit);
  fc_tail_fwd_kernel<<<batch, 256, 0, ST>>>(fc0_acc, b0, s1, w2, b2, s3, w4, b4, z1, z2, logit);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_fc_tail_bwd(const float* z1, const float* z2, const float* logit, const float* g_logit_in,
                              float target, float weight,
                              const float* s1, const float* w2, const float* s3, const float* w4, int batch,
                              float* loss_out, void* g_z1_bf16, float* ws /* [B*(1+128+256+256)] */, float* g_b0,
                              float* g_s1, float* g_w2, float* g_b2, float* g_s3, float* g_w4, float* g_b4,
                              float grad_scale, void* stream) {
  SG_CHECK_ARG(batch > 0 && z1 && z2 && logit && s1 && w2 && s3 && w4 && ws && g_z1_bf16);
  // g_w2 == NULL skips the parameter gradients (the G step); otherwise the kernel adds into every one of them
  SG_CHECK_ARG(!g_w2 || (g_b0 && g_s1 && g_b2 && g_s3 && g_w4 && g_b4));
  float* g_logit = ws;
  float* g_z2 = ws + batch;
  float* g_z1 = g_z2 + (int64_t)batch * FC2;
  float* g_h1 = g_z1 + (int64_t)batch * FC1;
  fc_tail_bwd_rows_kernel<<<batch, 256, 0, ST>>>(z1, z2, logit, g_logit_in, target, weight, s1, w2, s3, w4, batch,
                                                 loss_out, g_logit, g_z2, g_z1, g_h1, g_z1_bf16, grad_scale,
                                                 g_grad_dtype);
  SG_CHECK_LAUNCH();
  if (g_w2) {
    dim3 grid(FC2 + 1, (batch + FC_CHUNK - 1) / FC_CHUNK);
    fc_tail_bwd_params_kernel<<<grid, 256, 0, ST>>>(z1, z2, g_logit, g_z2, g_z1, g_h1, s1, s3, w4, batch, g_b0, g_s1,
                                                    g_w2, g_b2, g_s3, g_w4, g_b4);
    SG_CHECK_LAUNCH();
  }
  return SG_OK;
}

extern "C" int sg_l1_loss_bwd(const float* y, const float* clean, int64_t n, float weight, float* loss_out,
                              float* gy, int accumulate, float grad_scale, void* stream) {
  SG_CHECK_ARG(n > 0 && y && clean);
  reg_loss_bwd_kernel<REG_L1><<<REG_BLOCKS, 256, 0, ST>>>(y, clean, n, weight, loss_out, gy, accumulate, grad_scale);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_mse_loss_bwd(const float* y, const float* clean, int64_t n, float weight, float* loss_out,
                               float* gy, int accumulate, float grad_scale, void* stream) {
  SG_CHECK_ARG(n > 0 && y && clean);
  reg_loss_bwd_kernel<REG_MSE><<<REG_BLOCKS, 256, 0, ST>>>(y, clean, n, weight, loss_out, gy, accumulate, grad_scale);
  SG_CHECK_LAUNCH();
  return SG_OK;
}
