// HBM-bound glue kernels of the activation path, TMA-staged (SURVEY.md 8a: BatchNorm statistics, BN + PReLU forward
// with reflect halo + phase shift, and the two passes of their backward).
//
// The register-staged versions in elementwise.cu keep 32-48 KB of loads in flight per SM (256-thread CTAs x 2, a few
// 16-byte loads per thread).  With ~1 us of loaded HBM latency, streaming at HBM rate needs more bytes in flight per SM
// than the register file can hold next to the per-channel accumulators.  Here the bytes in flight live in shared memory instead: one producer thread
// per CTA streams contiguous row tiles with cp.async.bulk (1-D TMA, mbarrier complete_tx) through a ring of 16 KB
// stages -- 64-96 KB in flight per CTA, two CTAs per SM -- and eight consumer warps read the tiles with
// conflict-free 16-byte shared loads.  Outputs are coalesced 16-byte global stores.
//
// Tiles are runs of rows of ONE batch element.  The Discriminator's circular phase shift (discriminator.py:165-172)
// makes the consumer-view tensor a rotation of the exact-geometry one: each batch element is cut at the wrap point
// into two row ranges, so every tile is contiguous in BOTH tensors.
#include "common.cuh"

namespace sg {

__device__ __forceinline__ uint32_t s_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void sb_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s_u32(bar)), "r"(count));
}
__device__ __forceinline__ void sb_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void sb_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(s_u32(bar)) : "memory");
}
__device__ __forceinline__ uint32_t sb_try(uint32_t addr, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(done)
      : "r"(addr), "r"(parity)
      : "memory");
  return done;
}
__device__ __forceinline__ void sb_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = s_u32(bar);
  if (sb_try(addr, parity)) return;
  long long t0 = 0;                 // watchdog: a pipeline bug surfaces as a launch error, never as a hung GPU
  uint32_t spins = 0;
  while (!sb_try(addr, parity)) {
    if ((++spins & 1023u) == 0) {
      const long long now = clock64();
      if (t0 == 0) t0 = now;
      else if (now - t0 > 8000000000LL) __trap();
    }
  }
}
// 1-D bulk copy global -> shared (bytes: multiple of 16; both addresses 16-byte aligned)
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(s_u32(dst)), "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(s_u32(bar))
               : "memory");
}
__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

constexpr int SL = SG_STAT_SLICES;
constexpr int SE_CONSUMERS = 256;           // 8 consumer warps + 1 producer warp
constexpr int SE_THREADS = SE_CONSUMERS + 32;
constexpr int SE_U = 4;                     // row passes per tile: tile rows = SE_U * (256 / (C / 8))
constexpr int SE_MAX_STAGES = 6;

struct U4 { uint32_t w[4]; };
__device__ __forceinline__ U4 lds16(const uint16_t* p) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  U4 r; r.w[0] = u.x; r.w[1] = u.y; r.w[2] = u.z; r.w[3] = u.w;
  return r;
}
__device__ __forceinline__ U4 ldg16(const uint16_t* p) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  U4 r; r.w[0] = u.x; r.w[1] = u.y; r.w[2] = u.z; r.w[3] = u.w;
  return r;
}
__device__ __forceinline__ void unpack8(const U4& x, bool f16, float (&v)[8]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 f;
    if (f16) f = __half22float2(*reinterpret_cast<const __half2*>(&x.w[i]));
    else f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&x.w[i]));
    v[2 * i] = f.x; v[2 * i + 1] = f.y;
  }
}
// fp16 stores saturate at +-65504 (as in elementwise.cu and the tap-GEMM epilogue): every variant stores the same bits
__device__ __forceinline__ uint4 pack8(const float (&v)[8], bool f16) {
  uint32_t w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (f16) {
      w[i] = pack_half2_sat(v[2 * i], v[2 * i + 1]);
    } else {
      __nv_bfloat162 h2 = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
      w[i] = *reinterpret_cast<uint32_t*>(&h2);
    }
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}
__device__ __forceinline__ void lds_f8(const float* p, float (&v)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p);
  const float4 b = *reinterpret_cast<const float4*>(p + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

// Row tiles of a rotated batch element.  rp = roll mod L: exact rows [0, L - rp) sit at consumer rows [rp, L) (range
// A) and exact rows [L - rp, L) at consumer rows [0, rp) (range B).
struct TileWalk {
  int RT, L, LA, nA, tpb, total;
  int b, i;                                      // current tile: batch element, index within it
  __device__ __forceinline__ void init(int L_, int rp, int RT_, int batch) {
    RT = RT_; L = L_; LA = L_ - rp;
    nA = (LA + RT - 1) / RT;
    tpb = nA + (rp + RT - 1) / RT;
    total = batch * tpb;
  }
  __device__ __forceinline__ void seek(int t) { b = t / tpb; i = t - b * tpb; }
  __device__ __forceinline__ void step() { if (++i == tpb) { i = 0; ++b; } }
  // first exact row, row count, first consumer row of the current tile
  __device__ __forceinline__ void get(int& l0, int& n, int& qs) const {
    if (i < nA) { l0 = i * RT; n = min(RT, LA - l0); qs = l0 + (L - LA); }
    else { l0 = LA + (i - nA) * RT; n = min(RT, L - l0); qs = l0 - LA; }
  }
};

// combine per-thread partial sums part[NS][8] over the threads that own the same 8 channels, one double atomic per
// channel, statistic and CTA into slice (CTA % SL) of out[SL][NS][C]; sm: >= 256 * 8 floats, consumers only
template <int NS>
__device__ __forceinline__ void se_flush(float (&part)[NS][8], int cgs, int C, int c0, double* out, float* sm, int tid,
                                         const float* mean_invstd, bool centre) {
  double tot[NS][8];
  for (int s = 0; s < NS; ++s) {
    consumers_sync();
#pragma unroll
    for (int j = 0; j < 8; ++j) sm[tid * 8 + j] = part[s][j];
    consumers_sync();
    if (tid < cgs) {
#pragma unroll
      for (int j = 0; j < 8; ++j) tot[s][j] = 0;
      for (int q = tid; q < SE_CONSUMERS; q += cgs)
#pragma unroll
        for (int j = 0; j < 8; ++j) tot[s][j] += (double)sm[q * 8 + j];
    }
  }
  if (tid < cgs) {
    double* o = out + (int64_t)(blockIdx.x % SL) * NS * C + c0;
    if (!centre) {
      for (int s = 0; s < NS; ++s)
#pragma unroll
        for (int j = 0; j < 8; ++j) atomicAdd(o + (int64_t)s * C + j, tot[s][j]);
    } else {
      // activation backward (NS == 3): sum(g_pre * x) is centred into sum(g_pre * ahat) here, in double
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const double mu = mean_invstd ? (double)mean_invstd[c0 + j] : 0.0;
        const double is = mean_invstd ? (double)mean_invstd[C + c0 + j] : 1.0;
        atomicAdd(o + j, tot[0][j]);
        atomicAdd(o + C + j, tot[1][j]);
        atomicAdd(o + 2 * C + j, is * (tot[NS - 1][j] - mu * tot[1][j]));
      }
    }
  }
}

struct SeBwd {
  const uint16_t* g_h; const uint16_t* g_add; const uint16_t* a;
  uint16_t* g_a_out;
  const float* scale_shift; const float* mean_invstd; const float* slope;
  const double* red_in; double* red_out;
  const int* roll_dev;
  int H, roll, batch, L, C, cgs_log2, act, use_bn, a_f16, g_f16, nstages;
};

// dynamic smem: [full[S] | empty[S]] barriers (128 B) | per-channel constants 6 * C floats | S stages of
// ntens * TILE bytes (TILE = SE_U * RPB rows * C * 2 = 16 KB)
template <int MODE>
__global__ void __launch_bounds__(SE_THREADS, 2)
act_bwd_bulk_kernel(const SeBwd p) {
  extern __shared__ __align__(128) uint8_t se_smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(se_smem);
  uint64_t* empty = full + SE_MAX_STAGES;
  float* cst = reinterpret_cast<float*>(se_smem + 128);
  const int C = p.C, L = p.L, H = p.H;
  const int ntens = p.g_add ? 3 : 2;
  const int tile_bytes = 16384;
  uint8_t* stages = se_smem + 128 + (((MODE == 1 ? 6 : 3) * C * 4 + 127) & ~127);
  const int tid = threadIdx.x;
  const int S = p.nstages;
  if (tid == 0) {
    for (int s = 0; s < S; ++s) { sb_init(&full[s], 1); sb_init(&empty[s], SE_CONSUMERS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  int roll = p.roll_dev ? *p.roll_dev : p.roll;
  int rp = roll % L;
  if (rp < 0) rp += L;
  const int cgs = 1 << p.cgs_log2;
  const int RPB = SE_CONSUMERS >> p.cgs_log2;
  const int RT = SE_U * RPB;
  TileWalk tw;
  tw.init(L, rp, RT, p.batch);
  const int per_cta = (tw.total + gridDim.x - 1) / gridDim.x;
  const int t_begin = blockIdx.x * per_cta;
  const int t_end = min(t_begin + per_cta, tw.total);
  const int Lh = L + 2 * H;
  __syncthreads();

  if (tid >= SE_CONSUMERS) {
    // ---------------- producer: one thread issues the bulk copies
    if (tid == SE_CONSUMERS && t_begin < t_end) {
      tw.seek(t_begin);
      int it = 0;
      for (int t = t_begin; t < t_end; ++t, ++it, tw.step()) {
        const int st = it % S;
        sb_wait(&empty[st], ((it / S) & 1) ^ 1);
        int l0, n, qs;
        tw.get(l0, n, qs);
        const uint32_t bytes = (uint32_t)n * C * 2;
        uint8_t* dst = stages + (size_t)st * ntens * tile_bytes;
        sb_expect_tx(&full[st], bytes * ntens);
        bulk_g2s(dst, p.a + ((int64_t)tw.b * L + l0) * C, bytes, &full[st]);
        bulk_g2s(dst + tile_bytes, p.g_h + ((int64_t)tw.b * Lh + H + qs) * C, bytes, &full[st]);
        if (p.g_add) bulk_g2s(dst + 2 * tile_bytes, p.g_add + ((int64_t)tw.b * L + l0) * C, bytes, &full[st]);
      }
    }
    return;
  }

  // ---------------- consumers
  float* s_sc = cst;
  float* s_sh = cst + C;
  float* s_sl = cst + 2 * C;
  float* s_so = cst + 3 * C;
  float* s_ka = cst + 4 * C;
  float* s_kb = cst + 5 * C;
  const int rows_total = p.batch * L;
  for (int c = tid; c < C; c += SE_CONSUMERS) {
    const float sc = p.scale_shift ? p.scale_shift[c] : 1.f;
    s_sc[c] = sc;
    s_sh[c] = p.scale_shift ? p.scale_shift[C + c] : 0.f;
    s_sl[c] = (p.act == SG_ACT_PRELU) ? p.slope[c] : 1.f;
    if (MODE == 1) {
      float so = 1.f, ka = 0.f, kb = 0.f;
      if (p.use_bn) {
        double d1 = 0, d2 = 0;
        for (int i = 0; i < SL; ++i) {
          d1 += p.red_in[((int64_t)i * 3 + 1) * C + c];
          d2 += p.red_in[((int64_t)i * 3 + 2) * C + c];
        }
        const float r1 = (float)(d1 / (double)rows_total);
        const float r2 = (float)(d2 / (double)rows_total);
        const float mu = p.mean_invstd[c], is = p.mean_invstd[C + c];
        so = sc;
        ka = -sc * r2 * is;
        kb = sc * (r2 * is * mu - r1);
      }
      s_so[c] = so; s_ka[c] = ka; s_kb[c] = kb;
    }
  }
  consumers_sync();

  const int cg = tid & (cgs - 1);
  const int rr = tid >> p.cgs_log2;
  const int c0 = cg * 8;
  const bool f16 = p.a_f16 != 0, gf16 = p.g_f16 != 0;
  const bool prelu = p.act == SG_ACT_PRELU;
  float part[3][8];
#pragma unroll
  for (int s = 0; s < 3; ++s)
#pragma unroll
    for (int j = 0; j < 8; ++j) part[s][j] = 0.f;
  // a thread owns the same 8 channels for the whole kernel: their constants live in registers (shared-memory copies
  // would cost 3-6x the tile's own shared-memory traffic)
  float sc[8], sh[8], sl[8], so[8], ka[8], kb[8];
  lds_f8(s_sc + c0, sc); lds_f8(s_sh + c0, sh); lds_f8(s_sl + c0, sl);
  if (MODE == 1) { lds_f8(s_so + c0, so); lds_f8(s_ka + c0, ka); lds_f8(s_kb + c0, kb); }

  if (t_begin < t_end) tw.seek(t_begin);
  int it = 0;
  for (int t = t_begin; t < t_end; ++t, ++it, tw.step()) {
    const int st = it % S;
    int l0, n, qs;
    tw.get(l0, n, qs);
    // reflect-halo mirrors of this thread's rows (modules.py:92-98 backward): fetched from global memory before the
    // tile is waited for, so their latency hides behind the bulk copy
    U4 gm[SE_U];
    unsigned hm = 0;
    if (H > 0) {
#pragma unroll
      for (int u = 0; u < SE_U; ++u) {
        const int r = rr + u * RPB;
        if (r < n) {
          const int q0 = qs + r;
          int m = 0;
          bool has = false;
          if ((unsigned)(q0 - 1) < (unsigned)H) { m = -q0; has = true; }
          else if ((unsigned)(L - 2 - q0) < (unsigned)H) { m = 2 * (L - 1) - q0; has = true; }
          if (has) { gm[u] = ldg16(p.g_h + ((int64_t)tw.b * Lh + H + m) * C + c0); hm |= 1u << u; }
        }
      }
    }
    sb_wait(&full[st], (it / S) & 1);
    const uint16_t* sa = reinterpret_cast<const uint16_t*>(stages + (size_t)st * ntens * tile_bytes);
    const uint16_t* sg = sa + tile_bytes / 2;
    const uint16_t* sd = sg + tile_bytes / 2;
#pragma unroll
    for (int u = 0; u < SE_U; ++u) {
      const int r = rr + u * RPB;
      if (r < n) {
        float x[8], g[8], out[8];
        unpack8(lds16(sa + r * C + c0), f16, x);
        unpack8(lds16(sg + r * C + c0), gf16, g);
        if (hm & (1u << u)) {
          float m[8];
          unpack8(gm[u], gf16, m);
#pragma unroll
          for (int j = 0; j < 8; ++j) g[j] += m[j];
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float y = fmaf(x[j], sc[j], sh[j]);
          const bool neg = prelu && y <= 0.f;
          if (MODE == 0 && neg) part[0][j] = fmaf(g[j], y, part[0][j]);
          g[j] = neg ? g[j] * sl[j] : g[j];                   // g_pre
        }
        if (p.g_add) {
          float sk[8];
          unpack8(lds16(sd + r * C + c0), gf16, sk);
#pragma unroll
          for (int j = 0; j < 8; ++j) g[j] += sk[j];
        }
        if (MODE == 0) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            part[1][j] += g[j];
            part[2][j] = fmaf(g[j], x[j], part[2][j]);
            out[j] = g[j];
          }
        } else {
#pragma unroll
          for (int j = 0; j < 8; ++j) out[j] = fmaf(so[j], g[j], fmaf(ka[j], x[j], kb[j]));
        }
        if (p.g_a_out)
          *reinterpret_cast<uint4*>(p.g_a_out + ((int64_t)tw.b * L + l0 + r) * C + c0) = pack8(out, gf16);
      }
    }
    __syncwarp();
    if ((tid & 31) == 0) sb_arrive(&empty[st]);
  }
  if (MODE == 0) {
    // every consumer is past its last stage read (the arithmetic above only touched registers and the constants):
    // stage 0 is free to serve as the 8 KB combine buffer once all of them are here
    consumers_sync();
    se_flush<3>(part, cgs, C, c0, p.red_out, reinterpret_cast<float*>(stages), tid, p.mean_invstd, true);
  }
}

// ------------------------------------------------------------------------------------------
// BatchNorm batch statistics: stats[slice][0][c] += sum x, stats[slice][1][c] += sum x^2 over [rows][C]
// one tensor: 32 KB tiles
// ------------------------------------------------------------------------------------------
constexpr int SE_U1 = 8;
__global__ void __launch_bounds__(SE_THREADS, 2)
bn_stats_bulk_kernel(const uint16_t* __restrict__ a, int a_f16, int rows, int C, int cgs_log2, int nstages,
                     double* __restrict__ stats) {
  extern __shared__ __align__(128) uint8_t se_smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(se_smem);
  uint64_t* empty = full + SE_MAX_STAGES;
  uint8_t* stages = se_smem + 128;
  const int tile_bytes = 32768;
  const int tid = threadIdx.x;
  const int S = nstages;
  if (tid == 0) {
    for (int s = 0; s < S; ++s) { sb_init(&full[s], 1); sb_init(&empty[s], SE_CONSUMERS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  const int cgs = 1 << cgs_log2;
  const int RPB = SE_CONSUMERS >> cgs_log2;
  const int RT = SE_U1 * RPB;
  const int total = (rows + RT - 1) / RT;
  const int per_cta = (total + gridDim.x - 1) / gridDim.x;
  const int t_begin = blockIdx.x * per_cta;
  const int t_end = min(t_begin + per_cta, total);
  __syncthreads();
  if (tid >= SE_CONSUMERS) {
    if (tid == SE_CONSUMERS) {
      int it = 0;
      for (int t = t_begin; t < t_end; ++t, ++it) {
        const int st = it % S;
        sb_wait(&empty[st], ((it / S) & 1) ^ 1);
        const int r0 = t * RT;
        const uint32_t bytes = (uint32_t)min(RT, rows - r0) * C * 2;
        sb_expect_tx(&full[st], bytes);
        bulk_g2s(stages + (size_t)st * tile_bytes, a + (int64_t)r0 * C, bytes, &full[st]);
      }
    }
    return;
  }
  const int cg = tid & (cgs - 1);
  const int rr = tid >> cgs_log2;
  const int c0 = cg * 8;
  const bool f16 = a_f16 != 0;
  float part[2][8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { part[0][j] = 0.f; part[1][j] = 0.f; }
  int it = 0;
  for (int t = t_begin; t < t_end; ++t, ++it) {
    const int st = it % S;
    const int n = min(RT, rows - t * RT);
    sb_wait(&full[st], (it / S) & 1);
    const uint16_t* sa = reinterpret_cast<const uint16_t*>(stages + (size_t)st * tile_bytes);
    U4 av[SE_U1];
#pragma unroll
    for (int u = 0; u < SE_U1; ++u) {
      const int r = rr + u * RPB;
      if (r < n) av[u] = lds16(sa + r * C + c0);
    }
    __syncwarp();
    if ((tid & 31) == 0) sb_arrive(&empty[st]);
#pragma unroll
    for (int u = 0; u < SE_U1; ++u) {
      const int r = rr + u * RPB;
      if (r < n) {
        float x[8];
        unpack8(av[u], f16, x);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          part[0][j] += x[j];
          part[1][j] = fmaf(x[j], x[j], part[1][j]);
        }
      }
    }
  }
  consumers_sync();
  se_flush<2>(part, cgs, C, c0, stats, reinterpret_cast<float*>(stages), tid, nullptr, false);
}

// ------------------------------------------------------------------------------------------
// h[b][H + q][c] = act(a[b][l][c] * scale + shift) at q = (l + roll) mod L, and on the reflect-halo row that mirrors
// q when q lies within H of an end (modules.py:92-98).  One input tensor (32 KB tiles), scattered row stores.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SE_THREADS, 2)
act_fwd_bulk_kernel(const uint16_t* __restrict__ a, int a_f16, int batch, int L, int C, int cgs_log2, int nstages,
                    const float* __restrict__ scale_shift, const float* __restrict__ slope, int act, int roll,
                    const int* __restrict__ roll_dev, int H, uint16_t* __restrict__ h) {
  extern __shared__ __align__(128) uint8_t se_smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(se_smem);
  uint64_t* empty = full + SE_MAX_STAGES;
  float* cst = reinterpret_cast<float*>(se_smem + 128);
  uint8_t* stages = se_smem + 128 + ((3 * C * 4 + 127) & ~127);
  const int tile_bytes = 32768;
  const int tid = threadIdx.x;
  const int S = nstages;
  if (tid == 0) {
    for (int s = 0; s < S; ++s) { sb_init(&full[s], 1); sb_init(&empty[s], SE_CONSUMERS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (roll_dev) roll = *roll_dev;
  int rp = roll % L;
  if (rp < 0) rp += L;
  const int cgs = 1 << cgs_log2;
  const int RPB = SE_CONSUMERS >> cgs_log2;
  const int RT = SE_U1 * RPB;
  TileWalk tw;
  tw.init(L, rp, RT, batch);
  const int per_cta = (tw.total + gridDim.x - 1) / gridDim.x;
  const int t_begin = blockIdx.x * per_cta;
  const int t_end = min(t_begin + per_cta, tw.total);
  const int Lh = L + 2 * H;
  __syncthreads();
  if (tid >= SE_CONSUMERS) {
    if (tid == SE_CONSUMERS && t_begin < t_end) {
      tw.seek(t_begin);
      int it = 0;
      for (int t = t_begin; t < t_end; ++t, ++it, tw.step()) {
        const int st = it % S;
        sb_wait(&empty[st], ((it / S) & 1) ^ 1);
        int l0, n, qs;
        tw.get(l0, n, qs);
        const uint32_t bytes = (uint32_t)n * C * 2;
        sb_expect_tx(&full[st], bytes);
        bulk_g2s(stages + (size_t)st * tile_bytes, a + ((int64_t)tw.b * L + l0) * C, bytes, &full[st]);
      }
    }
    return;
  }
  for (int c = tid; c < C; c += SE_CONSUMERS) {
    cst[c] = scale_shift ? scale_shift[c] : 1.f;
    cst[C + c] = scale_shift ? scale_shift[C + c] : 0.f;
    cst[2 * C + c] = (act == SG_ACT_PRELU) ? slope[c] : 1.f;
  }
  consumers_sync();
  const int cg = tid & (cgs - 1);
  const int rr = tid >> cgs_log2;
  const int c0 = cg * 8;
  const bool f16 = a_f16 != 0;
  const bool prelu = act == SG_ACT_PRELU;
  float sc[8], sh[8], sl[8];
  lds_f8(cst + c0, sc); lds_f8(cst + C + c0, sh); lds_f8(cst + 2 * C + c0, sl);
  if (t_begin < t_end) tw.seek(t_begin);
  int it = 0;
  for (int t = t_begin; t < t_end; ++t, ++it, tw.step()) {
    const int st = it % S;
    int l0, n, qs;
    tw.get(l0, n, qs);
    sb_wait(&full[st], (it / S) & 1);
    const uint16_t* sa = reinterpret_cast<const uint16_t*>(stages + (size_t)st * tile_bytes);
    U4 av[SE_U1];
#pragma unroll
    for (int u = 0; u < SE_U1; ++u) {
      const int r = rr + u * RPB;
      if (r < n) av[u] = lds16(sa + r * C + c0);
    }
    __syncwarp();
    if ((tid & 31) == 0) sb_arrive(&empty[st]);
    uint16_t* hb = h + ((int64_t)tw.b * Lh + H) * C + c0;
#pragma unroll
    for (int u = 0; u < SE_U1; ++u) {
      const int r = rr + u * RPB;
      if (r < n) {
        float x[8];
        unpack8(av[u], f16, x);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float y = fmaf(x[j], sc[j], sh[j]);
          if (prelu) y = y > 0.f ? y : sl[j] * y;
          x[j] = y;
        }
        const uint4 o = pack8(x, f16);
        const int q = qs + r;
        *reinterpret_cast<uint4*>(hb + (int64_t)q * C) = o;
        if (H > 0) {
          if ((unsigned)(q - 1) < (unsigned)H) *reinterpret_cast<uint4*>(hb - (int64_t)q * C) = o;
          else if ((unsigned)(L - 2 - q) < (unsigned)H) *reinterpret_cast<uint4*>(hb + (int64_t)(2 * (L - 1) - q) * C) = o;
        }
      }
    }
  }
}

static inline int se_log2(int v) { int l = 0; while ((1 << l) < v) ++l; return l; }
static inline int se_grid(int64_t tiles) {
  const int64_t cap = 2 * (int64_t)NUM_SMS;
  return (int)(tiles < 1 ? 1 : (tiles < cap ? tiles : cap));
}

// shapes the bulk kernels serve: power-of-two C in [64, 1024] (threads own 8 channels; a row is >= 128 bytes)
bool stream_ew_ok(int C) { return C >= 64 && C <= 1024 && (C & (C - 1)) == 0; }

int launch_bn_stats_bulk(const void* a, int dtype, int64_t rows, int C, double* stats, cudaStream_t st) {
  static bool attr = false;
  const int S = 3;
  const int smem = 128 + S * 32768;
  if (!attr) {
    SG_CHECK_CUDA(cudaFuncSetAttribute(bn_stats_bulk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 128 + SE_MAX_STAGES * 32768));
    attr = true;
  }
  const int cgl = se_log2(C / 8);
  const int RT = SE_U1 * (SE_CONSUMERS >> cgl);
  bn_stats_bulk_kernel<<<se_grid(cdiv(rows, RT)), SE_THREADS, smem, st>>>(
      reinterpret_cast<const uint16_t*>(a), dtype == SG_F16, (int)rows, C, cgl, S, stats);
  return SG_OK;
}

int launch_act_fwd_bulk(const void* a, int dtype, int batch, int L, int C, const float* scale_shift, const float* slope,
                        int act, int roll, const int32_t* roll_dev, int H, void* h, cudaStream_t st) {
  static bool attr = false;
  const int S = 3;
  const int cst = (3 * C * 4 + 127) & ~127;
  const int smem = 128 + cst + S * 32768;
  if (!attr) {
    SG_CHECK_CUDA(cudaFuncSetAttribute(act_fwd_bulk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       128 + 12288 + SE_MAX_STAGES * 32768));
    attr = true;
  }
  const int cgl = se_log2(C / 8);
  const int RT = SE_U1 * (SE_CONSUMERS >> cgl);
  const int64_t tiles = (int64_t)batch * (cdiv(L, RT) + 1);
  act_fwd_bulk_kernel<<<se_grid(tiles), SE_THREADS, smem, st>>>(
      reinterpret_cast<const uint16_t*>(a), dtype == SG_F16, batch, L, C, cgl, S, scale_shift, slope, act, roll, roll_dev,
      H, reinterpret_cast<uint16_t*>(h));
  return SG_OK;
}

template <int MODE>
int launch_act_bwd_bulk(const void* g_h, int H, int roll, const int32_t* roll_dev, const void* g_add, const void* a,
                        int dtype, int g_dtype, int batch, int L, int C, const float* scale_shift,
                        const float* mean_invstd, const float* slope, int act, const double* red_in, double* red_out,
                        int use_bn, void* g_a_out, cudaStream_t st) {
  static bool attr = false;
  if (!attr) {
    SG_CHECK_CUDA(cudaFuncSetAttribute(act_bwd_bulk_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       128 + 24576 + SE_MAX_STAGES * 32768));
    attr = true;
  }
  const int ntens = g_add ? 3 : 2;
  const int cst = ((MODE == 1 ? 6 : 3) * C * 4 + 127) & ~127;
  // two CTAs per SM: 113 KB each
  int S = (113 * 1024 - 128 - cst) / (ntens * 16384);
  if (S > SE_MAX_STAGES) S = SE_MAX_STAGES;
  if (S < 2) S = 2;
  const int smem = 128 + cst + S * ntens * 16384;
  SeBwd p;
  p.g_h = reinterpret_cast<const uint16_t*>(g_h); p.g_add = reinterpret_cast<const uint16_t*>(g_add);
  p.a = reinterpret_cast<const uint16_t*>(a); p.g_a_out = reinterpret_cast<uint16_t*>(g_a_out);
  p.scale_shift = scale_shift; p.mean_invstd = mean_invstd; p.slope = slope;
  p.red_in = red_in; p.red_out = red_out; p.roll_dev = roll_dev;
  p.H = H; p.roll = roll; p.batch = batch; p.L = L; p.C = C; p.cgs_log2 = se_log2(C / 8); p.act = act;
  p.use_bn = use_bn; p.a_f16 = dtype == SG_F16; p.g_f16 = g_dtype == SG_F16; p.nstages = S;
  const int RT = SE_U * (SE_CONSUMERS >> p.cgs_log2);
  const int64_t tiles = (int64_t)batch * (cdiv(L, RT) + 1);
  act_bwd_bulk_kernel<MODE><<<se_grid(tiles), SE_THREADS, smem, st>>>(p);
  return SG_OK;
}
template int launch_act_bwd_bulk<0>(const void*, int, int, const int32_t*, const void*, const void*, int, int, int, int,
                                    int, const float*, const float*, const float*, int, const double*, double*, int,
                                    void*, cudaStream_t);
template int launch_act_bwd_bulk<1>(const void*, int, int, const int32_t*, const void*, const void*, int, int, int, int,
                                    int, const float*, const float*, const float*, int, const double*, double*, int,
                                    void*, cudaStream_t);

}  // namespace sg
