// Pooled Discriminator heads (discriminator.py:122-137, 175-190) on the last tower activation h, fp16 NLC
// [B][Lq][C] (no halo, no roll: the last layer has no phase shift after it):
//   conv  a[t] = pool_w . h[t] + pool_b   (Conv1d(C, 1, 1); a is int_act['avg_conv_h'])   y = fc_w . a + fc_b
//   gmax  p[c] = max_t h[t][c]            (AdaptiveMaxPool1d(1); first index of the max, a NaN wins)   y = fc_w . p + fc_b
//   gavg  p[c] = mean_t h[t][c]           (AdaptiveAvgPool1d(1))                                        y = fc_w . p + fc_b
//   mlp   y[t] = pool_w . h[t] + pool_b   (the last Conv1d(C, 1, 1) of the mlp head: one logit per position, no fc)
// One block per batch element.  The forward is deterministic (fixed-order block reductions, no atomics); the
// backward adds the parameter gradients with atomics so that concurrent passes can share one gradient bucket.
#include "common.cuh"

namespace sg {

constexpr int DHEAD_THREADS = 256;

// sum over the block, the same order every run; every thread gets the result
__device__ __forceinline__ float block_sum(float v, float* red /* [DHEAD_THREADS / 32] */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_sum(v);
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int i = 0; i < DHEAD_THREADS / 32; ++i) t += red[i];
  __syncthreads();
  return t;
}

__global__ void __launch_bounds__(DHEAD_THREADS)
dhead_fwd_kernel(int pool_type, const __half* __restrict__ h, int Lq, int C, const float* __restrict__ pool_w,
                 const float* __restrict__ pool_b, const float* __restrict__ fc_w, const float* __restrict__ fc_b,
                 float* __restrict__ pooled, int32_t* __restrict__ argmax, float* __restrict__ logit) {
  extern __shared__ float a_s[];             // conv / mlp: a[Lq]
  __shared__ float red[DHEAD_THREADS / 32];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const __half* hb = h + (int64_t)b * Lq * C;
  float part = 0.f;
  if (pool_type == SG_DHEAD_CONV || pool_type == SG_DHEAD_MLP) {
    // one warp per position, lanes over channel pairs
    const __half2* h2 = reinterpret_cast<const __half2*>(hb);
    const float2* w2 = reinterpret_cast<const float2*>(pool_w);
    for (int t = warp; t < Lq; t += DHEAD_THREADS / 32) {
      float s = 0.f;
      for (int c = lane; c < C / 2; c += 32) {
        const float2 v = __half22float2(h2[(int64_t)t * (C / 2) + c]);
        const float2 w = w2[c];
        s = fmaf(v.x, w.x, s);
        s = fmaf(v.y, w.y, s);
      }
      s = warp_sum(s);
      if (lane == 0) {
        const float a = s + pool_b[0];
        a_s[t] = a;
        if (pool_type == SG_DHEAD_MLP) logit[(int64_t)b * Lq + t] = a;
        else pooled[(int64_t)b * Lq + t] = a;
      }
    }
    if (pool_type == SG_DHEAD_MLP) return;
    __syncthreads();
    for (int t = tid; t < Lq; t += DHEAD_THREADS) part = fmaf(fc_w[t], a_s[t], part);
  } else {
    for (int c = tid; c < C; c += DHEAD_THREADS) {
      float p;
      if (pool_type == SG_DHEAD_GMAX) {
        float m = -INFINITY;
        int idx = 0;
        for (int t = 0; t < Lq; ++t) {
          const float v = __half2float(hb[(int64_t)t * C + c]);
          if (v > m || isnan(v)) { m = v; idx = t; }     // the rule of torch's adaptive max pooling
        }
        argmax[(int64_t)b * C + c] = idx;
        p = m;
      } else {
        float s = 0.f;
        for (int t = 0; t < Lq; ++t) s += __half2float(hb[(int64_t)t * C + c]);
        p = s / (float)Lq;
      }
      pooled[(int64_t)b * C + c] = p;
      part = fmaf(fc_w[c], p, part);
    }
  }
  const float y = block_sum(part, red);
  if (tid == 0) logit[b] = y + fc_b[0];
}

__global__ void __launch_bounds__(DHEAD_THREADS)
dhead_bwd_kernel(int pool_type, const __half* __restrict__ h, int batch, int Lq, int C,
                 const float* __restrict__ pool_w, const float* __restrict__ fc_w, const float* __restrict__ pooled,
                 const int32_t* __restrict__ argmax, const float* __restrict__ logit,
                 const float* __restrict__ g_logit_in, float target, float weight, float* __restrict__ loss_out,
                 void* __restrict__ g_h, int gdt, float* __restrict__ g_pool_w, float* __restrict__ g_pool_b,
                 float* __restrict__ g_fc_w, float* __restrict__ g_fc_b, float gscale) {
  extern __shared__ float ga_s[];            // conv / mlp: d loss / d a[t], loss-scaled
  __shared__ float red[DHEAD_THREADS / 32];
  const int b = blockIdx.x, tid = threadIdx.x;
  const __half* hb = h + (int64_t)b * Lq * C;
  const int64_t gb = (int64_t)b * Lq * C;
  if (pool_type == SG_DHEAD_MLP) {
    // B * Lq logits: the loss is their mean; d logit[t] is d a[t] of the conv branch below
    float part = 0.f, lpart = 0.f;
    const float n = (float)batch * (float)Lq;
    for (int t = tid; t < Lq; t += DHEAD_THREADS) {
      const int64_t i = (int64_t)b * Lq + t;
      const float diff = logit[i] - target;
      const float ga = g_logit_in ? g_logit_in[i] * gscale : 2.f * diff / n * weight * gscale;
      ga_s[t] = ga;
      part += ga;
      lpart += diff * diff / n * weight;
    }
    __syncthreads();
    const float gpb = block_sum(part, red);
    const float lsum = block_sum(lpart, red);
    if (tid == 0) {
      if (g_pool_b) atomicAdd(g_pool_b, gpb);
      if (loss_out) atomicAdd(loss_out, lsum);
    }
  }
  const float diff = pool_type == SG_DHEAD_MLP ? 0.f : logit[b] - target;
  // gscale: loss scale of the 16-bit gradient tensors (every gradient downstream carries it; the loss does not)
  const float gl = pool_type == SG_DHEAD_MLP ? 0.f
                   : g_logit_in ? g_logit_in[b] * gscale : 2.f * diff / (float)batch * weight * gscale;
  if (tid == 0 && pool_type != SG_DHEAD_MLP) {
    if (loss_out) atomicAdd(loss_out, diff * diff / (float)batch * weight);
    if (g_fc_b) atomicAdd(g_fc_b, gl);
  }
  if (pool_type == SG_DHEAD_CONV) {
    float part = 0.f;
    for (int t = tid; t < Lq; t += DHEAD_THREADS) {
      const float ga = gl * fc_w[t];
      ga_s[t] = ga;
      part += ga;
      if (g_fc_w) atomicAdd(g_fc_w + t, gl * pooled[(int64_t)b * Lq + t]);
    }
    __syncthreads();
    const float gpb = block_sum(part, red);
    if (tid == 0 && g_pool_b) atomicAdd(g_pool_b, gpb);
  }
  if (pool_type == SG_DHEAD_CONV || pool_type == SG_DHEAD_MLP) {
    for (int c = tid; c < C; c += DHEAD_THREADS) {
      const float w = pool_w[c];
      float gw = 0.f;
      for (int t = 0; t < Lq; ++t) {
        const float ga = ga_s[t];
        st16(g_h, gb + (int64_t)t * C + c, ga * w, gdt);
        if (g_pool_w) gw = fmaf(ga, __half2float(hb[(int64_t)t * C + c]), gw);
      }
      if (g_pool_w) atomicAdd(g_pool_w + c, gw);
    }
    return;
  }
  for (int c = tid; c < C; c += DHEAD_THREADS) {
    const float gp = gl * fc_w[c];
    if (g_fc_w) atomicAdd(g_fc_w + c, gl * pooled[(int64_t)b * C + c]);
    if (pool_type == SG_DHEAD_GMAX) {
      const int idx = argmax[(int64_t)b * C + c];
      for (int t = 0; t < Lq; ++t) st16(g_h, gb + (int64_t)t * C + c, t == idx ? gp : 0.f, gdt);
    } else {
      const float g = gp / (float)Lq;
      for (int t = 0; t < Lq; ++t) st16(g_h, gb + (int64_t)t * C + c, g, gdt);
    }
  }
}

}  // namespace sg

using namespace sg;
#define ST ((cudaStream_t)stream)

static bool dhead_args_ok(int pool_type, int batch, int Lq, int C) {
  return (pool_type == SG_DHEAD_CONV || pool_type == SG_DHEAD_GMAX || pool_type == SG_DHEAD_GAVG ||
          pool_type == SG_DHEAD_MLP) && batch > 0 &&
         Lq > 0 && Lq <= 4096 && C > 0 && C % 64 == 0;
}

extern "C" int sg_dhead_fwd(int pool_type, const void* h, int batch, int Lq, int C, const float* pool_w,
                            const float* pool_b, const float* fc_w, const float* fc_b, float* pooled, int32_t* argmax,
                            float* logit, void* stream) {
  SG_CHECK_ARG(dhead_args_ok(pool_type, batch, Lq, C));
  const bool mlp = pool_type == SG_DHEAD_MLP;
  SG_CHECK_ARG(h && logit && (mlp || (fc_w && fc_b && pooled)));
  SG_CHECK_ARG((pool_type != SG_DHEAD_CONV && !mlp) || (pool_w && pool_b));
  SG_CHECK_ARG(pool_type != SG_DHEAD_GMAX || argmax);
  const size_t smem = (pool_type == SG_DHEAD_CONV || mlp) ? sizeof(float) * Lq : 0;
  dhead_fwd_kernel<<<batch, DHEAD_THREADS, smem, ST>>>(pool_type, reinterpret_cast<const __half*>(h), Lq, C, pool_w,
                                                       pool_b, fc_w, fc_b, pooled, argmax, logit);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_dhead_bwd(int pool_type, const void* h, int batch, int Lq, int C, const float* pool_w,
                            const float* fc_w, const float* pooled, const int32_t* argmax, const float* logit,
                            const float* g_logit_in, float target, float weight, float* loss_out, void* g_h,
                            float* g_pool_w, float* g_pool_b, float* g_fc_w, float* g_fc_b, float grad_scale,
                            void* stream) {
  SG_CHECK_ARG(dhead_args_ok(pool_type, batch, Lq, C));
  const bool mlp = pool_type == SG_DHEAD_MLP;
  SG_CHECK_ARG(h && logit && g_h && (mlp || (fc_w && pooled)));
  SG_CHECK_ARG((pool_type != SG_DHEAD_CONV && !mlp) || pool_w);
  SG_CHECK_ARG(pool_type != SG_DHEAD_GMAX || argmax);
  const size_t smem = (pool_type == SG_DHEAD_CONV || mlp) ? sizeof(float) * Lq : 0;
  dhead_bwd_kernel<<<batch, DHEAD_THREADS, smem, ST>>>(
      pool_type, reinterpret_cast<const __half*>(h), batch, Lq, C, pool_w, fc_w, pooled, argmax, logit, g_logit_in,
      target, weight, loss_out, g_h, g_grad_dtype, g_pool_w, g_pool_b, g_fc_w, g_fc_b, grad_scale);
  SG_CHECK_LAUNCH();
  return SG_OK;
}
