// C-ABI plumbing: error slot, device probe, tap-GEMM argument validation + back-end dispatch.
#include "common.cuh"
#include <string.h>

namespace sg {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
int tapgemm_f_ffma_launch(const sg_tapgemm_f* q, cudaStream_t st);
int tapgemm_w_ffma_launch(const sg_tapgemm_w* q, cudaStream_t st);
int tapgemm_f_tc_launch(const sg_tapgemm_f* q, cudaStream_t st);
int tapgemm_w_tc_launch(const sg_tapgemm_w* q, cudaStream_t st);
int64_t tapgemm_f_workspace_bytes();
int tapgemm_f_debug_timeline(unsigned long long* host_out, int max_words);
extern int g_cta_pair;
extern int g_stream_k;
extern double g_sk_atomic_steps;
extern double g_sk_fixed_steps;
int g_grad_dtype = SG_F16;
}  // namespace sg

using namespace sg;

extern "C" int sg_abi_version(void) { return SG_ABI_VERSION; }
extern "C" const char* sg_last_error(void) { return g_err; }

extern "C" int sg_set_cta_pair(int on) {
  const int prev = g_cta_pair;
  g_cta_pair = on < 0 ? 0 : (on > 2 ? 2 : on);
  return prev;
}

extern "C" int sg_set_stream_k(int max_split, float atomic_steps) {
  const int prev = g_stream_k;
  if (max_split >= 0) g_stream_k = max_split;
  if (atomic_steps > 0.f) {
    g_sk_atomic_steps = atomic_steps;
    g_sk_fixed_steps = atomic_steps < 1e-3f ? 0.0 : 60.0;      // a vanishing constant forces the split (sweeps, tests)
  }
  return prev;
}

extern "C" int sg_set_grad_dtype(int dtype) {
  const int prev = g_grad_dtype;
  if (dtype == SG_F16 || dtype == SG_BF16) g_grad_dtype = dtype;
  return prev;
}

extern "C" int sg_device_ok(void) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  int major = 0, minor = 0;
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return 0;
  if (cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev) != cudaSuccess) return 0;
  return (major == 9 && minor == 0) ? 1 : 0;      // sm_90a code loads on compute capability 9.0 only
}

static int check_taps(const int32_t* k_lo, const int32_t* k_hi, const int32_t* n_lo, const int32_t* n_hi, int d_lo,
                      int d_hi, int kc, int nc) {
  for (int d = d_lo; d <= d_hi; ++d) {
    const int i = d + 4;
    if (k_lo[i] < 0 || k_hi[i] > kc || k_lo[i] % 64 || k_hi[i] % 64 || k_lo[i] >= k_hi[i]) return 0;
    if (n_lo[i] < 0 || n_hi[i] > nc || n_lo[i] % 64 || n_hi[i] % 64 || n_lo[i] >= n_hi[i]) return 0;
  }
  return 1;
}

extern "C" int64_t sg_tapgemm_f_workspace_bytes(void) { return tapgemm_f_workspace_bytes(); }
extern "C" int sg_debug_timeline(unsigned long long* host_out, int max_words) {
  return tapgemm_f_debug_timeline(host_out, max_words);
}

extern "C" int sg_tapgemm_f_run(const sg_tapgemm_f* p, void* stream) {
  SG_CHECK_ARG(p != nullptr);
  SG_CHECK_ARG(p->a0 && p->w && p->out);
  SG_CHECK_ARG(p->a0_c > 0 && p->a0_c % 64 == 0 && p->a1_c % 64 == 0 && p->kc == p->a0_c + p->a1_c);
  SG_CHECK_ARG((p->a1 != nullptr) == (p->a1_c > 0));
  SG_CHECK_ARG(p->nc % 64 == 0 && p->n_lo % 64 == 0 && p->n_hi % 64 == 0 && p->n_lo >= 0 && p->n_hi <= p->nc &&
               p->n_lo < p->n_hi);
  SG_CHECK_ARG(p->d_lo >= -4 && p->d_hi <= 4 && p->d_lo <= p->d_hi);
  SG_CHECK_ARG(check_taps(p->tap_k_lo, p->tap_k_hi, p->tap_n_lo, p->tap_n_hi, p->d_lo, p->d_hi, p->kc, p->nc));
  SG_CHECK_ARG(p->a_dtype == SG_F16 || p->a_dtype == SG_BF16);
  SG_CHECK_ARG(p->w_dtype == SG_F16 || p->w_dtype == SG_BF16);
  SG_CHECK_ARG(p->out_dtype == SG_F16 || p->out_dtype == SG_BF16 || p->out_dtype == SG_F32);
  SG_CHECK_ARG(p->ksplit <= 1 || p->out_dtype == SG_F32);
  SG_CHECK_ARG(p->m_lo >= -p->out_halo && p->m_hi <= p->out_rows + p->out_halo && p->m_lo < p->m_hi);
  SG_CHECK_ARG(p->batch > 0 && p->a_rows > 0 && p->a_halo >= 0);
  {
    // the launch's columns stay inside one row of `out`; column pairs are stored together (half2 / float2 / red.v2)
    const int ld = p->out_ld > 0 ? p->out_ld : p->nc, col0 = p->out_ld > 0 ? p->out_col0 : p->n_lo;
    const uintptr_t pair = p->out_dtype == SG_F32 ? 8 : 4;
    SG_CHECK_ARG(col0 >= 0 && col0 + (p->n_hi - p->n_lo) <= ld);
    SG_CHECK_ARG(ld % 2 == 0 && col0 % 2 == 0 && reinterpret_cast<uintptr_t>(p->out) % pair == 0);
    SG_CHECK_ARG(p->out2 == nullptr || reinterpret_cast<uintptr_t>(p->out2) % pair == 0);
  }
  // bias pairs are read without a wrap inside the pair
  SG_CHECK_ARG(p->bias == nullptr || p->bias_mod <= 0 || p->bias_mod % 64 == 0);
  if (p->out2 != nullptr || p->slope != nullptr) {
    SG_CHECK_ARG(p->slope != nullptr && p->slope_mod > 0 && p->slope_mod % 64 == 0 && p->out_dtype != SG_F32);
    SG_CHECK_ARG(p->ksplit <= 1 && p->out2_halo >= 0);
    SG_CHECK_ARG(p->out2_halo == 0 || (p->m_lo == 0 && p->m_hi == p->out_rows && p->out_rows >= 2 * p->out2_halo + 3));
  }
  if (p->backend == SG_BACKEND_TCGEN05) {
    SG_CHECK_ARG(p->a_dtype == p->w_dtype);
    return tapgemm_f_tc_launch(p, (cudaStream_t)stream);
  }
  if (p->backend == SG_BACKEND_FFMA) {
    if (p->bn_stats != nullptr || p->out2 != nullptr || p->slope != nullptr) {
      set_error("bn_stats / out2 (fused epilogues) need the tensor-core backend");
      return SG_ERR_UNSUPPORTED;
    }
    return tapgemm_f_ffma_launch(p, (cudaStream_t)stream);
  }
  set_error("unknown backend %d", p->backend);
  return SG_ERR_UNSUPPORTED;
}

extern "C" int sg_tapgemm_w_run(const sg_tapgemm_w* p, void* stream) {
  SG_CHECK_ARG(p != nullptr);
  SG_CHECK_ARG(p->g && p->a0 && p->dw);
  SG_CHECK_ARG(p->a0_c > 0 && p->a0_c % 64 == 0 && p->a1_c % 64 == 0 && p->kc == p->a0_c + p->a1_c);
  SG_CHECK_ARG((p->a1 != nullptr) == (p->a1_c > 0));
  SG_CHECK_ARG(p->nc % 128 == 0);
  SG_CHECK_ARG(p->d_lo >= -4 && p->d_hi <= 4 && p->d_lo <= p->d_hi);
  SG_CHECK_ARG(check_taps(p->tap_k_lo, p->tap_k_hi, p->tap_n_lo, p->tap_n_hi, p->d_lo, p->d_hi, p->kc, p->nc));
  SG_CHECK_ARG(p->g_dtype == SG_F16 || p->g_dtype == SG_BF16);
  SG_CHECK_ARG(p->a_dtype == SG_F16 || p->a_dtype == SG_BF16);
  SG_CHECK_ARG(p->batch > 0 && p->g_rows > 0 && (p->g_rows >= 64 ? p->g_rows % 64 == 0 : 64 % p->g_rows == 0));
  if (p->backend == SG_BACKEND_TCGEN05) {
    // wgmma takes A and B in one 16-bit format
    SG_CHECK_ARG(p->g_dtype == p->a_dtype);
    return tapgemm_w_tc_launch(p, (cudaStream_t)stream);
  }
  if (p->backend == SG_BACKEND_FFMA) return tapgemm_w_ffma_launch(p, (cudaStream_t)stream);
  set_error("unknown backend %d", p->backend);
  return SG_ERR_UNSUPPORTED;
}
