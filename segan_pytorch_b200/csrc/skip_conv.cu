// GSkip with skip_type='conv' (generator.py:43-49): nn.Conv1d(C, C, K, stride 1, padding K//2) on the encoder's
// pre-activation.  Read as the grouped rows [B][L/4][4C] (g = 4, include/segan_b200.h "HBM layout") the conv is a
// form-F tap-GEMM with kc = nc = 4C and taps d = -D..D, D = (K//2 + 3) / 4:
//     W'[d][(po, co)][(pi, ci)] = W[co][ci][t],   t = 4d + pi - po + K//2   (0 if t is outside [0, K))
// so every weight tap appears four times (once per output phase po).  The fp32 master stays in reference layout
// [C][C][K]; these kernels emit the redundant 16-bit operands and fold the GEMM's weight gradient back.
#include "common.cuh"

namespace sg {

__device__ __forceinline__ void st_out(void* p, int64_t i, float v, int dtype) {
  if (dtype == SG_F32) reinterpret_cast<float*>(p)[i] = v;
  else st16(p, i, v, dtype);
}

// weight tap of block (d, po, pi), or -1 when the block is structurally zero
__device__ __forceinline__ int skipconv_tap(int d, int po, int pi, int K) {
  const int t = 4 * d + pi - po + K / 2;
  return (t >= 0 && t < K) ? t : -1;
}

// One block = one 64 x 64 (n, k) tile of one tap slot s = d + D.  C % 64 == 0, so a tile has one (po, pi) phase pair.
//   forward operand        F [s][(po, co)][(pi, ci)] = W'[d]
//   data-gradient operand  Dg[2D - s][(pi, ci)][(po, co)] = W'[d]   (per-tap transpose, tap d <-> -d)
__global__ void __launch_bounds__(256)
skipconv_emit_kernel(const float* __restrict__ w, int C, int K, int D, void* __restrict__ f, void* __restrict__ dg,
                     int dt_f, int dt_dg) {
  __shared__ float tile[64][65];
  const int s = blockIdx.z, d = s - D;
  const int nc = 4 * C;
  const int n0 = blockIdx.y * 64, k0 = blockIdx.x * 64;
  const int po = n0 / C, co0 = n0 % C, pi = k0 / C, ci0 = k0 % C;
  const int t = skipconv_tap(d, po, pi, K);
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;      // 64 x 4
  const int64_t fbase = ((int64_t)s * nc + n0) * nc + k0;
#pragma unroll 4
  for (int r = ty; r < 64; r += 4) {
    const float v = t >= 0 ? w[((int64_t)(co0 + r) * C + ci0 + tx) * K + t] : 0.f;
    tile[r][tx] = v;
    if (f) st_out(f, fbase + (int64_t)r * nc + tx, v, dt_f);
  }
  if (!dg) return;
  __syncthreads();
  const int64_t dbase = ((int64_t)(2 * D - s) * nc + k0) * nc + n0;
#pragma unroll 4
  for (int r = ty; r < 64; r += 4) st_out(dg, dbase + (int64_t)r * nc + tx, tile[tx][r], dt_dg);
}

// dW[co][ci][t] += sum over the four output phases po of dW'[d][(po, co)][(pi, ci)] with 4d + pi - po + K//2 = t.
// One block = 4 output channels co x 64 input channels ci (threadIdx.x = ci lane: coalesced workspace reads).  The
// K tap sums of a (co, ci) pair are staged in shared memory ([co][ci][t] order, conflict-free for odd K), so that
// the block's rows of dw -- 64 K contiguous floats per co -- are read-modified-written coalesced.  Every workspace
// element the weight-gradient GEMM can have written -- the four copies and the structurally zero blocks inside the
// tap table's rectangles -- is zeroed again, so the workspace needs no fill before the next accumulation.  Plain
// (ordered) accumulation into dw: the caller serialises the launches that write one gradient slot.
constexpr int FOLD_CO = 4, FOLD_CI = 64, FOLD_KMAX = 33;
__global__ void __launch_bounds__(FOLD_CO * FOLD_CI)
skipconv_wgrad_fold_kernel(float* __restrict__ dwq, int C, int K, int D, float* __restrict__ dw) {
  // sized for the widest kernel: a K-sized dynamic allocation lets more blocks share an SM, which was measured slower
  // (0.57 against 0.27 ms for C = 512, K = 11 at batch 300 on an H100)
  __shared__ float acc[FOLD_CO * FOLD_CI * FOLD_KMAX];
  // per tap slot: po_lo, po_hi, pi_lo, pi_hi (inclusive) -- the bounding box of the tap's non-zero blocks, i.e. the
  // rectangle the tap table of the tap-GEMMs covers (engine.skipconv_geometry computes the same)
  __shared__ int box[9][4];
  const int tx = threadIdx.x % FOLD_CI, ty = threadIdx.x / FOLD_CI;
  const int ci0 = blockIdx.x * FOLD_CI, co0 = blockIdx.y * FOLD_CO;
  const int co = co0 + ty, ci = ci0 + tx;
  const int nc = 4 * C, P = K / 2;
  if (threadIdx.x <= 2 * D) {
    int po_lo = 4, po_hi = -1, pi_lo = 4, pi_hi = -1;
    for (int a = 0; a < 4; ++a)
      for (int b = 0; b < 4; ++b)
        if (skipconv_tap(threadIdx.x - D, a, b, K) >= 0) {
          po_lo = min(po_lo, a); po_hi = max(po_hi, a);
          pi_lo = min(pi_lo, b); pi_hi = max(pi_hi, b);
        }
    box[threadIdx.x][0] = po_lo; box[threadIdx.x][1] = po_hi;
    box[threadIdx.x][2] = pi_lo; box[threadIdx.x][3] = pi_hi;
  }
  auto at = [&](int d, int po, int pi) -> float* {
    return dwq + ((int64_t)(d + D) * nc + po * C + co) * nc + pi * C + ci;
  };
  for (int t = 0; t < K; ++t) {
    float v = 0.f;
#pragma unroll
    for (int po = 0; po < 4; ++po) {
      const int u = t - P + po;                 // = 4d + pi
      const int pi = u & 3, d = (u - pi) / 4;   // floor division (u may be negative)
      float* p = at(d, po, pi);
      v += *p;
      *p = 0.f;
    }
    acc[(ty * FOLD_CI + tx) * K + t] = v;
  }
  __syncthreads();
  float* row = dw + ((int64_t)co * C + ci0) * K;   // FOLD_CI * K contiguous floats of channel co
  for (int j = tx; j < FOLD_CI * K; j += FOLD_CI) row[j] += acc[ty * FOLD_CI * K + j];
  for (int s = 0; s <= 2 * D; ++s)
    for (int po = box[s][0]; po <= box[s][1]; ++po)
      for (int pi = box[s][2]; pi <= box[s][3]; ++pi)
        if (skipconv_tap(s - D, po, pi, K) < 0) *at(s - D, po, pi) = 0.f;
}

}  // namespace sg

using namespace sg;
#define ST ((cudaStream_t)stream)

static bool skipconv_shape_ok(int C, int K) { return C > 0 && C % 64 == 0 && K >= 1 && K <= 33 && K % 2 == 1; }
static bool skipconv_dtype_ok(int dt) { return dt == SG_F16 || dt == SG_BF16 || dt == SG_F32; }

extern "C" int sg_skipconv_emit(const float* w, int C, int K, void* w_fwd, void* w_dgrad, int dtype_fwd,
                                int dtype_dgrad, void* stream) {
  SG_CHECK_ARG(w && (w_fwd || w_dgrad) && skipconv_shape_ok(C, K));
  SG_CHECK_ARG((!w_fwd || skipconv_dtype_ok(dtype_fwd)) && (!w_dgrad || skipconv_dtype_ok(dtype_dgrad)));
  const int D = (K / 2 + 3) / 4;
  dim3 grid(4 * C / 64, 4 * C / 64, 2 * D + 1);
  skipconv_emit_kernel<<<grid, 256, 0, ST>>>(w, C, K, D, w_fwd, w_dgrad, dtype_fwd, dtype_dgrad);
  SG_CHECK_LAUNCH();
  return SG_OK;
}

extern "C" int sg_skipconv_wgrad_fold(float* dwq, int C, int K, float* dw, void* stream) {
  SG_CHECK_ARG(dwq && dw && skipconv_shape_ok(C, K));
  const int D = (K / 2 + 3) / 4;
  dim3 grid(C / FOLD_CI, C / FOLD_CO);
  skipconv_wgrad_fold_kernel<<<grid, FOLD_CO * FOLD_CI, 0, ST>>>(dwq, C, K, D, dw);
  SG_CHECK_LAUNCH();
  return SG_OK;
}
