// TMA / mbarrier / wgmma implementation of the two tap-GEMM forms (SG_BACKEND_TCGEN05), sm_90a.
//
// Both kernels are persistent (at most one CTA per SM, static round-robin tile schedule) and warp
// specialised by warpgroup -- warpgroup 0: TMA producer (one thread issues, the others give their
// registers back with setmaxnreg), warpgroups 1 and 2: consumers, each owning 64 of the tile's 128 M rows
// with its fp32 accumulator in registers (wgmma m64nNk16, N = the tile's width).  A shared-memory ring
// (full / empty mbarriers, 4 stages; form F sizes them to the tile width, see FSmem) keeps the producer ahead of the
// consumers, so the loads of tile i+1 overlap the epilogue of tile i.  Form F stages whole 16-bit output tiles in
// shared memory and writes them with TMA stores that drain during the next tile's MMAs (f_epilogue_tma); the
// other epilogues store from the fragment.
//
// Every operand tile is a TMA box of 64 channels (128 B) x rows, 128B-swizzled, so the same
// shared-memory bytes serve as
//   * a K-major  wgmma operand (rows = M/N, 64 channels = K)   -> form F (fwd / dgrad)
//   * an MN-major wgmma operand (64 channels = M/N, rows = K)  -> form W (wgrad)
// i.e. no im2col, no transposed copies in HBM: the 9 row-taps are just 9 different TMA
// coordinates into the same NLC-row tensor.
#include "common.cuh"
#include <cuda.h>
#include <stdlib.h>

namespace sg {

// ------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try(uint32_t addr, uint32_t parity) {
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
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  if (mbar_try(addr, parity)) return;
  // slow path.  watchdog: a pipeline bug must surface as a launch error, never as a hung GPU
  long long t0 = 0;
  uint32_t spins = 0;
  while (!mbar_try(addr, parity)) {
    if ((++spins & 1023u) == 0) {
      const long long now = clock64();
      if (t0 == 0) t0 = now;
      else if (now - t0 > 8000000000LL) __trap();
    }
  }
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
// TMA tensor store shared -> global (bulk async-group of the issuing thread); the box is clipped at the map's edges
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, uint32_t src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(src), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// every bulk store this thread issued has finished READING shared memory (the global writes may still be in flight)
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// ... all but the N most recently committed bulk groups of this thread
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
// this thread's generic-proxy shared-memory writes become visible to the async proxy (TMA)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void st_shared_u32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ uint4 ld_shared_v4(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
  return v;
}
// 8-byte vector reduction (sm_90+): one RED for two fp32 adds
__device__ __forceinline__ void red_add_v2(float* addr, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
// the 256 consumer threads of a CTA (named barrier 1; the producer warpgroup never joins it)
__device__ __forceinline__ void consumer_bar_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// wgmma m64nNk16, fp32 accumulators in registers, both operands from shared memory through descriptors.
// TA / TB: 0 = K-major operand, 1 = MN-major (transposed) operand.  scale_d = 0 starts a new accumulation.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_f16_n64(float (&d)[32], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_n64(float (&d)[32], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_f16_n128(float (&d)[64], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_n128(float (&d)[64], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_f16_n256(float (&d)[128], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, %131, %132;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_n256(float (&d)[128], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, %131, %132;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}

template <int N, int TA, int TB, bool BF16>
__device__ __forceinline__ void wgmma_tile(float (&d)[N / 2], uint64_t da, uint64_t db, int scale_d) {
  if constexpr (N == 64) {
    if constexpr (BF16) wgmma_bf16_n64<TA, TB>(d, da, db, scale_d);
    else wgmma_f16_n64<TA, TB>(d, da, db, scale_d);
  } else if constexpr (N == 128) {
    if constexpr (BF16) wgmma_bf16_n128<TA, TB>(d, da, db, scale_d);
    else wgmma_f16_n128<TA, TB>(d, da, db, scale_d);
  } else {
    static_assert(N == 256, "wgmma tile width");
    if constexpr (BF16) wgmma_bf16_n256<TA, TB>(d, da, db, scale_d);
    else wgmma_f16_n256<TA, TB>(d, da, db, scale_d);
  }
}

// ------------------------------------------------------------------------------------------
// descriptors
// ------------------------------------------------------------------------------------------
// shared-memory matrix descriptor (sm_90 wgmma), 128B swizzle.
//   K-major : rows of 128 B (64 x 16-bit along K); 8-row groups SBO bytes apart; LBO unused.
//   MN-major: 128 B lines hold 64 MN-elements for one K index; 8 K-lines form a 1024 B group,
//             groups SBO bytes apart; 64-element MN blocks LBO bytes apart.
// Stage bases are 1024 B aligned, so the base-offset field stays 0; a K step inside the swizzle atom
// advances the start address only.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;                           // SWIZZLE_128B
  return d;
}

// One 64-deep K block (one ring stage) as four k16 wgmmas.  a_step / b_step: descriptor advance per k16 in
// 16-byte units (K-major: 32 B along the row; MN-major: 16 lines of 128 B).
template <int N, int TA, int TB, bool BF16>
__device__ __forceinline__ void mma_k64(float (&acc)[N / 2], uint64_t da, uint64_t db, uint32_t a_step,
                                        uint32_t b_step, bool first) {
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < 4; ++kk)
    wgmma_tile<N, TA, TB, BF16>(acc, da + kk * a_step, db + kk * b_step, (first && kk == 0) ? 0 : 1);
  wgmma_commit();
}

constexpr int STAGES = 4;
constexpr int A_STAGE_BYTES = 128 * 128;   // 128 rows x 128 B
constexpr int B_STAGE_BYTES = 256 * 128;   // up to 256 rows x 128 B
constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/ + 2048 /*column statistics*/;
constexpr int SMEM_OPTIN_LIMIT = 232448;   // sm_90 per-block opt-in maximum
// Form F, per tile width TN: a ring of stages sized to the tile (16 KB of A + TN x 128 B of weights), then the output
// staging area of 16 KB chunks (each one 128-row x 64-column 16-bit chunk of a tile, 1024 B aligned for the 128B
// swizzle; the BatchNorm column statistics alias it, their launches store from the fragment), then the barriers.
//   TN  64: 4 x 24 KB ring, two 32 KB buffers used by alternate tiles, each a whole tile with out2: the single-tap
//           launches are store-bound, so a tile's staging must not wait for the previous tile's stores
//   TN 128: 4 x 32 KB ring, one 64 KB buffer: a whole tile with out2
//   TN 256: 4 x 48 KB ring, one 32 KB buffer: the tile leaves in rounds of two chunks.  Nothing larger fits next to
//           four stages, and a 3-stage ring lengthens the main loop of the 256-wide layers by more than whole-tile
//           staging saves
constexpr int OUT_CHUNK_BYTES = 128 * 128;
template <int TN>
struct FSmem {
  static constexpr int RING = 4;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + TN * 128;
  static constexpr int BUFS = TN == 64 ? 2 : 1;                   // staging buffers, used by alternate tiles
  static constexpr int BUF_BYTES = (TN == 256 ? 2 : 4) * OUT_CHUNK_BYTES / BUFS;
  static constexpr int STG_OFF = RING * STAGE_BYTES;
  static constexpr int CTL_OFF = STG_OFF + BUFS * BUF_BYTES;
  static constexpr int BYTES = CTL_OFF + 256 /*barriers*/ + 1024 /*align*/;
  static_assert(RING <= STAGES && STAGE_BYTES % 1024 == 0 && BUFS * BUF_BYTES >= 2048, "form-F shared memory");
};
static_assert(FSmem<64>::BYTES <= SMEM_OPTIN_LIMIT, "form-F TN 64 shared memory exceeds the sm_90 opt-in limit");
static_assert(FSmem<128>::BYTES <= SMEM_OPTIN_LIMIT, "form-F TN 128 shared memory exceeds the sm_90 opt-in limit");
static_assert(FSmem<256>::BYTES <= SMEM_OPTIN_LIMIT, "form-F TN 256 shared memory exceeds the sm_90 opt-in limit");
constexpr int NUM_THREADS = 384;           // producer warpgroup + two consumer warpgroups
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;

struct TapRangesTC {
  int k_lo[NTAP], k_hi[NTAP], n_lo[NTAP], n_hi[NTAP];
};

struct FTcParams {
  int a0_c, kc, nc, a_halo;
  int d_lo, d_hi;
  TapRangesTC tr;
  void* out; int out_dtype, out_rows, out_halo, out_ld, out_col0;
  int w_tap0;
  int m_lo, m_hi, n_lo;
  const float* bias; int bias_mod;
  int batch, ksplit;
  int TR, TB, TN;            // segment 0's M tile = TB batches x TR rows (<= 128), N tile
  int m_tiles_per_b, n_tiles;
  int m_tiles0, m_tiles;     // M tiles of segment 0 (m_tiles_per_b x its batch tiles), of both segments
  int m_lo1, TR1, TB1;       // segment 1 (rows [m_lo1, m_hi), TR1 < 128 of them, TB1 batches per tile), TR1 = 0: none
  int dbg;                   // SEGAN_B200_DEBUG (bit 20: phase timeline)
  double* stats;             // fused BatchNorm statistics [SG_STAT_SLICES][2][nc], or nullptr
  int sk_dp_tiles;           // tiles [0, sk_dp_tiles) are tile-strided; each of the rest is split along K over
  int sk_split;              // sk_split CTAs
  float* sk_ws;              // stream-K partial sums [ctas][128 x 256] fp32
  unsigned int* sk_cnt;      // k-step counters [leftover tiles][8 consumer warps] (zero between launches)
  void* out2;                // fused PReLU output (16-bit, out's dtype and column geometry), or nullptr
  int out2_halo;             // reflect halo rows of out2 (its buffer has out_rows + 2 * out2_halo rows per batch element)
  const float* slope; int slope_mod;
  int bias_mask, slope_mask; // mod - 1 when the modulus is a power of two (the channel counts are), else -1
  int tma_out;               // whole tiles leave through shared memory and TMA stores (16-bit out, no BatchNorm stats)
};

// tapgemm_f_tc's parameters: eight tensor maps and FTcParams, inside the classic 4 KB kernel-parameter space
static_assert(8 * sizeof(CUtensorMap) + sizeof(FTcParams) <= 4096, "tapgemm_f_tc parameter block exceeds 4 KB");

struct SharedCtl {
  uint64_t full[STAGES];
  uint64_t empty[STAGES];
};

// number of 64-channel K steps a tile with N range [n0, n0+TN) executes for interleaved K split `ks`
__device__ __forceinline__ int f_num_steps(const FTcParams& p, int n0, int ks) {
  int total = 0;
  for (int d = p.d_lo; d <= p.d_hi; ++d) {
    const int ti = d + 4;
    if (n0 + p.TN <= p.tr.n_lo[ti] || n0 >= p.tr.n_hi[ti]) continue;
    total += (p.tr.k_hi[ti] - p.tr.k_lo[ti]) >> 6;
  }
  return p.ksplit == 1 ? total : (total - ks + p.ksplit - 1) / p.ksplit;
}

// ---- work decomposition of tapgemm_f_tc -------------------------------------------------------------
// Tiles [0, sk_dp_tiles) are scheduled tile-strided over the CTAs.  With batch 300 many layers have a tile count
// just above a multiple of the CTA count, so the last wave ran a few tiles on an otherwise idle GPU.  Each leftover
// tile [sk_dp_tiles, total) is therefore split along K over sk_split CTAs (CTA c takes k-range c % sk_split of
// leftover tile c / sk_split): every one of them stores its fp32 partial sums into its own workspace slot and bumps
// the tile's counter; the warp whose bump completes the count adds the slots up in slot order (deterministic),
// applies bias / conversion, stores, and leaves the counter zeroed for the next launch.  No CTA ever waits for
// another one.  The split factor is chosen by the host: the partial sums cost L2 traffic in proportion to sk_split,
// the tail shrinks as 1 / sk_split (tapgemm_f_tc_launch).
struct Piece {
  int tile;      // tile index (mt fastest, then ksplit, then nt)
  int mt, rest;  // tile % m_tiles, tile / m_tiles (tracked incrementally: no division per tile)
  int kb, ke;    // k-step range [kb, ke) of the tile's `total` steps (split-K pieces; whole tile otherwise)
  int total;
};

// SEGAN_B200_DEBUG bit 20: phase timeline of tapgemm_f_tc (globaltimer ns; first consumer thread of every CTA):
// [cta][0] = kernel start, then per piece: accumulator ready, epilogue done (TMA-stored tiles: stores issued),
// (split tiles) finisher done; last = exit.
// Read back with sg_debug_timeline (diagnostics only).
constexpr int TL_SLOTS = 32;
constexpr int TL_CTAS = 160;
__device__ unsigned long long g_tc_timeline[TL_CTAS * TL_SLOTS];
__device__ __forceinline__ unsigned long long gtime_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

struct PieceIter {
  int m_tiles, nctas, dp_end, total_tiles, cta;
  int next_dp, cur_mt, cur_rest;
  int cache_rest, cache_steps;
  bool sk_done;

  __device__ __forceinline__ int steps_of_rest(const FTcParams& p, int rest) {
    if (rest != cache_rest) {
      cache_rest = rest;
      cache_steps = p.ksplit == 1 ? f_num_steps(p, p.n_lo + rest * p.TN, 0)
                                  : f_num_steps(p, p.n_lo + (rest / p.ksplit) * p.TN, rest % p.ksplit);
    }
    return cache_steps;
  }
  __device__ __forceinline__ void init(const FTcParams& p, int m_tiles_, int total_tiles_, int cta_, int nctas_) {
    m_tiles = m_tiles_; nctas = nctas_; total_tiles = total_tiles_; cta = cta_;
    dp_end = p.sk_dp_tiles < total_tiles_ ? p.sk_dp_tiles : total_tiles_;
    next_dp = cta_;
    cur_rest = cta_ / m_tiles_;
    cur_mt = cta_ - cur_rest * m_tiles_;
    cache_rest = -1; cache_steps = 0;
    sk_done = false;
  }
  __device__ __forceinline__ bool next(const FTcParams& p, Piece& pc) {
    if (next_dp < dp_end) {
      pc.tile = next_dp; pc.mt = cur_mt; pc.rest = cur_rest;
      pc.kb = 0; pc.total = pc.ke = steps_of_rest(p, cur_rest);
      next_dp += nctas;
      cur_mt += nctas;
      while (cur_mt >= m_tiles) { cur_mt -= m_tiles; ++cur_rest; }
      return true;
    }
    if (sk_done || dp_end >= total_tiles) return false;
    sk_done = true;
    const int t = dp_end + cta / p.sk_split;
    if (t >= total_tiles) return false;
    const int part = cta % p.sk_split;
    pc.tile = t; pc.rest = t / m_tiles; pc.mt = t - pc.rest * m_tiles;
    const int s = steps_of_rest(p, pc.rest);
    pc.total = s;
    pc.kb = (int)((long long)s * part / p.sk_split);
    pc.ke = (int)((long long)s * (part + 1) / p.sk_split);
    // an empty piece (a tile with fewer k-steps than sk_split: its N range misses some taps) still runs: it stores a
    // zero partial and counts, otherwise the tile is never finished and its counter is left non-zero
    return true;
  }
};

// Rows of M tile mt.  A launch's rows [m_lo, m_hi) are one or two segments, each packed into M tiles of TB batch
// elements x TR rows (tapgemm_f_tc_launch).  Segment 0's tiles come first (row tile fastest, then batch tile);
// segment 1, the last TR1 rows of every batch element, follows with one tile per TB1 batch elements.  The tile covers
// batch elements [b0, b0 + TB) x rows [m0, m0 + TR); m_rel is m0 relative to the first row of its segment's store map.
struct FTile {
  int b0, m0, m_rel, TR, TB, seg;
};
__device__ __forceinline__ FTile f_tile(const FTcParams& p, int mt) {
  FTile t;
  if (mt < p.m_tiles0) {
    const int mtb = p.m_tiles_per_b == 1 ? mt : mt / p.m_tiles_per_b;
    t.b0 = mtb * p.TB;
    t.m_rel = (mt - mtb * p.m_tiles_per_b) * p.TR;
    t.m0 = p.m_lo + t.m_rel;
    t.TR = p.TR; t.TB = p.TB; t.seg = 0;
  } else {
    t.b0 = (mt - p.m_tiles0) * p.TB1;
    t.m_rel = 0;
    t.m0 = p.m_lo1;
    t.TR = p.TR1; t.TB = p.TB1; t.seg = 1;
  }
  return t;
}

__device__ __forceinline__ int f_mod(int x, int mod, int mask) { return mask >= 0 ? (x & mask) : (x % mod); }

__device__ __forceinline__ uint32_t pack2(float x, float y, int dtype) {
  if (dtype == SG_F16) return pack_half2_sat(x, y);
  __nv_bfloat162 h = __floats2bfloat162_rn(x, y);
  return *reinterpret_cast<uint32_t*>(&h);
}

// Two adjacent columns (n_abs, n_abs + 1) of one output row: conversion / stores, and the fused second output
//   out2[b][row2][n] = PReLU(v) (16-bit), the consumer-ready activation of the Generator's conv / deconv blocks
//   (modules.py:99-101,139-141: no norm layer between the contraction and the PReLU), written next to the raw
//   pre-activation (`out`, the skip connection's source, generator.py:185,191) with its reflect halo
//   (modules.py:92-98): position m also lands on its mirror row when it lies within `out2_halo` of an end.
// x / y return the values stored into `out` (the BatchNorm statistics describe them).
__device__ __forceinline__ void f_store2(const FTcParams& p, float& x, float& y, int64_t o, int n_abs, bool atomic,
                                         int64_t o2, int64_t o2mirror) {
  if (p.out_dtype == SG_F32) {
    float* dst = reinterpret_cast<float*>(p.out) + o;
    if (atomic) red_add_v2(dst, x, y);
    else *reinterpret_cast<float2*>(dst) = make_float2(x, y);
    return;
  }
  float s0 = 0.f, s1 = 0.f;
  if (p.slope != nullptr) {
    const float* sp = p.slope + f_mod(n_abs, p.slope_mod, p.slope_mask);    // slope_mod is even: no wrap inside the pair
    s0 = __ldg(sp); s1 = __ldg(sp + 1);
    if (p.out2 == nullptr) {   // PReLU applied to the (only) output: blocks whose pre-activation nobody reads
      x = x > 0.f ? x : s0 * x;
      y = y > 0.f ? y : s1 * y;
    }
  }
  *reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(p.out) + o) = pack2(x, y, p.out_dtype);
  if (p.out2 != nullptr) {
    const uint32_t a = pack2(x > 0.f ? x : s0 * x, y > 0.f ? y : s1 * y, p.out_dtype);
    *reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(p.out2) + o2) = a;
    if (o2mirror >= 0) *reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(p.out2) + o2mirror) = a;
  }
}

__device__ __forceinline__ float round_as_stored(float x, int dtype) {
  if (dtype == SG_F16) return __half2float(__float2half_rn(x));
  if (dtype == SG_BF16) return __bfloat162float(__float2bfloat16_rn(x));
  return x;
}

// Epilogue of one consumer thread: wgmma accumulator fragment -> bias / conversion / stores (+ BatchNorm column
// statistics into shared memory).  Fragment layout of m64nN: consumer warp cw (0..7) owns tile rows 16 cw + lane/4
// and 16 cw + 8 + lane/4; register 4j + 2h + e holds column 8j + 2(lane%4) + e of the h-th of those rows.
template <int TN>
__device__ __forceinline__ void f_epilogue(const FTcParams& p, float (&acc)[TN / 2], const FTile& t, int n0, int ks,
                                           int ctid, float* colstat) {
  const int lane = ctid & 31, cw = ctid >> 5;
  const int out_buf_rows = p.out_rows + 2 * p.out_halo;
  const int out2_buf_rows = p.out_rows + 2 * p.out2_halo;
  const int col0 = n0 - p.n_lo + p.out_col0 + 2 * (lane & 3);
  int64_t obase[2], o2base[2], o2mirror[2];
  bool valid[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = cw * 16 + (lane >> 2) + 8 * h;
    const int tb = r / t.TR, tr = r - tb * t.TR;
    const int b = t.b0 + tb, m = t.m0 + tr;
    valid[h] = (tb < t.TB) && (b < p.batch) && (m < p.m_hi);
    obase[h] = ((int64_t)b * out_buf_rows + (m + p.out_halo)) * p.out_ld + col0;
    o2base[h] = 0; o2mirror[h] = -1;
    if (p.out2 != nullptr) {
      const int64_t rb = (int64_t)b * out2_buf_rows + p.out2_halo;
      o2base[h] = (rb + m) * p.out_ld + col0;
      if (p.out2_halo > 0) {
        int mm = 0;
        bool has = false;
        if (m >= 1 && m <= p.out2_halo) { mm = -m; has = true; }
        else if (m >= p.out_rows - 1 - p.out2_halo && m <= p.out_rows - 2) { mm = 2 * (p.out_rows - 1) - m; has = true; }
        if (has) o2mirror[h] = (rb + mm) * p.out_ld + col0;
      }
    }
  }
  const bool add_bias = p.bias != nullptr && ks == 0;
  const bool atomic = p.ksplit > 1;
#pragma unroll
  for (int j = 0; j < TN / 8; ++j) {
    const int c = 8 * j + 2 * (lane & 3);
    float bx = 0.f, by = 0.f;
    if (add_bias) {    // bias_mod is a multiple of 64: no wrap inside the pair
      const float* bp = p.bias + f_mod(n0 + c, p.bias_mod, p.bias_mask);
      bx = __ldg(bp); by = __ldg(bp + 1);
    }
    float sx = 0.f, sy = 0.f, qx = 0.f, qy = 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float x = acc[4 * j + 2 * h] + bx, y = acc[4 * j + 2 * h + 1] + by;
      if (valid[h]) {
        f_store2(p, x, y, obase[h] + 8 * j, n0 + c, atomic, o2base[h] + 8 * j, o2mirror[h] >= 0 ? o2mirror[h] + 8 * j : -1);
        x = round_as_stored(x, p.out_dtype);
        y = round_as_stored(y, p.out_dtype);
        sx += x; sy += y; qx += x * x; qy += y * y;
      }
    }
    if (p.stats != nullptr) {            // uniform branch: the reduction is warp-collective
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) {
        sx += __shfl_xor_sync(0xffffffffu, sx, o);
        sy += __shfl_xor_sync(0xffffffffu, sy, o);
        qx += __shfl_xor_sync(0xffffffffu, qx, o);
        qy += __shfl_xor_sync(0xffffffffu, qy, o);
      }
      if (lane < 4) {
        atomicAdd(colstat + c, sx);
        atomicAdd(colstat + c + 1, sy);
        atomicAdd(colstat + 256 + c, qx);
        atomicAdd(colstat + 256 + c + 1, qy);
      }
    }
  }
}

// Epilogue of a whole tile with a 16-bit `out` (every forward and data-gradient launch but fc.0 and BatchNorm-stat
// launches), all 256 consumer threads together.  The consumers write the tile into a staging buffer `buf` in
// 64-column chunks of 16 KB (rows in fragment order tb * TR + tr = the box's row order, 128B-swizzled so that the 8
// rows of one warp store hit different banks), then one thread issues a TMA tensor store per chunk, box {64, TR, TB}
// clipped at the launch's columns, rows and batch elements, and commits them as one bulk group.  The consumers go
// straight back to the MMAs while the stores drain; a buffer is rewritten only after the issuing thread has seen the
// bulk group that last read it finish reading (FSmem: with two buffers that is the group before the last one).  At
// TN 256 the buffer holds two chunks, so the tile leaves in rounds with such a wait between them (two chunks of
// `out`, or a chunk of `out` and the same chunk of `out2`).
// Per element the arithmetic is f_store2's: fp32 accumulator + bias, PReLU from fp32, one rounding.  The
// reflect-halo mirror rows of out2 (rows reversed: no box expresses them) are copied from the staged chunks with
// 16-byte stores.
// The body is fully unrolled over the tile's TN / 4 column pairs per thread, so everything that is uniform over the
// tile stays out of it: the output format F16 and MODE (0: out; 1: PReLU applied to out; 2: out and the PReLU
// output out2) are template parameters chosen once per tile, and the bias / slope column of each 64-column chunk is
// reduced modulo bias_mod / slope_mod once (both are multiples of 64, as is n0: a chunk never wraps), so a pair's
// parameters are two loads at fixed offsets.
template <bool F16>
__device__ __forceinline__ uint32_t pack2_t(float x, float y) {
  if constexpr (F16) return pack_half2_sat(x, y);
  __nv_bfloat162 h = __floats2bfloat162_rn(x, y);
  return *reinterpret_cast<uint32_t*>(&h);
}

template <int TN, bool F16, int MODE>
__device__ __forceinline__ void f_epilogue_tma_body(const FTcParams& p, const float (&acc)[TN / 2], const FTile& t,
                                                    int n0, int ctid, uint32_t buf, const CUtensorMap* tmO,
                                                    const CUtensorMap* tmO2) {
  constexpr bool two = MODE == 2;
  constexpr bool act_in_place = MODE == 1;
  const int lane = ctid & 31, cw = ctid >> 5;
  const int b0 = t.b0, m0 = t.m0;
  const bool add_bias = p.bias != nullptr;
  // this thread's 4-byte word of row cw * 16 + lane / 4 (+ 8 for h = 1, 1024 B further) in a staged chunk; the
  // row's 16-byte column block jj sits at block jj ^ (row & 7) = jj ^ (lane / 4)
  const uint32_t row_off = (uint32_t)(cw * 16 + (lane >> 2)) * 128u + 4u * (lane & 3);
  const int sw = lane >> 2;
  const int halo2 = p.out2_halo;
  const bool mirror_tile = two && halo2 > 0 &&
                           ((m0 <= halo2 && m0 + t.TR > 1) || (m0 + t.TR > p.out_rows - 1 - halo2 && m0 <= p.out_rows - 2));
  constexpr int NQ = TN / 64;
  // A round stages as many 64-column chunks as the buffer holds (CH slots; with out2 each chunk of out takes two
  // slots, out's and out2's), issues their stores and commits them as one bulk group.
  constexpr int CH = FSmem<TN>::BUF_BYTES / OUT_CHUNK_BYTES;
  constexpr int QPR = two ? CH / 2 : CH;          // chunks per round
  const int c_rel = n0 - p.n_lo, m_rel = t.m_rel;
#pragma unroll
  for (int q = 0; q < NQ; ++q) {
    const int qi = q % QPR;                       // position in the round
    const uint32_t slot = buf + (uint32_t)(two ? 2 * qi : qi) * OUT_CHUNK_BYTES;
    if (qi == 0) {
      if (ctid == 0) {                            // the stores that last read this buffer are done reading ...
        if (q == 0) bulk_wait_read<FSmem<TN>::BUFS - 1>();
        else bulk_wait_read<0>();
      }
      consumer_bar_sync();                        // ... before anyone writes it again
    }
    // this thread's first column of the chunk: n0 + 64 q + 2 (lane % 4); column pair jj is 8 jj further
    const int cq0 = n0 + 64 * q;
    const float* bq = p.bias + f_mod(cq0, p.bias_mod, p.bias_mask) + 2 * (lane & 3);
    const float* sq = p.slope + (MODE != 0 ? f_mod(cq0, p.slope_mod, p.slope_mask) + 2 * (lane & 3) : 0);
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const int j = 8 * q + jj;
      float bx = 0.f, by = 0.f;
      if (add_bias) { bx = __ldg(bq + 8 * jj); by = __ldg(bq + 8 * jj + 1); }
      float s0 = 0.f, s1 = 0.f;
      if constexpr (MODE != 0) { s0 = __ldg(sq + 8 * jj); s1 = __ldg(sq + 8 * jj + 1); }
      const uint32_t col_off = (uint32_t)((jj ^ sw) << 4);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float x = acc[4 * j + 2 * h] + bx, y = acc[4 * j + 2 * h + 1] + by;
        if constexpr (act_in_place) {
          x = x > 0.f ? x : s0 * x;
          y = y > 0.f ? y : s1 * y;
        }
        const uint32_t off = row_off + (uint32_t)h * 1024u + col_off;
        st_shared_u32(slot + off, pack2_t<F16>(x, y));
        if constexpr (two) st_shared_u32(slot + OUT_CHUNK_BYTES + off, pack2_t<F16>(x > 0.f ? x : s0 * x, y > 0.f ? y : s1 * y));
      }
    }
    if (qi != QPR - 1 && q != NQ - 1) continue;
    fence_proxy_async_smem();
    consumer_bar_sync();
    if (ctid == 0) {
#pragma unroll
      for (int k = 0; k <= qi; ++k) {
        const uint32_t src = buf + (uint32_t)(two ? 2 * k : k) * OUT_CHUNK_BYTES;
        const int cq = c_rel + 64 * (q - qi + k);
        tma_store_3d(tmO, src, cq, m_rel, b0);
        if constexpr (two) tma_store_3d(tmO2, src + OUT_CHUNK_BYTES, cq, m_rel, b0);
      }
      bulk_commit();
    }
    if (mirror_tile) {
      // out2 rows m in [1, halo] also land on row -m, rows m in [out_rows-1-halo, out_rows-2] on 2(out_rows-1)-m
      const int rows = t.TR * t.TB;
      const int out2_buf_rows = p.out_rows + 2 * halo2;
      for (int idx = ctid; idx < rows * 8 * (qi + 1); idx += 256) {
        const int k = idx / (rows * 8), rk = idx - k * rows * 8;
        const int r = rk >> 3, kb = rk & 7;
        const int tb = r / t.TR, tr = r - tb * t.TR;
        const int b = b0 + tb, m = m0 + tr;
        if (b >= p.batch || m >= p.m_hi) continue;
        int mm;
        if (m >= 1 && m <= halo2) mm = -m;
        else if (m >= p.out_rows - 1 - halo2 && m <= p.out_rows - 2) mm = 2 * (p.out_rows - 1) - m;
        else continue;
        const uint32_t src = buf + (uint32_t)(2 * k + 1) * OUT_CHUNK_BYTES;
        const uint4 v = ld_shared_v4(src + (uint32_t)r * 128u + (uint32_t)((kb ^ (r & 7)) << 4));
        const int64_t o = ((int64_t)b * out2_buf_rows + halo2 + mm) * p.out_ld + p.out_col0 + c_rel +
                          64 * (q - qi + k) + 8 * kb;
        *reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(p.out2) + o) = v;
      }
    }
  }
}

template <int TN>
__device__ __forceinline__ void f_epilogue_tma(const FTcParams& p, const float (&acc)[TN / 2], const FTile& t, int n0,
                                               int ctid, uint32_t buf, const CUtensorMap* tmO,
                                               const CUtensorMap* tmO2) {
  const int mode = p.out2 != nullptr ? 2 : (p.slope != nullptr ? 1 : 0);
  if (p.out_dtype == SG_F16) {
    if (mode == 2) f_epilogue_tma_body<TN, true, 2>(p, acc, t, n0, ctid, buf, tmO, tmO2);
    else if (mode == 1) f_epilogue_tma_body<TN, true, 1>(p, acc, t, n0, ctid, buf, tmO, tmO2);
    else f_epilogue_tma_body<TN, true, 0>(p, acc, t, n0, ctid, buf, tmO, tmO2);
  } else {
    if (mode == 2) f_epilogue_tma_body<TN, false, 2>(p, acc, t, n0, ctid, buf, tmO, tmO2);
    else if (mode == 1) f_epilogue_tma_body<TN, false, 1>(p, acc, t, n0, ctid, buf, tmO, tmO2);
    else f_epilogue_tma_body<TN, false, 0>(p, acc, t, n0, ctid, buf, tmO, tmO2);
  }
}

// ------------------------------------------------------------------------------------------
// form F:  out[b,m,n] = bias + sum_d sum_kc A[b,m+d,kc] * Wp[d+4][n][kc]
//   wgmma: M = 128 (rows: TB batches x TR rows; 64 per consumer warpgroup), N = TN output channels,
//   K = 64-channel blocks.  Optional: interleaved K split into fp32 (ksplit > 1, vector red), stream-K tail,
//   fused BatchNorm statistics, fused PReLU / second output.
// ------------------------------------------------------------------------------------------
// BF16: operand format (bf16 / fp16), a template parameter so that each wgmma has one fixed form.
// tmA0 / tmA1 / tmO: the A source and `out` maps of row segment 0 (boxes {64, TR, TB}); tmA0s1 / tmA1s1 / tmOs1:
// those of segment 1 (boxes {64, TR1, TB1}; copies of segment 0's when TR1 = 0).  out2 launches never split.
template <int TN, bool BF16>
__global__ void __launch_bounds__(NUM_THREADS, 1)
tapgemm_f_tc(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
             const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmO,
             const __grid_constant__ CUtensorMap tmO2, const __grid_constant__ CUtensorMap tmA0s1,
             const __grid_constant__ CUtensorMap tmA1s1, const __grid_constant__ CUtensorMap tmOs1,
             const FTcParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  using L = FSmem<TN>;
  SharedCtl* ctl = reinterpret_cast<SharedCtl*>(smem + L::CTL_OFF);
  float* colstat = reinterpret_cast<float*>(smem + L::STG_OFF);      // [2][256], aliases the output staging
  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA0); prefetch_tmap(&tmA1); prefetch_tmap(&tmW);
    if (p.tma_out) {
      prefetch_tmap(&tmO);
      if (p.out2 != nullptr) prefetch_tmap(&tmO2);
    }
    if (p.TR1 > 0) {
      prefetch_tmap(&tmA0s1); prefetch_tmap(&tmA1s1);
      if (p.tma_out) prefetch_tmap(&tmOs1);
    }
    for (int s = 0; s < L::RING; ++s) { mbar_init(&ctl->full[s], 1); mbar_init(&ctl->empty[s], 2); }
    fence_barrier_init();
  }
  if (p.stats != nullptr)
    for (int c = threadIdx.x; c < 512; c += NUM_THREADS) colstat[c] = 0.f;
  __syncthreads();

  const int total_tiles = p.m_tiles * p.n_tiles * p.ksplit;
  const uint32_t b_bytes = (uint32_t)TN * 128u;
  PieceIter it;
  it.init(p, p.m_tiles, total_tiles, blockIdx.x, gridDim.x);
  Piece pc;

  if (wg == 0) {
    // ================= TMA producer =================
    setmaxnreg_dec<PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      int stage = 0; uint32_t phase = 0;
      while (it.next(p, pc)) {
        const int ks = p.ksplit == 1 ? 0 : pc.rest % p.ksplit;
        const int nt = p.ksplit == 1 ? pc.rest : pc.rest / p.ksplit;
        const FTile t = f_tile(p, pc.mt);
        const int b0 = t.b0, m0 = t.m0;
        const CUtensorMap* mA0 = t.seg ? &tmA0s1 : &tmA0;
        const CUtensorMap* mA1 = t.seg ? &tmA1s1 : &tmA1;
        const uint32_t a_bytes = (uint32_t)t.TR * t.TB * 128u;     // the whole box: rows past the batch are zero-filled
        const int n0 = p.n_lo + nt * p.TN;
        // k-steps [kb, ke) of the tile's (tap, k-block) sequence; a split-K piece jumps to its first step.  An
        // interleaved k-split tile (ksplit > 1: the fc.0 GEMM, K = 16384) takes every ksplit-th (tap, k-block)
        // starting at block ks.
        const bool interleaved = p.ksplit > 1;
        int step = 0, sel = 0;              // step: first (tap, k-block) index of the current tap; sel: steps passed
        int skip = interleaved ? 0 : pc.kb;
        int next_sel = ks;                  // interleaved: global index of the next block this tile takes
        const int kstride = interleaved ? 64 * p.ksplit : 64;
        for (int d = p.d_lo; d <= p.d_hi; ++d) {
          const int ti = d + 4;
          if (n0 + p.TN <= p.tr.n_lo[ti] || n0 >= p.tr.n_hi[ti]) continue;
          const int klo = p.tr.k_lo[ti], khi = p.tr.k_hi[ti];
          const int nk = (khi - klo) >> 6;
          int k0 = klo;
          if (!interleaved) {
            if (skip >= nk) { skip -= nk; sel += nk; continue; }
            k0 += skip << 6; sel += skip; skip = 0;
            if (sel >= pc.ke) break;
          } else {
            if (next_sel >= step + nk) { step += nk; continue; }
            k0 += (next_sel - step) << 6;
          }
          for (; k0 < khi; k0 += kstride) {
            if (!interleaved) {
              if (sel++ >= pc.ke) break;
            } else {
              next_sel += p.ksplit;
            }
            mbar_wait(&ctl->empty[stage], phase ^ 1);
            uint8_t* sa = smem + stage * L::STAGE_BYTES;
            mbar_expect_tx(&ctl->full[stage], a_bytes + b_bytes);
            if (k0 < p.a0_c) tma_load_3d(sa, mA0, &ctl->full[stage], k0, m0 + d + p.a_halo, b0);
            else tma_load_3d(sa, mA1, &ctl->full[stage], k0 - p.a0_c, m0 + d + p.a_halo, b0);
            tma_load_2d(sa + A_STAGE_BYTES, &tmW, &ctl->full[stage], k0, (ti - p.w_tap0) * p.nc + n0);
            if (++stage == L::RING) { stage = 0; phase ^= 1; }
          }
          step += nk;
        }
      }
    }
    return;
  }

  // ================= consumers (warpgroups 1, 2): MMA + epilogue =================
  setmaxnreg_inc<CONSUMER_REGS>();
  const int ctid = threadIdx.x - 128;              // 0..255
  const int cwg = wg - 1;                          // rows [64 cwg, 64 cwg + 64) of the tile
  const bool wg_leader = (threadIdx.x & 127) == 0;
  const uint32_t smem0 = smem_u32(smem);
  int stage = 0; uint32_t phase = 0;
  int stat_nt = -1;
  auto flush_stats = [&](int nt_done) {
    consumer_bar_sync();
    const int n0s = p.n_lo + nt_done * p.TN;
    double* o = p.stats + (int64_t)(blockIdx.x % SG_STAT_SLICES) * 2 * p.nc;
    for (int c = ctid; c < p.TN; c += 256) {
      atomicAdd(o + n0s + c, (double)colstat[c]);
      atomicAdd(o + p.nc + n0s + c, (double)colstat[256 + c]);
      colstat[c] = 0.f;
      colstat[256 + c] = 0.f;
    }
    consumer_bar_sync();
  };
  const bool tl_on = (p.dbg & (1 << 20)) && ctid == 0 && blockIdx.x < TL_CTAS;
  int tl_i = 0;
  unsigned long long* tl = g_tc_timeline + (blockIdx.x < TL_CTAS ? blockIdx.x : 0) * TL_SLOTS;
  if (tl_on) { for (int i = 0; i < TL_SLOTS; ++i) tl[i] = 0; tl[tl_i++] = gtime_ns(); }

  int staged = 0;                                  // tiles this CTA has staged (selects the staging buffer)
  float acc[TN / 2];
  while (it.next(p, pc)) {
    const int ks = p.ksplit == 1 ? 0 : pc.rest % p.ksplit;
    const int nt = p.ksplit == 1 ? pc.rest : pc.rest / p.ksplit;
    const int n0 = p.n_lo + nt * p.TN;
    const bool partial = pc.tile >= it.dp_end;                     // one K range (possibly empty) of a split tile
    if (p.stats != nullptr && nt != stat_nt) {
      if (stat_nt >= 0) flush_stats(stat_nt);
      stat_nt = nt;
    }
    const int nsteps = pc.ke - pc.kb;
    if (nsteps == 0) {
#pragma unroll
      for (int j = 0; j < TN / 2; ++j) acc[j] = 0.f;
    }
    int prev = 0;
    for (int i = 0; i < nsteps; ++i) {
      mbar_wait(&ctl->full[stage], phase);
      const uint32_t sa = smem0 + (uint32_t)stage * L::STAGE_BYTES;
      mma_k64<TN, 0, 0, BF16>(acc, make_smem_desc(sa + (uint32_t)cwg * 8192u, 16, 1024),
                        make_smem_desc(sa + A_STAGE_BYTES, 16, 1024), 2, 2, i == 0);
      wgmma_wait<1>();                               // the MMAs of step i-1 have retired: free their stage
      if (i > 0 && wg_leader) mbar_arrive(&ctl->empty[prev]);
      prev = stage;
      if (++stage == L::RING) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    if (nsteps > 0 && wg_leader) mbar_arrive(&ctl->empty[prev]);
    if (tl_on && tl_i < TL_SLOTS - 1) tl[tl_i++] = gtime_ns();

    if (!partial) {
      if (p.tma_out) {
        const uint32_t buf = smem0 + L::STG_OFF + (uint32_t)(staged++ % L::BUFS) * L::BUF_BYTES;
        const FTile t = f_tile(p, pc.mt);
        f_epilogue_tma<TN>(p, acc, t, n0, ctid, buf, t.seg ? &tmOs1 : &tmO, &tmO2);
      } else f_epilogue<TN>(p, acc, f_tile(p, pc.mt), n0, ks, ctid, colstat);
      if (tl_on && tl_i < TL_SLOTS - 1) tl[tl_i++] = gtime_ns();
      continue;
    }
    // split tile: this CTA's fp32 partial sums go to ITS workspace slot (plain stores, fragment order: only the same
    // consumer thread of another CTA ever reads a value back); the warp that counts the tile's last contribution
    // adds the sk_split slots up in slot order (deterministic) and finishes the tile.
    constexpr int64_t SLOT_F2 = 128 * 256 / 2;
    float2* myslot = reinterpret_cast<float2*>(p.sk_ws) + (int64_t)blockIdx.x * SLOT_F2 + ctid;
#pragma unroll
    for (int j = 0; j < TN / 4; ++j) __stcg(myslot + j * 256, make_float2(acc[2 * j], acc[2 * j + 1]));
    if (tl_on && tl_i < TL_SLOTS - 1) tl[tl_i++] = gtime_ns();
    const int slot = pc.tile - it.dp_end;
    unsigned int* cnt = p.sk_cnt + slot * 8 + (ctid >> 5);
    __threadfence();                               // this warp's partial sums are visible ...
    __syncwarp();
    unsigned int old = 0;
    if ((ctid & 31) == 0) old = atomicAdd(cnt, 1u);    // ... before its contribution is counted
    old = __shfl_sync(0xffffffffu, old, 0);
    if (old + 1u == (unsigned int)p.sk_split) {
      __threadfence();
#pragma unroll
      for (int j = 0; j < TN / 2; ++j) acc[j] = 0.f;
      const float2* base0 = reinterpret_cast<const float2*>(p.sk_ws) + (int64_t)slot * p.sk_split * SLOT_F2 + ctid;
      for (int sp = 0; sp < p.sk_split; ++sp) {
#pragma unroll
        for (int j = 0; j < TN / 4; ++j) {
          const float2 t = __ldcg(base0 + sp * SLOT_F2 + j * 256);
          acc[2 * j] += t.x; acc[2 * j + 1] += t.y;
        }
      }
      f_epilogue<TN>(p, acc, f_tile(p, pc.mt), n0, 0, ctid, colstat);
      __syncwarp();
      if ((ctid & 31) == 0) *cnt = 0u;             // ready for the next launch
      if (tl_on && tl_i < TL_SLOTS - 1) tl[tl_i++] = gtime_ns() | (1ull << 63);      // flagged: finisher
    }
  }
  if (tl_on && tl_i < TL_SLOTS) tl[tl_i++] = gtime_ns();
  if (p.stats != nullptr && stat_nt >= 0) flush_stats(stat_nt);
  if (p.tma_out && ctid == 0) bulk_wait_read_all();   // shared memory outlives the last stores' reads
}

// ------------------------------------------------------------------------------------------
// form W:  dWp[d+4][n][kc] += sum_{b,m} G[b,m,n] * A[b,m+d,kc]
//   wgmma: M = 128 channels n (MN-major from G; 64 per consumer warpgroup), N = TK channels kc (MN-major
//   from A), K = 64 positions per stage (PB batches x PR rows).
// ------------------------------------------------------------------------------------------
struct WTcParams {
  int a0_c, kc, nc, a_halo;
  int d_lo, d_hi;
  TapRangesTC tr;
  float* dw; int dw_tap0;
  int g_rows, batch, ksplit;
  int PR, PB;                // K block = PB batches x PR rows = 64 positions
  int n_tiles, k_tiles;      // nc/128, kc/TK
  int row_chunks, b_chunks;  // ceil(g_rows/PR), ceil(batch/PB)
  const float* out_scale;    // device scalar applied to the products before the atomic accumulation, or nullptr
};

template <int TK, bool BF16>
__global__ void __launch_bounds__(NUM_THREADS, 1)
tapgemm_w_tc(const __grid_constant__ CUtensorMap tmG, const __grid_constant__ CUtensorMap tmA0,
             const __grid_constant__ CUtensorMap tmA1, const WTcParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  SharedCtl* ctl = reinterpret_cast<SharedCtl*>(smem + STAGES * STAGE_BYTES);
  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmG); prefetch_tmap(&tmA0); prefetch_tmap(&tmA1);
    for (int s = 0; s < STAGES; ++s) { mbar_init(&ctl->full[s], 1); mbar_init(&ctl->empty[s], 2); }
    fence_barrier_init();
  }
  __syncthreads();

  const int ntaps = p.d_hi - p.d_lo + 1;
  const int total_tiles = ntaps * p.n_tiles * p.k_tiles * p.ksplit;
  const int pos_steps = p.row_chunks * p.b_chunks;
  const int steps_per_split = (pos_steps + p.ksplit - 1) / p.ksplit;
  constexpr int KBOXES = TK / 64;
  constexpr uint32_t STAGE_TX = (uint32_t)(2 + KBOXES) * 64u * 128u;

  // tile -> (d, n0, kc0, split); returns false when the (tap, n, kc) block is structurally zero
  auto decode = [&](int tile, int& d, int& n0, int& kc0, int& sp) -> bool {
    // taps fastest: the CTAs that run at the same time work on the SAME position range with
    // different taps / channel tiles, so G and the (row-shifted) A rows are shared through L2
    // instead of being streamed from HBM once per tap
    d = p.d_lo + tile % ntaps; tile /= ntaps;
    const int kt = tile % p.k_tiles; tile /= p.k_tiles;
    const int nt = tile % p.n_tiles; tile /= p.n_tiles;
    sp = tile;
    n0 = nt * 128; kc0 = kt * TK;
    const int ti = d + 4;
    if (n0 + 128 <= p.tr.n_lo[ti] || n0 >= p.tr.n_hi[ti]) return false;
    if (kc0 + TK <= p.tr.k_lo[ti] || kc0 >= p.tr.k_hi[ti]) return false;
    return true;
  };

  if (wg == 0) {
    // ================= TMA producer: two 64-channel G boxes + TK/64 A boxes per stage =================
    setmaxnreg_dec<PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        int d, n0, kc0, sp;
        if (!decode(tile, d, n0, kc0, sp)) continue;
        const int s_lo = sp * steps_per_split;
        const int s_hi = min(pos_steps, s_lo + steps_per_split);
        int rc = s_lo % p.row_chunks, bc = s_lo / p.row_chunks;
        for (int s = s_lo; s < s_hi; ++s) {
          mbar_wait(&ctl->empty[stage], phase ^ 1);
          uint8_t* st = smem + stage * STAGE_BYTES;
          mbar_expect_tx(&ctl->full[stage], STAGE_TX);
          const int r = rc * p.PR, b = bc * p.PB;
#pragma unroll
          for (int j = 0; j < 2; ++j) tma_load_3d(st + 8192 * j, &tmG, &ctl->full[stage], n0 + 64 * j, r, b);
#pragma unroll
          for (int j = 0; j < KBOXES; ++j) {     // a kc tile may straddle the two sources: every box picks its map
            const int kk = kc0 + 64 * j;
            if (kk < p.a0_c) tma_load_3d(st + 2 * 8192 + 8192 * j, &tmA0, &ctl->full[stage], kk, r + d + p.a_halo, b);
            else tma_load_3d(st + 2 * 8192 + 8192 * j, &tmA1, &ctl->full[stage], kk - p.a0_c, r + d + p.a_halo, b);
          }
          if (++rc == p.row_chunks) { rc = 0; ++bc; }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ================= consumers: warpgroup cwg owns gradient channels [n0 + 64 cwg, n0 + 64 cwg + 64) =========
  setmaxnreg_inc<CONSUMER_REGS>();
  const int ctid = threadIdx.x - 128;
  const int cwg = wg - 1;
  const int lane = ctid & 31, cw = (ctid >> 5) & 3;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  const uint32_t smem0 = smem_u32(smem);
  const float osc = p.out_scale ? __ldg(p.out_scale) : 1.f;
  int stage = 0; uint32_t phase = 0;
  float acc[TK / 2];
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    int d, n0, kc0, sp;
    if (!decode(tile, d, n0, kc0, sp)) continue;
    const int s_lo = sp * steps_per_split;
    const int s_hi = min(pos_steps, s_lo + steps_per_split);
    if (s_lo >= s_hi) continue;
    int prev = 0;
    for (int s = s_lo; s < s_hi; ++s) {
      mbar_wait(&ctl->full[stage], phase);
      const uint32_t st = smem0 + (uint32_t)stage * STAGE_BYTES;
      // 16 positions = 16 lines of 128 B = 2048 B along K: +128 in descriptor address units
      mma_k64<TK, 1, 1, BF16>(acc, make_smem_desc(st + (uint32_t)cwg * 8192u, 8192, 1024),
                        make_smem_desc(st + 2 * 8192, 8192, 1024), 128, 128, s == s_lo);
      wgmma_wait<1>();
      if (s > s_lo && wg_leader) mbar_arrive(&ctl->empty[prev]);
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    if (wg_leader) mbar_arrive(&ctl->empty[prev]);

    const int ti = d + 4;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int n = n0 + 64 * cwg + cw * 16 + (lane >> 2) + 8 * h;      // this row's gradient channel
      if (n < p.tr.n_lo[ti] || n >= p.tr.n_hi[ti]) continue;
      float* o = p.dw + ((int64_t)(ti - p.dw_tap0) * p.nc + n) * p.kc + kc0 + 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < TK / 8; ++j) {
        // column blocks that are structurally zero for this tap are not written
        if (kc0 + 8 * j + 8 <= p.tr.k_lo[ti] || kc0 + 8 * j >= p.tr.k_hi[ti]) continue;
        red_add_v2(o + 8 * j, osc * acc[4 * j + 2 * h], osc * acc[4 * j + 2 * h + 1]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// host side: tensor maps + launch
// ------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* ptr = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess)
    return nullptr;
  fn = reinterpret_cast<EncodeTiledFn>(ptr);
  return fn;
}

// 3-D map over [B][rows][C] 16-bit, box (64, box_rows, box_b), 128B swizzle, OOB -> 0
static int make_map3(CUtensorMap* m, const void* base, int dtype, int C, int rows, int B, int box_rows, int box_b) {
  EncodeTiledFn enc = get_encode();
  if (!enc) { set_error("cuTensorMapEncodeTiled unavailable"); return SG_ERR_LAUNCH; }
  cuuint64_t dims[3] = {(cuuint64_t)C, (cuuint64_t)rows, (cuuint64_t)B};
  cuuint64_t strides[2] = {(cuuint64_t)C * 2, (cuuint64_t)C * 2 * (cuuint64_t)rows};
  cuuint32_t box[3] = {64, (cuuint32_t)box_rows, (cuuint32_t)box_b};
  cuuint32_t es[3] = {1, 1, 1};
  CUresult r = enc(m, dtype == SG_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3,
                   const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(3d C=%d rows=%d B=%d box=%d,%d) failed: %d", C, rows, B, box_rows, box_b, (int)r);
    return SG_ERR_LAUNCH;
  }
  return SG_OK;
}
static int make_map2(CUtensorMap* m, const void* base, int dtype, int C, int64_t rows, int box_rows) {
  EncodeTiledFn enc = get_encode();
  if (!enc) { set_error("cuTensorMapEncodeTiled unavailable"); return SG_ERR_LAUNCH; }
  cuuint64_t dims[2] = {(cuuint64_t)C, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)C * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
  cuuint32_t es[2] = {1, 1};
  CUresult r = enc(m, dtype == SG_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2,
                   const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(2d C=%d rows=%lld box=%d) failed: %d", C, (long long)rows, box_rows, (int)r);
    return SG_ERR_LAUNCH;
  }
  return SG_OK;
}

// 3-D store map over the columns [col0, col0 + C) and rows [row0, row0 + rows) of every batch element of a 16-bit
// [B][buf_rows][ld] tensor, box (64, box_rows, box_b), 128B swizzle.  TMA needs 16-byte aligned bases and strides.
static int make_store_map3(CUtensorMap* m, void* base, int dtype, int C, int rows, int B, int ld, int buf_rows,
                           int row0, int col0, int box_rows, int box_b) {
  EncodeTiledFn enc = get_encode();
  if (!enc) { set_error("cuTensorMapEncodeTiled unavailable"); return SG_ERR_LAUNCH; }
  uint8_t* p0 = reinterpret_cast<uint8_t*>(base) + ((int64_t)row0 * ld + col0) * 2;
  SG_CHECK_ARG(ld % 8 == 0 && col0 % 8 == 0 && (reinterpret_cast<uintptr_t>(p0) & 15) == 0);
  cuuint64_t dims[3] = {(cuuint64_t)C, (cuuint64_t)rows, (cuuint64_t)B};
  cuuint64_t strides[2] = {(cuuint64_t)ld * 2, (cuuint64_t)ld * 2 * (cuuint64_t)buf_rows};
  cuuint32_t box[3] = {64, (cuuint32_t)box_rows, (cuuint32_t)box_b};
  cuuint32_t es[3] = {1, 1, 1};
  CUresult r = enc(m, dtype == SG_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, p0, dims,
                   strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(store C=%d rows=%d B=%d ld=%d box=%d,%d) failed: %d", C, rows, B, ld, box_rows,
              box_b, (int)r);
    return SG_ERR_LAUNCH;
  }
  return SG_OK;
}

// split-K workspace: counters [leftover tiles][8 consumer warps] u32 (8 KB), then one partial-sum slot per CTA
// [SK_MAX_CTAS][128][256] fp32
constexpr int SK_MAX_CTAS = 160;
constexpr int64_t SK_CNT_BYTES = 8192;
constexpr int64_t SK_WS_BYTES = SK_CNT_BYTES + (int64_t)SK_MAX_CTAS * 128 * 256 * 4;
int64_t tapgemm_f_workspace_bytes() { return SK_WS_BYTES; }
int tapgemm_f_debug_timeline(unsigned long long* host_out, int max_words) {
  const int n = max_words < TL_CTAS * TL_SLOTS ? max_words : TL_CTAS * TL_SLOTS;
  if (cudaMemcpyFromSymbol(host_out, g_tc_timeline, (size_t)n * sizeof(unsigned long long)) != cudaSuccess) return -1;
  return n;
}
// SEGAN_B200_STREAMK: 0 = off, n = largest split factor per leftover tile (default 16);
// SEGAN_B200_SK_ATOMIC / SEGAN_B200_SK_FIXED: cost-model constants in k-steps (tapgemm_f_tc_launch)
int g_stream_k = [] { const char* e = getenv("SEGAN_B200_STREAMK"); return e ? atoi(e) : 16; }();
double g_sk_atomic_steps = [] { const char* e = getenv("SEGAN_B200_SK_ATOMIC"); return e ? atof(e) : 4.5; }();
double g_sk_fixed_steps = [] { const char* e = getenv("SEGAN_B200_SK_FIXED"); return e ? atof(e) : 60.0; }();

// sg_set_cta_pair(): recorded for the C ABI; every setting runs the one sm_90a forward-form kernel
int g_cta_pair = 1;

static int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = NUM_SMS;
  }
  return n;
}

template <typename K>
static int launch_persistent(K kern, int grid, const CUtensorMap& t0, const CUtensorMap& t1, const CUtensorMap& t2,
                             const void* params, cudaStream_t st);

int tapgemm_f_tc_launch(const sg_tapgemm_f* q, cudaStream_t st) {
  FTcParams p;
  p.a0_c = q->a0_c; p.kc = q->kc; p.nc = q->nc; p.a_halo = q->a_halo;
  p.d_lo = q->d_lo; p.d_hi = q->d_hi;
  for (int i = 0; i < NTAP; ++i) {
    p.tr.k_lo[i] = q->tap_k_lo[i]; p.tr.k_hi[i] = q->tap_k_hi[i];
    p.tr.n_lo[i] = q->tap_n_lo[i]; p.tr.n_hi[i] = q->tap_n_hi[i];
  }
  p.out = q->out; p.out_dtype = q->out_dtype; p.out_rows = q->out_rows; p.out_halo = q->out_halo;
  p.out_ld = q->out_ld > 0 ? q->out_ld : q->nc;
  p.out_col0 = q->out_ld > 0 ? q->out_col0 : q->n_lo;
  p.w_tap0 = q->w_tap0;
  p.m_lo = q->m_lo; p.m_hi = q->m_hi; p.n_lo = q->n_lo;
  p.bias = q->bias; p.bias_mod = q->bias_mod > 0 ? q->bias_mod : q->nc;
  p.batch = q->batch; p.ksplit = q->ksplit < 1 ? 1 : q->ksplit;
  const int rows_m = q->m_hi - q->m_lo;
  const int ncols = q->n_hi - q->n_lo;
  p.TN = (ncols % 256 == 0) ? 256 : (ncols % 128 == 0 ? 128 : 64);
  if ((q->tile_n == 64 || q->tile_n == 128 || q->tile_n == 256) && ncols % q->tile_n == 0 && q->tile_n < p.TN)
    p.TN = q->tile_n;      // narrow tiles: the caller split this launch off as the tail of a larger one
  p.n_tiles = ncols / p.TN;
  // M tiling.  A segment of R rows per batch element is packed into 128-row tiles: TR = min(R, 128) rows of
  // TB = min(128 / TR, batch) batch elements.  Row counts just above a multiple of 128 or of a power of two waste most
  // of a tile (a data gradient computes R + 8 rows: 72 rows leave 56 of 128 dead, 264 rows a third tile of 8), so the
  // rows may be split into a leading segment R0 (a multiple of 128, or the largest power of two <= rows_m) and the
  // remaining R1 < 128 rows, packed on their own.  The split is taken when it strictly lowers the M tile count and
  // still leaves at least one tile per SM: launches smaller than that (none of the step's at batch 300) keep their
  // tiling and with it their stream-K tail.  out2 and BatchNorm-stat launches keep one segment: they compute a layer's
  // own rows (powers of two in the step), and their second output and column statistics are written and tested with
  // one segment only.
  auto seg_tiles = [&](int R, int& TR, int& TB) {
    if (R >= 128) { TR = 128; TB = 1; }
    else { TR = R; TB = 128 / R; if (TB > q->batch) TB = q->batch; }
    return ((R + TR - 1) / TR) * ((q->batch + TB - 1) / TB);
  };
  int R0 = rows_m;
  p.m_tiles0 = seg_tiles(rows_m, p.TR, p.TB);
  p.m_tiles = p.m_tiles0;
  p.m_lo1 = q->m_hi; p.TR1 = 0; p.TB1 = 0;
  if (q->out2 == nullptr && q->bn_stats == nullptr) {
    int r0 = 128 * (rows_m / 128);
    if (rows_m <= 128) for (r0 = 1; 2 * r0 <= rows_m; r0 *= 2) {}
    if (r0 < rows_m) {
      int TR0, TB0, TR1, TB1;
      const int t0 = seg_tiles(r0, TR0, TB0), t1 = seg_tiles(rows_m - r0, TR1, TB1);
      if (t0 + t1 < p.m_tiles && (t0 + t1) * p.n_tiles * p.ksplit >= num_sms()) {
        R0 = r0;
        p.TR = TR0; p.TB = TB0; p.m_tiles0 = t0; p.m_tiles = t0 + t1;
        p.m_lo1 = q->m_lo + r0; p.TR1 = TR1; p.TB1 = TB1;
      }
    }
  }
  p.m_tiles_per_b = (R0 + p.TR - 1) / p.TR;
  static const bool verbose = getenv("SEGAN_B200_SK_VERBOSE") != nullptr;
  if (verbose)
    fprintf(stderr, "tapgemm_f M tiles: %d rows x %d: %d rows as %d x %d -> %d, %d rows as %d x %d -> %d\n", rows_m,
            q->batch, R0, p.TR, p.TB, p.m_tiles0, rows_m - R0, p.TR1, p.TB1, p.m_tiles - p.m_tiles0);
  {
    static const int dbg_env = [] { const char* e = getenv("SEGAN_B200_DEBUG"); return e ? atoi(e) : 0; }();
    p.dbg = dbg_env;
  }
  p.stats = q->bn_stats;
  p.sk_dp_tiles = 0x7fffffff; p.sk_split = 1; p.sk_ws = nullptr; p.sk_cnt = nullptr;
  p.out2 = q->out2; p.out2_halo = q->out2_halo; p.slope = q->slope; p.slope_mod = q->slope_mod;
  p.bias_mask = (p.bias_mod & (p.bias_mod - 1)) == 0 ? p.bias_mod - 1 : -1;
  p.slope_mask = (p.slope_mod > 0 && (p.slope_mod & (p.slope_mod - 1)) == 0) ? p.slope_mod - 1 : -1;
  if (q->bn_stats != nullptr) SG_CHECK_ARG(p.ksplit == 1 && q->out_dtype != SG_F32 && q->n_lo == 0 && q->n_hi == q->nc);
  CUtensorMap tmA0, tmA1, tmW;
  const int a_buf_rows = q->a_rows + 2 * q->a_halo;
  int rc = make_map3(&tmA0, q->a0, q->a_dtype, q->a0_c, a_buf_rows, q->batch, p.TR, p.TB);
  if (rc) return rc;
  if (q->a1) rc = make_map3(&tmA1, q->a1, q->a_dtype, q->a1_c, a_buf_rows, q->batch, p.TR, p.TB);
  else tmA1 = tmA0;
  if (rc) return rc;
  CUtensorMap tmA0s1 = tmA0, tmA1s1 = tmA1;       // segment 1: the same rows, its own box
  if (p.TR1 > 0) {
    rc = make_map3(&tmA0s1, q->a0, q->a_dtype, q->a0_c, a_buf_rows, q->batch, p.TR1, p.TB1);
    if (rc) return rc;
    if (q->a1) rc = make_map3(&tmA1s1, q->a1, q->a_dtype, q->a1_c, a_buf_rows, q->batch, p.TR1, p.TB1);
    else tmA1s1 = tmA0s1;
    if (rc) return rc;
  }
  rc = make_map2(&tmW, q->w, q->w_dtype, q->kc, (int64_t)(q->d_hi + 4 - q->w_tap0 + 1) * q->nc, p.TN);
  if (rc) return rc;
  const int tiles = p.m_tiles * p.n_tiles * p.ksplit;
  int nctas = num_sms();
  if (tiles < nctas) nctas = tiles;
  // split-K over the last, partial wave (see PieceIter).  Cost model in k-steps of this launch's tile: leaving the
  // leftover tiles whole costs `steps`; splitting each over S CTAs costs steps / S for the MMAs, the finisher's
  // ordered sum of S partial tiles (g_sk_atomic_steps each for a 256-wide tile) and a fixed ~g_sk_fixed_steps of
  // fences, counters and pipeline refill.  Short-K layers are left alone.
  if (q->sk_ws != nullptr && g_stream_k > 1 && p.ksplit == 1 && q->bn_stats == nullptr && nctas <= SK_MAX_CTAS &&
      tiles > nctas && tiles % nctas != 0) {
    const int r = tiles % nctas;
    int steps = 0;                                  // k-steps of a leftover tile (the last N tile: the longest)
    for (int d = q->d_lo; d <= q->d_hi; ++d) steps += (q->tap_k_hi[d + 4] - q->tap_k_lo[d + 4]) / 64;
    int best_s = 1;
    double best = (double)steps;
    int s_max = nctas / r < g_stream_k ? nctas / r : g_stream_k;
    if (s_max > steps / 2) s_max = steps / 2;       // every piece keeps at least two k-steps
    const double per_partial = g_sk_atomic_steps * 256.0 / p.TN;      // narrower tiles have shorter k-steps
    for (int S = 2; S <= s_max; ++S) {
      const double c = (double)steps / S + per_partial * S + g_sk_fixed_steps;
      if (c < best) { best = c; best_s = S; }
    }
    const bool split = best_s > 1 && best < 0.92 * steps && steps >= 2 * best_s;
    if (verbose)
      fprintf(stderr, "tapgemm_f split-K: %d tiles on %d CTAs, %d left over, %d k-steps, TN %d -> split %d\n",
              tiles, nctas, r, steps, p.TN, split ? best_s : 1);
    if (split) {
      p.sk_dp_tiles = (tiles / nctas) * nctas;
      p.sk_split = best_s;
      p.sk_cnt = reinterpret_cast<unsigned int*>(q->sk_ws);
      p.sk_ws = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(q->sk_ws) + SK_CNT_BYTES);
    }
  }
  // whole tiles of a 16-bit output leave through shared memory and TMA stores (f_epilogue_tma); fp32 outputs (atomic
  // k-split, the waveform-end P), BatchNorm-stat launches and the split-K pieces store from the fragment
  p.tma_out = q->out_dtype != SG_F32 && q->bn_stats == nullptr;
  CUtensorMap tmO = tmA0, tmO2 = tmA0, tmOs1 = tmA0;
  if (p.tma_out) {
    rc = make_store_map3(&tmO, q->out, q->out_dtype, ncols, R0, q->batch, p.out_ld, q->out_rows + 2 * q->out_halo,
                         q->out_halo + q->m_lo, p.out_col0, p.TR, p.TB);
    if (rc) return rc;
    if (p.TR1 > 0) {
      rc = make_store_map3(&tmOs1, q->out, q->out_dtype, ncols, rows_m - R0, q->batch, p.out_ld,
                           q->out_rows + 2 * q->out_halo, q->out_halo + p.m_lo1, p.out_col0, p.TR1, p.TB1);
      if (rc) return rc;
    }
    if (q->out2 != nullptr) {
      rc = make_store_map3(&tmO2, q->out2, q->out_dtype, ncols, rows_m, q->batch, p.out_ld,
                           q->out_rows + 2 * q->out2_halo, q->out2_halo + q->m_lo, p.out_col0, p.TR, p.TB);
      if (rc) return rc;
    }
  }
  const bool bf = q->a_dtype == SG_BF16;
  void (*kern)(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap,
               FTcParams);
  int smem_bytes;
  if (p.TN == 256) { kern = bf ? tapgemm_f_tc<256, true> : tapgemm_f_tc<256, false>; smem_bytes = FSmem<256>::BYTES; }
  else if (p.TN == 128) { kern = bf ? tapgemm_f_tc<128, true> : tapgemm_f_tc<128, false>; smem_bytes = FSmem<128>::BYTES; }
  else { kern = bf ? tapgemm_f_tc<64, true> : tapgemm_f_tc<64, false>; smem_bytes = FSmem<64>::BYTES; }
  SG_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
  void* args[] = {&tmA0, &tmA1, &tmW, &tmO, &tmO2, &tmA0s1, &tmA1s1, &tmOs1, &p};
  SG_CHECK_CUDA(cudaLaunchKernel(reinterpret_cast<const void*>(kern), dim3(nctas), dim3(NUM_THREADS), args,
                                 (size_t)smem_bytes, st));
  return SG_OK;
}

template <typename K>
static int launch_persistent(K kern, int grid, const CUtensorMap& t0, const CUtensorMap& t1, const CUtensorMap& t2,
                             const void* params, cudaStream_t st) {
  SG_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
  void* args[] = {const_cast<CUtensorMap*>(&t0), const_cast<CUtensorMap*>(&t1), const_cast<CUtensorMap*>(&t2),
                  const_cast<void*>(params)};
  SG_CHECK_CUDA(cudaLaunchKernel(reinterpret_cast<const void*>(kern), dim3(grid), dim3(NUM_THREADS), args,
                                 (size_t)SMEM_BYTES, st));
  return SG_OK;
}

int tapgemm_w_tc_launch(const sg_tapgemm_w* q, cudaStream_t st) {
  WTcParams p;
  p.a0_c = q->a0_c; p.kc = q->kc; p.nc = q->nc; p.a_halo = q->a_halo;
  p.d_lo = q->d_lo; p.d_hi = q->d_hi;
  for (int i = 0; i < NTAP; ++i) {
    p.tr.k_lo[i] = q->tap_k_lo[i]; p.tr.k_hi[i] = q->tap_k_hi[i];
    p.tr.n_lo[i] = q->tap_n_lo[i]; p.tr.n_hi[i] = q->tap_n_hi[i];
  }
  p.dw = q->dw; p.dw_tap0 = q->dw_tap0; p.g_rows = q->g_rows; p.batch = q->batch;
  p.PR = q->g_rows >= 64 ? 64 : q->g_rows;
  p.PB = 64 / p.PR;
  const int TK = q->kc % 256 == 0 ? 256 : (q->kc % 128 == 0 ? 128 : 64);
  p.n_tiles = q->nc / 128;
  p.k_tiles = q->kc / TK;
  p.row_chunks = (q->g_rows + p.PR - 1) / p.PR;
  p.b_chunks = (q->batch + p.PB - 1) / p.PB;
  const int pos_steps = p.row_chunks * p.b_chunks;
  p.ksplit = q->ksplit < 1 ? 1 : q->ksplit;
  if (p.ksplit > pos_steps) p.ksplit = pos_steps;
  p.out_scale = q->out_scale;
  CUtensorMap tmG, tmA0, tmA1;
  int rc = make_map3(&tmG, q->g, q->g_dtype, q->nc, q->g_rows, q->batch, p.PR, p.PB);
  if (rc) return rc;
  const int a_buf_rows = q->a_rows + 2 * q->a_halo;
  rc = make_map3(&tmA0, q->a0, q->a_dtype, q->a0_c, a_buf_rows, q->batch, p.PR, p.PB);
  if (rc) return rc;
  if (q->a1) rc = make_map3(&tmA1, q->a1, q->a_dtype, q->a1_c, a_buf_rows, q->batch, p.PR, p.PB);
  else tmA1 = tmA0;
  if (rc) return rc;
  const int total = (q->d_hi - q->d_lo + 1) * p.n_tiles * p.k_tiles * p.ksplit;
  const int grid = total < num_sms() ? total : num_sms();
  const bool bf = q->g_dtype == SG_BF16;
  if (TK == 256) return launch_persistent(bf ? tapgemm_w_tc<256, true> : tapgemm_w_tc<256, false>, grid, tmG, tmA0, tmA1, &p, st);
  if (TK == 128) return launch_persistent(bf ? tapgemm_w_tc<128, true> : tapgemm_w_tc<128, false>, grid, tmG, tmA0, tmA1, &p, st);
  return launch_persistent(bf ? tapgemm_w_tc<64, true> : tapgemm_w_tc<64, false>, grid, tmG, tmA0, tmA1, &p, st);
}

}  // namespace sg
