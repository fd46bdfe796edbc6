// tc_common.cuh -- sm_90a primitives used by the tensor-core path: mbarrier, TMA (cp.async.bulk.tensor), wgmma
// (warpgroup MMA with shared-memory descriptors), cp.async.  Inline PTX only; the descriptor layout follows the PTX
// ISA "matrix descriptor" table for wgmma.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "grl_common.cuh"

namespace grl {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  // suspend-time hint: the thread sleeps in hardware until the phase completes (or ~1 ms passes) instead of
  // spinning -- waiting warps must not eat the issue slots of the warps doing the softmax / epilogue math.
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(1000000u)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug traps (-> CUDA error reported through the C ABI) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  int spins = 0;
  long long t0 = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 63) == 0) {  // wall-clock bound (~2 s), checked rarely so that waiting costs no issue slots
      const long long now = clock64();
      if (t0 == 0) t0 = now;
      else if (now - t0 > 4000000000ll) __trap();
    }
  }
}

// ------------------------------------------------------------------ proxies / fences
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ------------------------------------------------------------------ TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// ------------------------------------------------------------------ cp.async (LDGSTS) for gathered rows
__device__ __forceinline__ void cp_async_16(void* smem, const void* gmem, bool valid) {
  const int sz = valid ? 16 : 0;  // src-size 0 -> zero fill
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem)), "l"(gmem), "r"(sz) : "memory");
}
// 1-D bulk copy global -> shared (TMA engine, no tensor map): bytes % 16 == 0, both addresses 16-byte aligned
__device__ __forceinline__ void bulk_load_1d(void* smem, const void* gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem)),
               "l"(gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// ------------------------------------------------------------------ wgmma (sm_90a warpgroup MMA)
// Shared-memory matrix descriptor (64-bit): start address, leading / stride byte offsets (16-byte units), layout
// (swizzle) type in bits [62,64).  Operand tiles start at an address aligned to their swizzle repeat (512 B for 64B,
// 1024 B for 128B), so the base-offset field stays 0; a K step inside a swizzle atom advances the start address.
enum : uint32_t { SWZ_NONE = 0, SWZ_128B = 1, SWZ_64B = 2, SWZ_32B = 3 };
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t swz) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= (uint64_t)swz << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Pins accumulator registers in program order, so that the compiler moves no arithmetic on them across an in-flight
// wgmma's issue or wait (it does not know that the MMA writes them asynchronously).
template <int N>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// Accumulator fragment of one m64nN warpgroup MMA: thread t (warp w = t / 32, lane l) holds, for every 8-column block i,
// d[4i + {0,1}] = D[16w + l/4][8i + 2(l%4) + {0,1}] and d[4i + {2,3}] = the same columns of row 16w + l/4 + 8.
// D[64 x N] (+)= A[64 x 16] * B[16 x N]; A K-major, B K-major (n64) or MN-major (n32, transposed B).  All 128 threads of
// the warpgroup execute these.
#define GRL_D16 "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
#define GRL_D32 GRL_D16, "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
#define GRL_R16 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
#define GRL_R32 GRL_R16 ", %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
// NAME(d, adesc, bdesc, accumulate): one m64nNk16 MMA with fp32 accumulators d[NREG = N / 2]; A, B, P: the asm operand
// numbers of the two descriptors and of the accumulate flag; TNSPB = 1: B is MN-major.
#define GRL_WGMMA(NAME, N, NREG, REGS, OUTS, A, B, P, TY, TNSPB)                                                    \
  __device__ __forceinline__ void NAME(float (&d)[NREG], uint64_t adesc, uint64_t bdesc, bool accumulate) {         \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #P ", 0;\n\t"                                                 \
                 "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32." TY "." TY " {" REGS "}, %" #A ", %" #B ", p, 1, 1, 0, " \
                 #TNSPB ";\n\t}"                                                                                     \
                 : OUTS                                                                                              \
                 : "l"(adesc), "l"(bdesc), "r"((uint32_t)accumulate));                                               \
  }
GRL_WGMMA(wgmma_n64_bf16, 64, 32, GRL_R32, GRL_D32, 32, 33, 34, "bf16", 0)
GRL_WGMMA(wgmma_n64_f16, 64, 32, GRL_R32, GRL_D32, 32, 33, 34, "f16", 0)
GRL_WGMMA(wgmma_n32t_bf16, 32, 16, GRL_R16, GRL_D16, 16, 17, 18, "bf16", 1)
GRL_WGMMA(wgmma_n32t_f16, 32, 16, GRL_R16, GRL_D16, 16, 17, 18, "f16", 1)
// Register-A form: m64n32k16, D += A B with A[64 x 16] from registers and B MN-major in shared memory.  Thread t (warp w,
// lane l) supplies a[0] = A[16w + l/4][2(l%4) + {0,1}], a[1] = the same columns of row 16w + l/4 + 8, a[2] / a[3] = columns
// 8 + 2(l%4) + {0,1} of those two rows (low half = lower column) -- for k = 16j..16j+15 that is exactly the accumulator
// fragment of an m64nN product over those columns (blocks 2j and 2j + 1 above), packed to 16 bits.
#define GRL_WGMMA_RS(NAME, TY)                                                                                        \
  __device__ __forceinline__ void NAME(float (&d)[16], const uint32_t (&a)[4], uint64_t bdesc) {                     \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"                                                    \
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32." TY "." TY " {" GRL_R16 "}, {%16, %17, %18, %19}, %20, " \
                 "p, 1, 1, 1;\n\t}"                                                                                 \
                 : GRL_D16                                                                                          \
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc));                                         \
  }
GRL_WGMMA_RS(wgmma_rs_n32t_bf16, "bf16")
GRL_WGMMA_RS(wgmma_rs_n32t_f16, "f16")

__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
// Operand formats of the tensor-core path: FMT_F16 (default: 11-bit mantissa, saturating converts) or FMT_BF16.
enum : int { FMT_F16 = 0, FMT_BF16 = 1 };
inline int check_fmt(int fmt) {
  GRL_REQUIRE(fmt == 0 || fmt == 1, "tc: operand format must be 0 (fp16) or 1 (bf16), got %d", fmt);
  return GRL_OK;
}
// GrlTcGemm::epi: the fused epilogues of gemm_tc_kernel
enum { EPI_BIAS_ACT = 0, EPI_QKV = 1, EPI_LN = 2 };
__device__ __forceinline__ uint32_t pack_f16(float lo, float hi) {
  uint32_t d;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
  return d;
}
__device__ __forceinline__ uint32_t pack16(float lo, float hi, int fmt) {
  return fmt == FMT_BF16 ? pack_bf16(lo, hi) : pack_f16(lo, hi);
}
__device__ __forceinline__ float2 unpack16(uint32_t v, int fmt) {
  if (fmt == FMT_BF16) return make_float2(__uint_as_float(v << 16), __uint_as_float(v & 0xFFFF0000u));
  return __half22float2(*reinterpret_cast<const __half2*>(&v));
}
__device__ __forceinline__ float unpack16_one(uint16_t v, int fmt) {
  if (fmt == FMT_BF16) return __uint_as_float((uint32_t)v << 16);
  return __half2float(*reinterpret_cast<const __half*>(&v));
}

// ------------------------------------------------------------------ host: tensor maps without linking libcuda
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_tiled_fn();  // gemm_tc.cu

}  // namespace tc
}  // namespace grl
