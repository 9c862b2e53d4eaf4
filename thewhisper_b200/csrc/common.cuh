// Shared device helpers for the sm_90a kernels: mbarrier / TMA / wgmma PTX wrappers, small math.
// Everything here is hand-written PTX for Hopper; no CUTLASS/CuTe templates are used.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

// Every kernel source is compiled twice: once with 16-bit elements = bfloat16 (namespace bw) and once, with -DBW_F16, = IEEE half
// (namespace bw_f16) -- the reference's streaming / benchmark paths run fp16 (REF streaming_pipeline.py:369-370).  Same byte cost,
// same wgmma instructions with the operand type .bf16 or .f16; accumulation, softmax,
// LayerNorm and the residual stream are fp32 in both.  `bf16` below is the historical name of "the engine's 16-bit element type".
#ifdef BW_F16
#define BW_NS bw_f16
#define BW_TMAP_DTYPE CU_TENSOR_MAP_DATA_TYPE_FLOAT16
#define BW_WGMMA_AB "f16"  // wgmma operand type
#else
#define BW_NS bw
#define BW_TMAP_DTYPE CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
#define BW_WGMMA_AB "bf16"
#endif

namespace BW_NS {

#ifdef BW_F16
typedef __half bf16;
__host__ __device__ __forceinline__ bf16 f2e(float x) { return __float2half_rn(x); }
__host__ __device__ __forceinline__ float e2f(bf16 x) { return __half2float(x); }
#else
typedef __nv_bfloat16 bf16;
__host__ __device__ __forceinline__ bf16 f2e(float x) { return __float2bfloat16(x); }
__host__ __device__ __forceinline__ float e2f(bf16 x) { return __bfloat162float(x); }
#endif

// ------------------------------------------------------------------------------------------------
// error plumbing (host)
// ------------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
const char* get_error();
#define BW_CUDA_OK(expr)                                                                       \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess) {                                                                   \
      BW_NS::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e));     \
      return -1;                                                                               \
    }                                                                                          \
  } while (0)
#define BW_CHECK(cond, ...)                                                                    \
  do {                                                                                         \
    if (!(cond)) {                                                                             \
      BW_NS::set_error(__VA_ARGS__);                                                              \
      return -2;                                                                               \
    }                                                                                          \
  } while (0)

// ------------------------------------------------------------------------------------------------
// generic device helpers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// 2^x on the SFU, one instruction (MUFU.EX2; flush-to-zero): exp2f() wraps the same instruction in denormal-range fix-ups
// (FSETP + 2 FMUL) that the softmax kernels do not need -- their arguments are <= 8 and underflow to 0 is what they want
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// exact (erf) GELU, as torch.nn.functional.gelu(approximate="none")
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

#ifdef BW_F16
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __half2 t = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ float2 unpack_bf16(uint32_t u) {
  __half2 t = *reinterpret_cast<__half2*>(&u);
  return __half22float2(t);
}
#else
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ float2 unpack_bf16(uint32_t u) {
  __nv_bfloat162 t = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(t);
}
#endif

// Four signed int8 weight codes (int8 decoder weights) -> four exact floats without I2F (16 per clock per SM on sm_90): byte
// b + 128 is permuted into the low mantissa byte of 2^23 (0x4B0000xx = 2^23 + b + 128), one FADD removes 2^23 + 128.
// A zero word gives four zeros.
__device__ __forceinline__ void unpack_s8x4(uint32_t u, float (&f)[4]) {
  const uint32_t b = u ^ 0x80808080u;
  f[0] = __uint_as_float(__byte_perm(b, 0x4B000000u, 0x7540)) - 8388736.f;
  f[1] = __uint_as_float(__byte_perm(b, 0x4B000000u, 0x7541)) - 8388736.f;
  f[2] = __uint_as_float(__byte_perm(b, 0x4B000000u, 0x7542)) - 8388736.f;
  f[3] = __uint_as_float(__byte_perm(b, 0x4B000000u, 0x7543)) - 8388736.f;
}

// 16-byte streaming load that does not pollute L1 (weights / KV are read once per step)
__device__ __forceinline__ uint4 ld_nc_u4(const void* p) {
  uint4 r;
  // volatile + "memory": the compiler must not sink these below later smem traffic / barriers -- the decode kernels
  // rely on all of a CTA's loads being issued up front (one DRAM round trip)
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p)
               : "memory");
  return r;
}
__device__ __forceinline__ uint2 ld_nc_u2(const void* p) {
  uint2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p) : "memory");
  return r;
}

// ------------------------------------------------------------------------------------------------
// programmatic dependent launch (the batched decoder step: ~360 kernels per token in one CUDA graph).  A kernel launched with
// the programmatic-serialization attribute may START while its predecessor still runs: everything that touches memory the
// predecessor writes (or reads: WAR) comes after pdl_wait(); weights and other constants may be requested before it.
// pdl_launch() lets the NEXT kernel's CTAs be scheduled early.  Both are no-ops in a kernel launched the plain way.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
extern int g_pdl;  // host: 1 while a launcher should attach the programmatic-serialization attribute (set by step_batched)

template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = g_pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// ------------------------------------------------------------------------------------------------
// mbarrier
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok;
}
// non-blocking test (try_wait may park the thread for a while): for issuers that poll several barriers
__device__ __forceinline__ uint32_t mbar_test(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok;
}
// Bounded wait: a protocol bug must surface as a trapped kernel (an error code at the C-ABI), never as a
// hung GPU box.  ~2^32 cycles is about 2 s at 1.9 GHz, far beyond any legitimate wait in these kernels.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > (1ll << 32)) {
      printf("[bw] mbarrier wait timed out: block (%d,%d,%d) thread %d bar %p parity %u\n", blockIdx.x, blockIdx.y,
             blockIdx.z, threadIdx.x, (void*)bar, parity);
      __trap();
    }
  }
}
// The same bounded wait without the diagnostic printf, for kernels that issue wgmma: a function call anywhere in such a kernel
// makes ptxas serialise its wgmma instructions.
__device__ __forceinline__ void mbar_wait_wg(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity))
    if (clock64() - t0 > (1ll << 32)) __trap();
}

// generic-proxy smem writes -> visible to the async proxy (TMA / wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ------------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor), loads only; tensor maps are passed as __grid_constant__ kernel params
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// ------------------------------------------------------------------------------------------------
// wgmma (sm_90a warpgroup MMA): D in registers, A and B from shared memory (or A from registers)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// The accumulator registers are operands of asynchronous instructions between wg_fence() and wg_wait(): this keeps the compiler
// from moving their reads / writes across those points.
template <int R>
__device__ __forceinline__ void wg_pin(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// shared-memory matrix descriptor, 128-byte swizzle (what a TMA box of 64 16-bit elements x rows with CU_TENSOR_MAP_SWIZZLE_128B
// produces).  K-major: 8-row groups 1024 B apart (SBO), LBO unused; +2 on the descriptor = +32 B = the next 16 elements of K.
// MN-major (N = 64 = one swizzle atom wide): 8-row groups of K 1024 B apart (SBO); +128 = +2048 B = the next 16 rows of K.
// Field layout (sm_90 GMMA descriptor): addr>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46), base offset [49,52), layout [62,64) with
// SWIZZLE_128B = 1.  Every operand tile is 1024-byte aligned, so the base offset is 0.
__device__ __forceinline__ uint64_t wg_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// Accumulator layout of m64nNk16 (per warpgroup, fp32): warp w of the group owns rows 16 w + (lane >> 2) and that + 8;
// d[4 j + 2 h + c] is row 16 w + (lane >> 2) + 8 h, column 8 j + 2 (lane & 3) + c.
template <int N>
struct Wgmma;
template <>
struct Wgmma<32> {
  // D[64 x 32] (+)= A[64 x 16] (smem) * B[32 x 16]^T (smem); TB = 1: B is MN-major
  template <int TB>
  static __device__ __forceinline__ void ss(float (&d)[16], uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32." BW_WGMMA_AB "." BW_WGMMA_AB " "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "%16, %17, p, 1, 1, 0, %19;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TB));
  }
};
template <>
struct Wgmma<64> {
  // D[64 x 64] (+)= A[64 x 16] (smem) * B[64 x 16]^T (smem); TB = 1: B is MN-major
  template <int TB>
  static __device__ __forceinline__ void ss(float (&d)[32], uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32." BW_WGMMA_AB "." BW_WGMMA_AB " "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1, 0, %35;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TB));
  }
  // A from registers (four 32-bit registers per thread: the m16n8k16 A fragment layout per warp)
  template <int TB>
  static __device__ __forceinline__ void rs(float (&d)[32], const uint32_t (&a)[4], uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32." BW_WGMMA_AB "." BW_WGMMA_AB " "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "{%32, %33, %34, %35}, %36, p, 1, 1, %38;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(scale_d), "n"(TB));
  }
};
template <>
struct Wgmma<128> {
  // D[64 x 128] (+)= A[64 x 16] (smem) * B[128 x 16]^T (smem); TB = 1: B is MN-major
  template <int TB>
  static __device__ __forceinline__ void ss(float (&d)[64], uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32." BW_WGMMA_AB "." BW_WGMMA_AB " "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, %67;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TB));
  }
};
template <>
struct Wgmma<256> {
  // D[64 x 256] (+)= A[64 x 16] (smem) * B[256 x 16]^T (smem); TB = 1: B is MN-major
  template <int TB>
  static __device__ __forceinline__ void ss(float (&d)[128], uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32." BW_WGMMA_AB "." BW_WGMMA_AB " "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
        "%128, %129, p, 1, 1, 0, %131;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TB));
  }
};

// One 64-deep k-block of a warpgroup's 64 x BN tile: 4 x m64nBNk16 over K-major 128B-swizzled operands (A: 64 rows at sa,
// B: BN rows at sb).  The caller brackets it with wg_fence() / wg_commit().
template <int BN>
__device__ __forceinline__ void wg_kblock(float (&d)[BN / 2], uint32_t sa, uint32_t sb) {
  const uint64_t a0 = wg_desc_sw128(sa), b0 = wg_desc_sw128(sb);
#pragma unroll
  for (int k = 0; k < 4; ++k) Wgmma<BN>::template ss<0>(d, a0 + 2 * k, b0 + 2 * k, 1u);
}

// ------------------------------------------------------------------------------------------------
// host: TMA tensor-map encoding without linking libcuda (driver entry point fetched at run time)
// ------------------------------------------------------------------------------------------------
// 2-D bf16 tensor, inner dimension contiguous.  rows x cols logical, row pitch in BYTES (multiple of 16; rows
// may overlap, which is how the conv stem reads its im2col view), box = box_rows x box_cols (box_cols*2 == 128
// for the 128-byte swizzle used everywhere here).
int make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t row_pitch_bytes,
                      uint32_t box_rows, uint32_t box_cols);
// the same for a 2-D uint8 tensor (int8 weight codes), unswizzled: box_cols bytes per row
int make_tmap_2d_u8(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t row_pitch_bytes, uint32_t box_rows,
                    uint32_t box_cols);
// 3-D: batch x rows x cols, both pitches in bytes; coordinates past rows (or batch) read as zeros
int make_tmap_3d_bf16(CUtensorMap* out, const void* base, uint64_t batch, uint64_t rows, uint64_t cols, uint64_t row_pitch_bytes,
                      uint64_t batch_pitch_bytes, uint32_t box_rows, uint32_t box_cols);
// multiprocessor count of the current device (queried once)
int device_sms();

}  // namespace bw
