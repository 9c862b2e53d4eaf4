// wgmma / TMA GEMM for sm_90a:  C[b,t,n] = epi( sum_k A(b,t,k) * W[n,k] ).
//
// Replaces the cuBLAS GEMMs + cuDNN convs the reference reaches through torch
// (TF/models/whisper/modeling_whisper.py:279-336 q/k/v/out projections, :404-407 fc1/fc2, :619-620 conv stem).
//
// Structure (one 128 x BN output tile per CTA, 288 threads):
//   warps 0-7  two consumer warpgroups: warpgroup g issues 4 x wgmma m64nBNk16 per 64-wide k-block for tile rows [64 g, 64 g + 64),
//              keeps one k-block in flight and hands the previous smem stage back; the epilogue (bias/alpha/GELU/pos/residual)
//              runs on the accumulator registers
//   warp  8    TMA producer (one lane): 128B-swizzled K-major boxes of A (3-D map, wrapping k for the conv
//              stem) and W into a STAGES-deep smem ring, completion on mbarriers
// Tiles walk n-fastest (blockIdx.x): the CTAs running together work on a few 128-row bands of A against all of W (<= 13 MB:
// L2-resident), so A streams from DRAM about once.
// gemm_tc2 runs the same kernel over the encoder's activations of all B items as ONE [B * rows, K] matrix (no per-item tail tiles:
// 1500 rows per item leave a 92-row tail); its epilogue maps the flat row r back to b = r / rows_per_item, t = r % rows_per_item,
// and is compiled once per combination the encoder uses (MODE) with the 2-MUFU GELU below.
#include <limits.h>

#include "kernels.h"

namespace BW_NS {

namespace {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int A_STAGE_BYTES = BM * BK * 2;  // 16 KB
constexpr int THREADS = 288;
constexpr int CONSUMER_WARPS = 8;

// BN = 32 is the decoder-step shape (q_len = 1 for up to 128 sequences per tile): the GEMM is a stream over the weight matrix, so
// the tile is narrow (N / 32 CTAs cover the SMs without split-K for N >= 3840) and the ring is deep (8 stages x 20 KB in flight per SM
// hide the DRAM latency).  Wider tiles take as many stages as fit in 227 KB of shared memory.
template <int BN>
struct Cfg {
  static constexpr int STAGES = (BN == 256) ? 4 : (BN == 128) ? 6 : 8;
  static constexpr int B_STAGE_BYTES = BN * BK * 2;
  static constexpr int SMEM_BYTES = STAGES * (A_STAGE_BYTES + B_STAGE_BYTES) + 1024 /*align slack*/ + 256 /*barriers*/;
};

// epilogue specialisations: the runtime-parameterised generic one executes every option's instructions predicated off
enum { EPI_GENERIC = 0, EPI_GELU = 1 /* bias, GELU -> 16 bit */, EPI_RESID = 2 /* bias, + fp32 residual -> fp32 */, EPI_PLAIN = 3 /* bias -> 16 bit */ };

struct GemmParams {
  int B, rows, N, K;
  int rows_per_item = INT_MAX;  // epilogue address map of a flat launch (B = 1): b = t / rows_per_item, t = t % rows_per_item
  int fast_gelu = 0;            // GELU through gelu_as (gemm_tc2) instead of erff
  int kwrap;
  int tiles_m;  // per item
  int ksplit;   // gridDim.z: split z handles k-blocks [z * kper, min(nk, (z + 1) * kper)) and writes its partial sums at
  int kper;     // out + z * split_stride (no bias / residual: the consumer adds the partials -- deterministic, no atomics)
  long long split_stride;
  GemmEpi epi;
};

__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
          smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// exact (erf) GELU to 4e-7 absolute: Phi(x) through Abramowitz-Stegun 7.1.26 (|erf error| <= 1.5e-7) -- 2 MUFU + 12 fp32 operations where erff
// costs ~25; the result is rounded to 16 bits right after (half an ulp there is >= 2.4e-4 relative).  tests/test_ops_gpu.py pins it to erf.
__device__ __forceinline__ float gelu_as(float x) {
  const float ax = fabsf(x);
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f * 0.70710678f, ax, 1.0f)));
  float q = 0.5f * 1.061405429f;
  q = fmaf(q, t, 0.5f * -1.453152027f);
  q = fmaf(q, t, 0.5f * 1.421413741f);
  q = fmaf(q, t, 0.5f * -0.284496736f);
  q = fmaf(q, t, 0.5f * 0.254829592f);
  q = (q * t) * ex2_approx((x * -0.72134752f) * x);  // 0.5 erfc(|x| / sqrt 2) = Phi(-|x|)
  return fmaf(-ax, q, fmaxf(x, 0.f));               // x >= 0: x - x q;  x < 0: x q
}

template <int BN, int MODE>
__global__ void __launch_bounds__(THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW, const GemmParams p) {
  using C = Cfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + C::STAGES * A_STAGE_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sB + C::STAGES * C::B_STAGE_BYTES);
  uint64_t* full = bars;
  uint64_t* empty = bars + C::STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.y / p.tiles_m;
  const int t0 = (blockIdx.y % p.tiles_m) * BM;
  const int n0 = blockIdx.x * BN;
  const int nk_all = (p.K + BK - 1) / BK;
  const int kb0 = (int)blockIdx.z * p.kper;
  const int nk = min(nk_all, kb0 + p.kper) - kb0;  // >= 1 (the launcher picks ksplit so that every split owns a k-block)

  if (threadIdx.x == 0) {
    for (int s = 0; s < C::STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], CONSUMER_WARPS);
    }
    fence_mbar_init();
  }
  if (warp == CONSUMER_WARPS && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmW);
  }
  __syncthreads();

  if (warp == CONSUMER_WARPS) {
    if (lane == 0) {
      // The weight tiles of the first ring pass do not depend on the previous kernel: under programmatic dependent launch they are
      // requested before the wait (their DRAM latency runs beside the predecessor's tail); the activations after it.
      const int npre = nk < C::STAGES ? nk : C::STAGES;
      for (int kb = 0; kb < npre; ++kb) {
        mbar_arrive_expect_tx(&full[kb], A_STAGE_BYTES + C::B_STAGE_BYTES);
        tma_load_2d(sB + kb * C::B_STAGE_BYTES, &tmW, &full[kb], (kb0 + kb) * BK, n0);
      }
      pdl_wait();
      pdl_launch();
      for (int kb = 0; kb < nk; ++kb) {
        const int s = kb % C::STAGES;
        const uint32_t ph = (kb / C::STAGES) & 1;
        const int k = (kb0 + kb) * BK;
        if (kb >= npre) {
          mbar_wait_wg(&empty[s], ph ^ 1);
          mbar_arrive_expect_tx(&full[s], A_STAGE_BYTES + C::B_STAGE_BYTES);
          tma_load_2d(sB + s * C::B_STAGE_BYTES, &tmW, &full[s], k, n0);
        }
        tma_load_3d(sA + s * A_STAGE_BYTES, &tmA, &full[s], k % p.kwrap, t0 + k / p.kwrap, b);
      }
    }
  } else {
    // ---------------- consumer warpgroup g: tile rows [64 g, 64 g + 64) ----------------
    const int g = warp >> 2;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < nk; ++kb) {
      const int s = kb % C::STAGES;
      mbar_wait_wg(&full[s], (kb / C::STAGES) & 1);
      wg_fence();
      wg_kblock<BN>(acc, smem_u32(sA + s * A_STAGE_BYTES + g * (A_STAGE_BYTES / 2)), smem_u32(sB + s * C::B_STAGE_BYTES));
      wg_commit();
      wg_wait<1>();  // k-block kb - 1 is complete: its stage goes back to the producer
      if (kb > 0 && lane == 0) mbar_arrive(&empty[(kb - 1) % C::STAGES]);
    }
    wg_wait<0>();
    wg_pin(acc);

    // ---------------- epilogue: this thread holds rows r and r + 8, two adjacent columns of every 8-column group ----------------
    pdl_wait();  // (residual reads / output stores: after the predecessor grid)
    const GemmEpi& e = p.epi;
    constexpr bool GEN = MODE == EPI_GENERIC;
    const bool do_alpha = GEN && e.alpha != 1.0f;
    const bool do_act = GEN ? e.act == 1 : MODE == EPI_GELU;
    const bool fast_gelu = GEN ? p.fast_gelu != 0 : true;
    const bool has_pos = GEN && e.pos != nullptr;
    const bool has_res = GEN ? e.residual != nullptr : MODE == EPI_RESID;
    const bool f32out = GEN ? e.out_f32 != nullptr : MODE == EPI_RESID;
    const int r = g * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int t = t0 + r + 8 * h;
      if (t >= p.rows) continue;
      const int bi = t / p.rows_per_item, ti = t - bi * p.rows_per_item;  // (bi = 0 unless a flat launch)
      const long long row_off = (long long)(b + bi) * e.batch_stride + (long long)ti * e.row_stride + (long long)blockIdx.z * p.split_stride;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int n = n0 + 8 * j + 2 * (lane & 3);
        if (n >= p.N) break;  // N % 32 == 0: uniform over the 8 x 4 threads of a 32-column chunk
        float f0 = acc[4 * j + 2 * h], f1 = acc[4 * j + 2 * h + 1];
        if (e.bias) {
          const float2 bb = __ldg(reinterpret_cast<const float2*>(e.bias + n));
          f0 += bb.x; f1 += bb.y;
        }
        if (do_alpha && n < e.alpha_cols) { f0 *= e.alpha; f1 *= e.alpha; }
        if (do_act) {
          if (fast_gelu) { f0 = gelu_as(f0); f1 = gelu_as(f1); }
          else { f0 = gelu_erf(f0); f1 = gelu_erf(f1); }
        }
        if (has_pos) {
          const float2 q = *reinterpret_cast<const float2*>(e.pos + (long long)t * p.N + n);
          f0 += q.x; f1 += q.y;
        }
        const long long off = row_off + (long long)(n >> 6) * e.head_stride + (n & 63);
        if (has_res) {
          const float2 q = *reinterpret_cast<const float2*>(e.residual + off);
          f0 += q.x; f1 += q.y;
        }
        if (f32out) *reinterpret_cast<float2*>(e.out_f32 + off) = make_float2(f0, f1);
        else *reinterpret_cast<uint32_t*>(e.out_bf16 + off) = pack_bf16(f0, f1);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// CUDA-core sibling (comparator / bring-up fallback).  One thread per output, 16x16 tile, no staging.
// ------------------------------------------------------------------------------------------------
__global__ void gemm_simt_kernel(GemmA a, const bf16* __restrict__ W, GemmParams p) {
  const int n = blockIdx.x * 16 + threadIdx.x;
  const int t = (blockIdx.y % p.tiles_m) * 16 + threadIdx.y;
  const int b = blockIdx.y / p.tiles_m;
  if (n >= p.N || t >= p.rows) return;
  const bf16* ab = a.base + (long long)b * a.batch_stride;
  const bf16* w = W + (long long)n * p.K;
  float acc = 0.f;
  const int kend = (p.epi.n_valid > 0 && n >= p.epi.n_valid) ? 0 : p.K;  // rows of W beyond n_valid do not exist: zero
  for (int k = 0; k < kend; ++k) {
    const float av = e2f(ab[(long long)(t + k / p.kwrap) * a.pitch + (k % p.kwrap)]);
    acc = fmaf(av, e2f(w[k]), acc);
  }
  const GemmEpi& e = p.epi;
  const long long off = (long long)b * e.batch_stride + (long long)t * e.row_stride + (long long)(n >> 6) * e.head_stride + (n & 63);
  if (e.bias) acc += e.bias[n];
  if (n < e.alpha_cols) acc *= e.alpha;
  if (e.act == 1) acc = gelu_erf(acc);
  if (e.pos) acc += e.pos[(long long)t * p.N + n];
  if (e.residual) acc += e.residual[off];
  if (e.out_f32) e.out_f32[off] = acc;
  else e.out_bf16[off] = f2e(acc);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !p) {
    set_error("cudaGetDriverEntryPoint(cuTensorMapEncodeTiled) failed: %s", cudaGetErrorString(e));
    return nullptr;
  }
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

int check_epi(const GemmEpi& e, int N) {
  BW_CHECK((e.out_f32 != nullptr) != (e.out_bf16 != nullptr), "gemm: exactly one of out_f32/out_bf16 must be set");
  BW_CHECK(N % 32 == 0, "gemm: N=%d must be a multiple of 32", N);
  BW_CHECK(e.row_stride % 8 == 0 && e.batch_stride % 8 == 0 && e.head_stride % 8 == 0, "gemm: output strides must be multiples of 8");
  return 0;
}

}  // namespace

int device_sms() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0) sms = n;
    else return 132;  // H100 SXM
  }
  return sms;
}

int make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t row_pitch_bytes,
                      uint32_t box_rows, uint32_t box_cols) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return -1;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {row_pitch_bytes};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t es[2] = {1, 1};
  CUresult r = fn(out, BW_TMAP_DTYPE, 2, const_cast<void*>(base), dims, strides, box, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  BW_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(2d rows=%llu cols=%llu pitch=%llu box=%ux%u) -> %d",
           (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)row_pitch_bytes, box_rows, box_cols, (int)r);
  return 0;
}

int make_tmap_2d_u8(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t row_pitch_bytes, uint32_t box_rows,
                    uint32_t box_cols) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return -1;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {row_pitch_bytes};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t es[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  BW_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(2d u8 rows=%llu cols=%llu pitch=%llu box=%ux%u) -> %d",
           (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)row_pitch_bytes, box_rows, box_cols, (int)r);
  return 0;
}

int make_tmap_3d_bf16(CUtensorMap* out, const void* base, uint64_t batch, uint64_t rows, uint64_t cols,
                      uint64_t row_pitch_bytes, uint64_t batch_pitch_bytes, uint32_t box_rows, uint32_t box_cols) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return -1;
  cuuint64_t dims[3] = {cols, rows, batch};
  cuuint64_t strides[2] = {row_pitch_bytes, batch_pitch_bytes};
  cuuint32_t box[3] = {box_cols, box_rows, 1};
  cuuint32_t es[3] = {1, 1, 1};
  CUresult r = fn(out, BW_TMAP_DTYPE, 3, const_cast<void*>(base), dims, strides, box, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  BW_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(3d batch=%llu rows=%llu cols=%llu pitch=%llu/%llu) -> %d",
           (unsigned long long)batch, (unsigned long long)rows, (unsigned long long)cols,
           (unsigned long long)row_pitch_bytes, (unsigned long long)batch_pitch_bytes, (int)r);
  return 0;
}

template <int BN, int MODE = EPI_GENERIC>
static int launch_tc(cudaStream_t st, const CUtensorMap& tmA, const bf16* W, const GemmParams& p) {
  using C = Cfg<BN>;
  CUtensorMap tmW;
  if (int rc = make_tmap_2d_bf16(&tmW, W, p.epi.n_valid > 0 ? p.epi.n_valid : p.N, p.K, (uint64_t)p.K * 2, BN, BK)) return rc;
  static bool attr_set = false;
  if (!attr_set) {
    BW_CUDA_OK(cudaFuncSetAttribute(gemm_tc_kernel<BN, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES));
    attr_set = true;
  }
  dim3 grid((p.N + BN - 1) / BN, p.tiles_m * p.B, p.ksplit);
  BW_CUDA_OK(launch_k(gemm_tc_kernel<BN, MODE>, grid, dim3(THREADS), (size_t)C::SMEM_BYTES, st, tmA, tmW, p));
  return 0;
}

int gemm_tc(cudaStream_t st, const GemmA& a, const bf16* W, int B, int rows, int N, int K, const GemmEpi& epi, int force_bn) {
  return gemm_tc_split(st, a, W, B, rows, N, K, epi, force_bn, 1, 0);
}

int gemm_tc_ksplit(int K, int ksplit) {
  const int nk = K / BK;
  if (ksplit > nk) ksplit = nk;
  if (ksplit < 1) ksplit = 1;
  const int kper = (nk + ksplit - 1) / ksplit;
  return (nk + kper - 1) / kper;
}

int gemm_tc_split(cudaStream_t st, const GemmA& a, const bf16* W, int B, int rows, int N, int K, const GemmEpi& epi, int force_bn,
                  int ksplit, long long split_stride) {
  if (int rc = check_epi(epi, N)) return rc;
  BW_CHECK(ksplit >= 1 && (ksplit == 1 || (epi.out_f32 && !epi.bias && !epi.residual && !epi.pos && epi.act == 0 && epi.alpha == 1.0f)),
           "gemm_tc: split-K writes raw fp32 partial sums (no bias / activation / residual)");
  BW_CHECK(K % 64 == 0, "gemm_tc: K=%d must be a multiple of 64", K);
  BW_CHECK(a.pitch % 8 == 0 && a.batch_stride % 8 == 0, "gemm_tc: A pitch/batch stride must be multiples of 8 elements");
  BW_CHECK(a.kwrap >= K || a.kwrap % 64 == 0, "gemm_tc: kwrap=%d must be a multiple of 64", a.kwrap);
  GemmParams p;
  p.B = B; p.rows = rows; p.N = N; p.K = K;
  p.kwrap = a.kwrap >= K ? INT_MAX : a.kwrap;
  p.tiles_m = (rows + BM - 1) / BM;
  p.epi = epi;
  {
    const int nk = K / BK;
    p.ksplit = gemm_tc_ksplit(K, ksplit);  // every split owns >= 1 k-block
    p.kper = (nk + p.ksplit - 1) / p.ksplit;
    p.split_stride = split_stride;
  }
  const uint64_t inner = (uint64_t)(a.kwrap >= K ? K : a.kwrap);
  CUtensorMap tmA;
  if (int rc = make_tmap_3d_bf16(&tmA, a.base, (uint64_t)B, (uint64_t)a.rows_base, inner, (uint64_t)a.pitch * 2,
                                 (uint64_t)(B > 1 ? a.batch_stride : (long long)a.rows_base * a.pitch) * 2, BM, BK))
    return rc;
  int bn = force_bn;
  if (bn == 0) {
    // enough CTAs to cover the SMs matters more than the wider tile when the grid is small
    const long long tiles128 = (long long)((N + 127) / 128) * p.tiles_m * B;
    bn = (N % 256 == 0 && tiles128 >= 4 * device_sms()) ? 256 : 128;
    if (N < 128) bn = 64;
  }
  switch (bn) {
    case 32: return launch_tc<32>(st, tmA, W, p);
    case 64: return launch_tc<64>(st, tmA, W, p);
    case 128: return launch_tc<128>(st, tmA, W, p);
    case 256: return launch_tc<256>(st, tmA, W, p);
  }
  BW_CHECK(false, "gemm_tc: unsupported BN=%d", bn);
}

bool gemm_tc2_supported(int M, int N, int K) { return K % BK == 0 && K >= BK && (N % 256 == 0 || N % 128 == 0) && M >= 1; }

int gemm_tc2(cudaStream_t st, const bf16* A, const bf16* W, int M, int N, int K, int rows_per_item, const GemmEpi& epi, int force_bn) {
  BW_CHECK((epi.out_f32 != nullptr) != (epi.out_bf16 != nullptr), "gemm_tc2: exactly one of out_f32/out_bf16 must be set");
  BW_CHECK(gemm_tc2_supported(M, N, K), "gemm_tc2: unsupported shape M=%d N=%d K=%d", M, N, K);
  BW_CHECK(!epi.pos, "gemm_tc2: positional-table epilogue is not supported (conv stem stays on gemm_tc)");
  BW_CHECK(epi.row_stride % 8 == 0 && epi.batch_stride % 8 == 0 && epi.head_stride % 8 == 0, "gemm_tc2: output strides must be multiples of 8");
  GemmParams p;
  p.B = 1; p.rows = M; p.N = N; p.K = K;
  p.rows_per_item = rows_per_item > 0 ? rows_per_item : INT_MAX;
  p.fast_gelu = 1;
  p.kwrap = INT_MAX;
  p.tiles_m = (M + BM - 1) / BM;
  p.ksplit = 1; p.kper = K / BK; p.split_stride = 0;
  p.epi = epi;
  CUtensorMap tmA;
  if (int rc = make_tmap_3d_bf16(&tmA, A, 1, (uint64_t)M, (uint64_t)K, (uint64_t)K * 2, (uint64_t)M * K * 2, BM, BK)) return rc;
  int force_mode = -1;
  if (force_bn >= 1000) {  // tests: 1000 + bn = the generic (runtime-parameterised) epilogue instead of the specialised one
    force_mode = EPI_GENERIC;
    force_bn -= 1000;
  }
  int bn = force_bn;
  if (bn == 0) {
    // 256-wide tiles halve the L2 traffic per MAC; fall back to 128 when 256 does not divide N or leaves the last wave thin
    bn = (N % 256 == 0) ? 256 : 128;
    if (bn == 256) {
      const int sms = device_sms();
      const long long t256 = (long long)p.tiles_m * (N / 256);
      const long long waves = (t256 + sms - 1) / sms;
      if (t256 * 10 < waves * sms * 8) bn = 128;  // < 80 % of the last wave's slots used
    }
  }
  BW_CHECK(bn == 128 || bn == 256, "gemm_tc2: unsupported tile width %d", bn);
  BW_CHECK(N % bn == 0, "gemm_tc2: N=%d is not a multiple of the tile width %d", N, bn);
  int mode = EPI_GENERIC;
  if (epi.alpha == 1.0f) {
    if (epi.act == 1 && !epi.residual && epi.out_bf16) mode = EPI_GELU;
    else if (epi.act == 0 && epi.residual && epi.out_f32) mode = EPI_RESID;
    else if (epi.act == 0 && !epi.residual && epi.out_bf16) mode = EPI_PLAIN;
  }
  if (force_mode >= 0) mode = force_mode;
#define BW_TC2_CASE(BNV, MODEV) \
  if (bn == BNV && mode == MODEV) return launch_tc<BNV, MODEV>(st, tmA, W, p);
  BW_TC2_CASE(256, EPI_GENERIC) BW_TC2_CASE(256, EPI_GELU) BW_TC2_CASE(256, EPI_RESID) BW_TC2_CASE(256, EPI_PLAIN)
  BW_TC2_CASE(128, EPI_GENERIC) BW_TC2_CASE(128, EPI_GELU) BW_TC2_CASE(128, EPI_RESID) BW_TC2_CASE(128, EPI_PLAIN)
#undef BW_TC2_CASE
  BW_CHECK(false, "gemm_tc2: no kernel for bn=%d mode=%d", bn, mode);
}

int gemm_simt(cudaStream_t st, const GemmA& a, const bf16* W, int B, int rows, int N, int K, const GemmEpi& epi) {
  if (int rc = check_epi(epi, N)) return rc;
  GemmParams p;
  p.B = B; p.rows = rows; p.N = N; p.K = K;
  p.kwrap = a.kwrap >= K ? INT_MAX : a.kwrap;
  p.tiles_m = (rows + 15) / 16;
  p.ksplit = 1; p.kper = 0; p.split_stride = 0;
  p.epi = epi;
  dim3 grid((N + 15) / 16, p.tiles_m * B);
  gemm_simt_kernel<<<grid, dim3(16, 16), 0, st>>>(a, W, p);
  BW_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace bw
