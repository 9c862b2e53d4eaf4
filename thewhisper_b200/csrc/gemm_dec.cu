// Weight-streaming wgmma GEMM of the batched decoder step (q_len = 1 for Q sequences): out[q, n] = sum_k X[q, k] * W[n, k].
//
// Shape of the problem: W is 3-13 MB and read once per step, X is Q x K with Q = 3..320 rows.  The step runs ~190 of these per
// token, so what matters is the LATENCY of one launch, not its peak rate: a generic kernel (128-row activation tile, 32-column weight
// tile, deep ring) walks 20-80 k-blocks per CTA, i.e. several dependent DRAM round trips.  Here the operands are swapped and K is split:
//   * the WEIGHT tile is the 128-row M side of the MMA (two consumer warpgroups of 64 rows), the activations are the N side (Q rounded
//     up to a wgmma width of 32, 64, 128 or 256): a k-block costs 16 KB of W + QB x 128 B of X, so several k-blocks fit in smem at once;
//   * grid = (N / 128) x q-tiles x ksplit with ksplit the smallest count that gives >= 64 CTAs and lets a CTA's k-blocks fit its
//     ring: every byte a CTA needs is requested by ONE thread before anything is awaited -- one DRAM round trip per launch;
//   * under programmatic dependent launch the weight boxes are requested BEFORE griddepcontrol.wait (weights do not depend on the
//     previous kernel), the activation boxes after it;
//   * split-K partial sums are written raw (fp32, [split][q][n]) and added by the consumer in a fixed order (resid_ln, the
//     attention kernels' q/k/v loads, gelu_bias): deterministic, no atomics; ksplit = 1 launches (LM head) apply bias / alpha /
//     GELU here and may write bf16.
// Epilogue: accumulator row = weight row n, column = sequence q, so for a fixed q the 8 row-groups of a warp store 8 consecutive n.
// Int8 weights (W8, a scale per row): the weight box is 128 rows x 64 one-byte codes (8 KB, TMA UINT8, unswizzled); each consumer
// warpgroup converts its 64 rows, exactly, into the 16-bit 128-byte-swizzled layout the TMA would have written, in one of two
// tiles of its own (the wgmma of k-block kb - 2 read the other), and multiplies by s[n] in the epilogue, before the partial sum is
// written: the consumers of the partial sums stay as they are.
#include <limits.h>

#include "kernels.h"

namespace BW_NS {

namespace {

constexpr int DM = 128;  // weight rows per CTA
constexpr int DK = 64;
constexpr int W_STAGE_BYTES = DM * DK * 2;  // 16 KB
constexpr int MAX_STAGES = 8;
constexpr int SMEM_BUDGET = 200 * 1024;
constexpr int THREADS = 288;  // two consumer warpgroups + one TMA producer warp
constexpr int CONSUMER_WARPS = 8;
constexpr int W8_STAGE_BYTES = DM * DK;        // 8 KB of int8 codes
constexpr int W8_DEQ_BYTES = 2 * 2 * 64 * 128;  // W8: two 16-bit tiles of 64 rows per consumer warpgroup

// named barrier of consumer warpgroup g (128 threads; barrier 0 is the CTA's)
__device__ __forceinline__ void wg_sync(int g) { asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory"); }

struct DecParams {
  int Q, N, K;
  int stages;   // ring depth (<= MAX_STAGES)
  int kper;     // k-blocks per split
  int n_store;  // columns n >= n_store are not written (weight rows that do not exist: tied LM head)
  long long split_stride;
  const float* wscale;  // W8: scale per weight row
  GemmEpi epi;  // bias / alpha / act / out_f32 / out_bf16 / row_stride (= ldo); batch/head strides unused
};

template <int QB, bool W8>
__global__ void __launch_bounds__(THREADS, 1)
gemm_dec_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmX, const DecParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int x_stage_bytes = QB * DK * 2;
  constexpr int WB = W8 ? W8_STAGE_BYTES : W_STAGE_BYTES;
  constexpr int stage_bytes = WB + ((x_stage_bytes + 1023) & ~1023);  // both operands 1024-byte aligned (128 B swizzle atoms)
  uint8_t* deq = smem + (size_t)p.stages * stage_bytes;  // W8: [buffer][warpgroup] 16-bit tiles of 64 rows
  uint64_t* bars = reinterpret_cast<uint64_t*>(deq + (W8 ? W8_DEQ_BYTES : 0));
  uint64_t* full = bars;
  uint64_t* empty = bars + MAX_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = blockIdx.x * DM;
  const int q0 = blockIdx.y * QB;
  const int nk_all = p.K / DK;
  const int kb0 = (int)blockIdx.z * p.kper;
  const int nk = min(nk_all, kb0 + p.kper) - kb0;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], CONSUMER_WARPS);
    }
    fence_mbar_init();
  }
  if (warp == CONSUMER_WARPS && lane == 0) {
    tma_prefetch_desc(&tmW);
    tma_prefetch_desc(&tmX);
  }
  __syncthreads();

  if (warp == CONSUMER_WARPS) {
    if (lane == 0) {
      const int npre = nk < p.stages ? nk : p.stages;
      for (int kb = 0; kb < npre; ++kb) {  // weights: before the programmatic-launch wait
        mbar_arrive_expect_tx(&full[kb], WB + x_stage_bytes);
        tma_load_2d(smem + (size_t)kb * stage_bytes, &tmW, &full[kb], (kb0 + kb) * DK, n0);
      }
      pdl_wait();
      pdl_launch();
      for (int kb = 0; kb < nk; ++kb) {
        const int s = kb % p.stages;
        if (kb >= npre) {
          mbar_wait_wg(&empty[s], ((kb / p.stages) & 1) ^ 1);
          mbar_arrive_expect_tx(&full[s], WB + x_stage_bytes);
          tma_load_2d(smem + (size_t)s * stage_bytes, &tmW, &full[s], (kb0 + kb) * DK, n0);
        }
        tma_load_2d(smem + (size_t)s * stage_bytes + WB, &tmX, &full[s], (kb0 + kb) * DK, q0);
      }
    }
    return;
  }
  // ---------------- consumer warpgroup g: weight rows [n0 + 64 g, +64) ----------------
  const int g = warp >> 2;
  float acc[QB / 2];
#pragma unroll
  for (int i = 0; i < QB / 2; ++i) acc[i] = 0.f;
  for (int kb = 0; kb < nk; ++kb) {
    const int s = kb % p.stages;
    mbar_wait_wg(&full[s], (kb / p.stages) & 1);
    wg_fence();
    uint8_t* st = smem + (size_t)s * stage_bytes;
    if constexpr (W8) {
      uint8_t* dst = deq + ((kb & 1) * 2 + g) * (64 * 128);
      wg_sync(g);  // every warp of the warpgroup has waited for the wgmma (k-block kb - 2) that last read dst
      const int t = threadIdx.x & 127;
#pragma unroll
      for (int j = 0; j < 2; ++j) {  // 16 codes of row rl, k in [16 c, 16 c + 16) -> 16-byte chunks 2c, 2c + 1 of the swizzled row
        const int i = t + 128 * j, rl = i >> 2, c = i & 3;
        const uint4 v = *reinterpret_cast<const uint4*>(st + (64 * g + rl) * DK + c * 16);
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
        uint32_t o[8];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          float f[4];
          unpack_s8x4(w[u], f);
          o[2 * u] = pack_bf16(f[0], f[1]);  // |q| <= 128: exact in bf16 and fp16
          o[2 * u + 1] = pack_bf16(f[2], f[3]);
        }
        uint8_t* row = dst + rl * 128;
        *reinterpret_cast<uint4*>(row + (((2 * c) ^ (rl & 7)) << 4)) = make_uint4(o[0], o[1], o[2], o[3]);
        *reinterpret_cast<uint4*>(row + (((2 * c + 1) ^ (rl & 7)) << 4)) = make_uint4(o[4], o[5], o[6], o[7]);
      }
      fence_proxy_async_smem();  // the generic-proxy writes before the wgmma (async proxy) reads them
      wg_sync(g);
      wg_fence();
      wg_kblock<QB>(acc, smem_u32(dst), smem_u32(st + WB));
    } else {
      wg_kblock<QB>(acc, smem_u32(st + g * (W_STAGE_BYTES / 2)), smem_u32(st + W_STAGE_BYTES));
    }
    wg_commit();
    wg_wait<1>();
    if (kb > 0 && lane == 0) mbar_arrive(&empty[(kb - 1) % p.stages]);
  }
  wg_wait<0>();
  wg_pin(acc);

  // ---------------- epilogue: this thread holds weight rows n and n + 8, two adjacent sequences of every 8 ----------------
  pdl_wait();
  const GemmEpi& e = p.epi;
  const int qn = min(QB, p.Q - q0);  // valid sequences of this q-tile
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int n = n0 + g * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
    if (n >= p.n_store) continue;
    const float bias = e.bias ? e.bias[n] : 0.f;
    const float sc = W8 ? p.wscale[n] : 1.f;  // (n < n_store: the tied LM head's V rows)
    const float alpha = (n < e.alpha_cols) ? e.alpha : 1.0f;
    float* of = e.out_f32 ? e.out_f32 + (long long)blockIdx.z * p.split_stride + n : nullptr;
    bf16* ob = e.out_bf16 ? e.out_bf16 + n : nullptr;
#pragma unroll
    for (int j = 0; j < QB / 8; ++j) {
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int q = 8 * j + 2 * (lane & 3) + c;
        if (q < qn) {
          float f;
          if constexpr (W8) f = (acc[4 * j + 2 * h + c] * sc + bias) * alpha;
          else f = (acc[4 * j + 2 * h + c] + bias) * alpha;
          if (e.act == 1) f = gelu_erf(f);
          const long long off = (long long)(q0 + q) * e.row_stride;
          if (of) of[off] = f;
          else ob[off] = f2e(f);
        }
      }
    }
  }
}

template <int QB, bool W8>
int launch_dec(cudaStream_t st, const CUtensorMap& tmW, const CUtensorMap& tmX, const DecParams& p, const DecGemmPlan& pl) {
  static size_t attr = 0;
  if (pl.smem > attr) {
    BW_CUDA_OK(cudaFuncSetAttribute(gemm_dec_kernel<QB, W8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.smem));
    attr = pl.smem;
  }
  dim3 grid((p.N + DM - 1) / DM, pl.q_tiles, pl.ksplit);
  BW_CUDA_OK(launch_k(gemm_dec_kernel<QB, W8>, grid, dim3(THREADS), pl.smem, st, tmW, tmX, p));
  return 0;
}

template <bool W8>
int launch_dec_q(cudaStream_t st, const CUtensorMap& tmW, const CUtensorMap& tmX, const DecParams& p, const DecGemmPlan& pl) {
  switch (pl.QB) {
    case 32: return launch_dec<32, W8>(st, tmW, tmX, p, pl);
    case 64: return launch_dec<64, W8>(st, tmW, tmX, p, pl);
    case 128: return launch_dec<128, W8>(st, tmW, tmX, p, pl);
    default: return launch_dec<256, W8>(st, tmW, tmX, p, pl);
  }
}

// h[q, n] = bf16( GELU( sum_s part[s][q][n] + bias[n] ) ): the consumer of fc1's split-K partial sums (operand of fc2)
__global__ void __launch_bounds__(256) gelu_bias_kernel(const float* __restrict__ part, int nsplit, long long split_stride,
                                                        const float* __restrict__ bias, bf16* __restrict__ h, long long total, int N) {
  pdl_wait();
  pdl_launch();
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (i >= total) return;
  float4 a = *reinterpret_cast<const float4*>(part + i);
  for (int s = 1; s < nsplit; ++s) {
    const float4 b = *reinterpret_cast<const float4*>(part + (long long)s * split_stride + i);
    a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
  }
  const int n = (int)(i % N);
  const float4 bb = *reinterpret_cast<const float4*>(bias + n);
  uint2 w;
  w.x = pack_bf16(gelu_erf(a.x + bb.x), gelu_erf(a.y + bb.y));
  w.y = pack_bf16(gelu_erf(a.z + bb.z), gelu_erf(a.w + bb.w));
  *reinterpret_cast<uint2*>(h + i) = w;
}

}  // namespace

// Plan of one decoder projection: q-tiling, ring depth and split count.  want_split = false forces ksplit = 1 (epilogue applies
// bias / activation itself).  w8: int8 weights (8 KB weight stages, plus the warpgroups' 16-bit tiles).
DecGemmPlan gemm_dec_plan(int Q, int N, int K, int num_sms, bool want_split, bool w8) {
  DecGemmPlan pl;
  pl.q_tiles = (Q + 255) / 256;
  const int per_tile = (Q + pl.q_tiles - 1) / pl.q_tiles;
  pl.QB = 32;  // a wgmma width: 32, 64, 128 or 256
  while (pl.QB < per_tile) pl.QB <<= 1;
  const int stage_bytes = (w8 ? W8_STAGE_BYTES : W_STAGE_BYTES) + ((pl.QB * DK * 2 + 1023) & ~1023);
  const int extra = w8 ? W8_DEQ_BYTES : 0;
  pl.stages = (SMEM_BUDGET - extra) / stage_bytes;
  if (pl.stages > MAX_STAGES) pl.stages = MAX_STAGES;
  const int nk = K / DK;
  const int n_tiles = (N + DM - 1) / DM;
  // as few splits as give (a) a CTA all of its k-blocks in one ring pass and (b) >= 64 CTAs: every extra split is another partial-sum
  // row the consumer has to read
  int ks = 1;
  if (want_split) {
    const int ctas1 = n_tiles * pl.q_tiles;
    const int ks_ring = (nk + pl.stages - 1) / pl.stages;
    const int ks_fill = (64 + ctas1 - 1) / ctas1;
    ks = ks_ring > ks_fill ? ks_ring : ks_fill;
    const int ks_max = num_sms / ctas1 > 0 ? num_sms / ctas1 : 1;
    if (ks > ks_max) ks = ks_max;
    if (ks > nk) ks = nk;
    if (ks < 1) ks = 1;
  }
  pl.kper = (nk + ks - 1) / ks;
  pl.ksplit = (nk + pl.kper - 1) / pl.kper;
  pl.smem = (size_t)pl.stages * stage_bytes + extra + 1024 + 256;
  return pl;
}

int gemm_dec(cudaStream_t st, const bf16* X, const void* W, const float* wscale, int Q, int N, int K, int n_valid, const GemmEpi& epi,
             const DecGemmPlan& pl, long long split_stride) {
  BW_CHECK(K % DK == 0 && K >= DK, "gemm_dec: K=%d must be a multiple of 64", K);
  BW_CHECK((epi.out_f32 != nullptr) != (epi.out_bf16 != nullptr), "gemm_dec: exactly one of out_f32/out_bf16 must be set");
  BW_CHECK(pl.ksplit == 1 || (epi.out_f32 && !epi.bias && epi.act == 0 && epi.alpha == 1.0f), "gemm_dec: split-K writes raw fp32 partial sums");
  BW_CHECK((pl.QB == 32 || pl.QB == 64 || pl.QB == 128 || pl.QB == 256) && pl.stages >= 2 && pl.stages <= MAX_STAGES,
           "gemm_dec: bad plan (QB=%d stages=%d)", pl.QB, pl.stages);
  CUtensorMap tmW, tmX;
  const int w_rows = (n_valid > 0 && n_valid < N) ? n_valid : N;
  if (wscale) {
    if (int rc = make_tmap_2d_u8(&tmW, W, (uint64_t)w_rows, (uint64_t)K, (uint64_t)K, DM, DK)) return rc;
  } else {
    if (int rc = make_tmap_2d_bf16(&tmW, W, (uint64_t)w_rows, (uint64_t)K, (uint64_t)K * 2, DM, DK)) return rc;
  }
  if (int rc = make_tmap_2d_bf16(&tmX, X, (uint64_t)Q, (uint64_t)K, (uint64_t)K * 2, (uint32_t)pl.QB, DK)) return rc;
  DecParams p;
  p.Q = Q; p.N = N; p.K = K; p.stages = pl.stages; p.kper = pl.kper; p.n_store = w_rows; p.split_stride = split_stride;
  p.epi = epi;
  p.wscale = wscale;
  return wscale ? launch_dec_q<true>(st, tmW, tmX, p, pl) : launch_dec_q<false>(st, tmW, tmX, p, pl);
}

int launch_gelu_bias(cudaStream_t st, const float* part, int nsplit, long long split_stride, const float* bias, bf16* h, int Q, int N) {
  BW_CHECK(N % 4 == 0, "gelu_bias: N=%d must be a multiple of 4", N);
  const long long total = (long long)Q * N;
  const int blocks = (int)((total / 4 + 255) / 256);
  BW_CUDA_OK(launch_k(gelu_bias_kernel, dim3(blocks), dim3(256), 0, st, part, nsplit, split_stride, bias, h, total, N));
  return 0;
}

}  // namespace bw
