// Prompt prefill of the decoder: the teacher-forced positions t0 .. t0 + n - 1 of all Q sequences in one pass of R = Q * n rows
// (row r = q * n + i is sequence q at position t0 + i).  The projections are the batched step's gemm_dec launches at Q' = R; this
// file holds what a one-row step does not have:
//   * the embedding gather at per-row positions;
//   * the split-K sum of a q / qkv projection, which rounds q / 8 to the 16-bit operand of the attention kernels and, for the self
//     projection, appends the rows' K / V to the cache (a kernel of its own: every K / V row of the pass is in the cache before any
//     query tile reads it);
//   * a wgmma flash-attention kernel (head_dim 64) over 64-row query tiles, either causal over the cache rows [0, t] of the row's
//     own sequence, or over the S encoder positions of the row's audio (its G beams x n positions share one audio's cross K/V).
#include <math.h>

#include "decode.cuh"
#include "kernels.h"

namespace BW_NS {

namespace {

constexpr int DH = 64;
constexpr int TQ = 64;                   // query rows per CTA (one consumer warpgroup)
constexpr int TK = 64;                   // keys per tile
constexpr int TILE_BYTES = 64 * DH * 2;  // 8 KB: a Q, K or V tile (64 rows of 128 B, 128-byte swizzle)
constexpr int KV_STAGES = 4;
constexpr int PF_SMEM = TILE_BYTES * (1 + 2 * KV_STAGES) + 1024 /*align slack*/ + 256 /*barriers*/;
constexpr int PF_THREADS = 160;  // one consumer warpgroup + one TMA producer warp
constexpr int CONSUMER_WARPS = 4;
constexpr float LOG2E = 1.4426950408889634f;

// x[r] = E[tok] + P[t] (16-bit rows) or Es[tok] * E[tok] + P[t] (int8 rows): the arithmetic of embed_kernel / embed_s8_kernel
template <bool W8>
__global__ void prefill_embed_kernel(const void* __restrict__ E, const float* __restrict__ Es, const float* __restrict__ P,
                                     const int* __restrict__ tokens, float* __restrict__ x, int D, int Tmax, int n, int t0) {
  const int r = blockIdx.x, q = r / n, t = t0 + r % n;
  const int tok = tokens[q * Tmax + t];
  if constexpr (W8) {
    const int8_t* e = static_cast<const int8_t*>(E) + (long long)tok * D;
    const float s = Es[tok];
    for (int d = threadIdx.x; d < D; d += blockDim.x) x[(long long)r * D + d] = s * (float)e[d] + P[(long long)t * D + d];
  } else {
    const bf16* e = static_cast<const bf16*>(E) + (long long)tok * D;
    for (int d = threadIdx.x; d < D; d += blockDim.x) x[(long long)r * D + d] = e2f(e[d]) + P[(long long)t * D + d];
  }
}

// v = sum_s part[s][r][c] (s ascending) + bias[c].  Columns [0, D): q / 8 -> qout (16-bit); with kc, columns [D, 2D) / [2D, 3D) are
// the K / V rows of the row's (sequence, position), rounded to the element type and written to the cache [Q][Tmax][D].
__global__ void prefill_proj_sum_kernel(const float* __restrict__ part, int nsplit, long long split_stride, const float* __restrict__ bias,
                                        int N, int D, bf16* __restrict__ qout, bf16* __restrict__ kc, bf16* __restrict__ vc, int n, int t0,
                                        int Tmax) {
  const int r = blockIdx.x, q = r / n, t = t0 + r % n;
  const long long cache_row = ((long long)q * Tmax + t) * D;
  for (int c = threadIdx.x; c < N; c += blockDim.x) {
    const float* p = part + (long long)r * N + c;
    float v = p[0];
    for (int s = 1; s < nsplit; ++s) v += p[(long long)s * split_stride];
    v += bias[c];
    if (c < D) {
      if (qout) qout[(long long)r * D + c] = f2e(v * 0.125f);
    } else if (c < 2 * D) {
      kc[cache_row + c - D] = f2e(v);
    } else {
      vc[cache_row + c - 2 * D] = f2e(v);
    }
  }
}

__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
          smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

struct PfAttnParams {
  int rows;       // query rows per group: n (causal: one sequence) or G * n (cross: one audio)
  int n, t0;      // positions per pass, first position
  int S;          // cross: encoder positions
  int H, D;
  float scale_log2e;
  bf16* out;      // [R][D]
  const int* k0;  // causal: key start per sequence [Q] or null (keys below it are absent and never loaded)
};

// One CTA = 64 query rows of one (group, head).  Group z is sequence z (CAUSAL: keys = cache rows [0, t] of that sequence, a 3-D map
// [Q][t0 + n][D] so that rows past the pass read as zeros) or audio z (keys = its S encoder positions, a 3-D map [A * H][S][64]).
// Query tiles may run past their group into the next group's rows (or the map's zero fill): those rows are computed and not stored.
// With a key start k0 (causal), key tiles start at row k0 of the sequence: the rows below it are never loaded, so whatever they hold
// (left padding) cannot reach a valid row; a row with no visible key (t0 + i < k0) writes zeros.
template <bool CAUSAL>
__global__ void __launch_bounds__(PF_THREADS, 1)
prefill_attn_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                    const PfAttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + TILE_BYTES;
  uint8_t* sV = sK + KV_STAGES * TILE_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + KV_STAGES * TILE_BYTES);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;
  uint64_t* kv_empty = bars + 1 + KV_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i0 = blockIdx.x * TQ, h = blockIdx.y, z = blockIdx.z;
  // keys this tile needs: causal, up to the position of its last row in the group; cross, all S
  const int last = min(i0 + TQ, p.rows) - 1;
  const int kstart = (CAUSAL && p.k0) ? p.k0[z] : 0;
  const int n_keys = CAUSAL ? p.t0 + last + 1 - kstart : p.S;
  const int NT = n_keys > 0 ? (n_keys + TK - 1) / TK : 0;

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int i = 0; i < KV_STAGES; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], CONSUMER_WARPS);
    }
    fence_mbar_init();
  }
  if (warp == CONSUMER_WARPS && lane == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
  }
  __syncthreads();

  if (warp == CONSUMER_WARPS) {
    if (lane == 0) {
      mbar_arrive_expect_tx(q_full, TILE_BYTES);
      tma_load_2d(sQ, &tmQ, q_full, h * DH, z * p.rows + i0);
      for (int j = 0; j < NT; ++j) {
        const int s = j % KV_STAGES;
        mbar_wait_wg(&kv_empty[s], ((j / KV_STAGES) & 1) ^ 1);
        mbar_arrive_expect_tx(&kv_full[s], 2 * TILE_BYTES);
        if (CAUSAL) {
          tma_load_3d(sK + s * TILE_BYTES, &tmK, &kv_full[s], h * DH, kstart + j * TK, z);
          tma_load_3d(sV + s * TILE_BYTES, &tmV, &kv_full[s], h * DH, kstart + j * TK, z);
        } else {
          tma_load_3d(sK + s * TILE_BYTES, &tmK, &kv_full[s], 0, j * TK, z * p.H + h);
          tma_load_3d(sV + s * TILE_BYTES, &tmV, &kv_full[s], 0, j * TK, z * p.H + h);
        }
      }
    }
    return;
  }

  // ---------------- consumer warpgroup: this thread holds query rows r and r + 8 of the tile ----------------
  const int r = warp * 16 + (lane >> 2);
  const uint64_t qd = wg_desc_sw128(smem_u32(sQ));
  // causal: a key is visible to row i iff key <= t0 + (i mod n); rows of the next group are garbage either way
  int lim[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) lim[hh] = CAUSAL ? p.t0 + (i0 + r + 8 * hh) % p.n : p.S - 1;
  float o[DH / 2];
#pragma unroll
  for (int i = 0; i < DH / 2; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  mbar_wait_wg(q_full, 0);
  for (int j = 0; j < NT; ++j) {
    const int s = j % KV_STAGES;
    mbar_wait_wg(&kv_full[s], (j / KV_STAGES) & 1);
    float sc[TK / 2];
#pragma unroll
    for (int i = 0; i < TK / 2; ++i) sc[i] = 0.f;
    wg_fence();
    {
      const uint64_t kd = wg_desc_sw128(smem_u32(sK + s * TILE_BYTES));
#pragma unroll
      for (int k = 0; k < DH / 16; ++k) Wgmma<TK>::template ss<0>(sc, qd + 2 * k, kd + 2 * k, 1u);
    }
    wg_commit();
    wg_wait<0>();
    wg_pin(sc);
    const int key0 = kstart + j * TK;
    if (key0 + TK - 1 > min(lim[0], lim[1])) {
#pragma unroll
      for (int jj = 0; jj < TK / 8; ++jj)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int key = key0 + 8 * jj + 2 * (lane & 3) + c;
          if (key > lim[0]) sc[4 * jj + c] = -INFINITY;
          if (key > lim[1]) sc[4 * jj + 2 + c] = -INFINITY;
        }
    }
    float alpha[2], mb[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float t = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < TK / 8; ++jj) t = fmaxf(t, fmaxf(sc[4 * jj + 2 * hh], sc[4 * jj + 2 * hh + 1]));
      t = fmaxf(t, __shfl_xor_sync(0xffffffffu, t, 1));
      t = fmaxf(t, __shfl_xor_sync(0xffffffffu, t, 2));
      // finite once the row has seen a key: the first key is visible to every row at or past the key start; a row below it keeps
      // m = -inf and takes a zero reference, so that its probabilities are exactly 0 and never NaN
      const float m_new = fmaxf(m[hh], t);
      const float m_ref = m_new == -INFINITY ? 0.f : m_new;
      alpha[hh] = ex2_approx((m[hh] - m_ref) * p.scale_log2e);
      mb[hh] = m_ref * p.scale_log2e;
      m[hh] = m_new;
    }
    uint32_t pa[TK / 16][4];
    float ls[2] = {0.f, 0.f};
#pragma unroll
    for (int kk = 0; kk < TK / 16; ++kk) {
      float pf[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        pf[i] = ex2_approx(fmaf(sc[8 * kk + i], p.scale_log2e, -mb[(i >> 1) & 1]));
        ls[(i >> 1) & 1] += pf[i];
      }
      pa[kk][0] = pack_bf16(pf[0], pf[1]);
      pa[kk][1] = pack_bf16(pf[2], pf[3]);
      pa[kk][2] = pack_bf16(pf[4], pf[5]);
      pa[kk][3] = pack_bf16(pf[6], pf[7]);
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) l[hh] = l[hh] * alpha[hh] + ls[hh];
#pragma unroll
    for (int i = 0; i < DH / 2; ++i) o[i] *= alpha[(i >> 1) & 1];
    wg_fence();
#pragma unroll
    for (int kk = 0; kk < TK / 16; ++kk)  // V rows = keys, 128 B each: an MN-major operand, 16 keys = 2048 B
      Wgmma<DH>::template rs<1>(o, pa[kk], wg_desc_sw128(smem_u32(sV + s * TILE_BYTES + kk * 2048)), 1u);
    wg_commit();
    wg_wait<0>();
    wg_pin(o);
    if (lane == 0) mbar_arrive(&kv_empty[s]);
  }
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float t = l[hh];
    t += __shfl_xor_sync(0xffffffffu, t, 1);
    t += __shfl_xor_sync(0xffffffffu, t, 2);
    const float inv = t > 0.f ? 1.0f / t : 0.f;  // (t = 0: a row below its key start)
    const int i = i0 + r + 8 * hh;
    if (i < p.rows) {
      bf16* op = p.out + ((long long)(z * p.rows + i) * p.D + h * DH);
#pragma unroll
      for (int jj = 0; jj < DH / 8; ++jj)
        *reinterpret_cast<uint32_t*>(op + 8 * jj + 2 * (lane & 3)) = pack_bf16(o[4 * jj + 2 * hh] * inv, o[4 * jj + 2 * hh + 1] * inv);
    }
  }
}

template <bool CAUSAL>
int launch_pf_attn(cudaStream_t st, const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV, const PfAttnParams& p,
                   int groups) {
  static bool attr_set = false;
  if (!attr_set) {
    BW_CUDA_OK(cudaFuncSetAttribute(prefill_attn_kernel<CAUSAL>, cudaFuncAttributeMaxDynamicSharedMemorySize, PF_SMEM));
    attr_set = true;
  }
  dim3 grid((p.rows + TQ - 1) / TQ, p.H, groups);
  BW_CUDA_OK(launch_k(prefill_attn_kernel<CAUSAL>, grid, dim3(PF_THREADS), (size_t)PF_SMEM, st, tmQ, tmK, tmV, p));
  return 0;
}

}  // namespace

int launch_prefill_embed(cudaStream_t st, const void* E, const float* Es, const float* P, const int* tokens, float* x, int Q, int n, int t0,
                         int D, int Tmax) {
  if (Es) BW_CUDA_OK(launch_k(prefill_embed_kernel<true>, dim3(Q * n), dim3(256), 0, st, E, Es, P, tokens, x, D, Tmax, n, t0));
  else BW_CUDA_OK(launch_k(prefill_embed_kernel<false>, dim3(Q * n), dim3(256), 0, st, E, Es, P, tokens, x, D, Tmax, n, t0));
  return 0;
}

int launch_prefill_proj_sum(cudaStream_t st, const float* part, int nsplit, long long split_stride, const float* bias, int N, int D, int R,
                            bf16* qout, bf16* kc, bf16* vc, int n, int t0, int Tmax) {
  BW_CHECK(N == D || (N == 3 * D && kc && vc), "prefill_proj_sum: N=%d must be D, or 3D with the K / V cache", N);
  BW_CUDA_OK(launch_k(prefill_proj_sum_kernel, dim3(R), dim3(256), 0, st, part, nsplit, split_stride, bias, N, D, qout, kc, vc, n, t0, Tmax));
  return 0;
}

int launch_prefill_self_attn(cudaStream_t st, const bf16* q, const bf16* kc, const bf16* vc, bf16* out, int Q, int n, int t0, int H, int Tmax,
                             const int* k0) {
  const int D = H * DH;
  CUtensorMap tmQ, tmK, tmV;
  if (int rc = make_tmap_2d_bf16(&tmQ, q, (uint64_t)Q * n, (uint64_t)D, (uint64_t)D * 2, TQ, DH)) return rc;
  // rows past t0 + n - 1 (not written yet, or stale) read as zeros: masked scores, and zero V rows under a zero probability
  if (int rc = make_tmap_3d_bf16(&tmK, kc, (uint64_t)Q, (uint64_t)(t0 + n), (uint64_t)D, (uint64_t)D * 2, (uint64_t)Tmax * D * 2, TK, DH)) return rc;
  if (int rc = make_tmap_3d_bf16(&tmV, vc, (uint64_t)Q, (uint64_t)(t0 + n), (uint64_t)D, (uint64_t)D * 2, (uint64_t)Tmax * D * 2, TK, DH)) return rc;
  PfAttnParams p;
  p.rows = n; p.n = n; p.t0 = t0; p.S = 0; p.H = H; p.D = D; p.scale_log2e = LOG2E; p.out = out; p.k0 = k0;  // q already carries the 1/8
  return launch_pf_attn<true>(st, tmQ, tmK, tmV, p, Q);
}

int launch_prefill_cross_attn(cudaStream_t st, const bf16* q, const bf16* kc, const bf16* vc, bf16* out, int A, int G, int n, int S, int H) {
  const int D = H * DH;
  CUtensorMap tmQ, tmK, tmV;
  if (int rc = make_tmap_2d_bf16(&tmQ, q, (uint64_t)A * G * n, (uint64_t)D, (uint64_t)D * 2, TQ, DH)) return rc;
  // [A * H][S][64]: a key tile past S reads zeros, never the next head's rows
  if (int rc = make_tmap_3d_bf16(&tmK, kc, (uint64_t)A * H, (uint64_t)S, DH, DH * 2, (uint64_t)S * DH * 2, TK, DH)) return rc;
  if (int rc = make_tmap_3d_bf16(&tmV, vc, (uint64_t)A * H, (uint64_t)S, DH, DH * 2, (uint64_t)S * DH * 2, TK, DH)) return rc;
  PfAttnParams p;
  p.rows = G * n; p.n = n; p.t0 = 0; p.S = S; p.H = H; p.D = D; p.scale_log2e = LOG2E; p.out = out; p.k0 = nullptr;
  return launch_pf_attn<false>(st, tmQ, tmK, tmV, p, A);
}

}  // namespace bw
