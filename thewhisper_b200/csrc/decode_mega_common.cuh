// Building blocks shared by the persistent decoder-step kernels (decode_mega.cu and its second / third generation):
// launch geometry, memory-ordering and TMA primitives, the row-per-warp dot products, the in-smem attention of one work
// item, the transposing warp reduction and the shared-memory plan.  Everything is __forceinline__ device code (or inline
// host code): including this header adds no symbols and does not change the code of a kernel that used the same text.
#pragma once
#include <math.h>

#include "decode.cuh"
#include "kernels.h"

namespace BW_NS {
namespace mega {

constexpr int MT = 384;        // threads per CTA (12 warps: <= 170 registers per thread)
constexpr int MW = MT / 32;    // warps per CTA
constexpr int RMAX = 4;        // weight rows per warp in a GEMV phase: row r is finished by lanes [8r, 8r + MB)
constexpr int DMA_T = MT - 32;  // first lane of the last warp: issues every TMA operation (it takes no part in x staging)
constexpr int KG = MT / 8;     // key groups of 8 lanes in the attention phases
constexpr int MAXKEYS = 448;   // self-attention keys held in smem (Tmax)
constexpr int XKMAX = 256;     // cross-attention keys per work item held in smem
constexpr int MAXD = 1280;
constexpr int ATT_OFF = 32 * 1024;  // attention scratch starts here inside the pool (above the R=1 weight slabs)

__device__ __forceinline__ void unpack8m(const uint4& u, float (&f)[8]) {
  float2 t;
  t = unpack_bf16(u.x); f[0] = t.x; f[1] = t.y;
  t = unpack_bf16(u.y); f[2] = t.x; f[3] = t.y;
  t = unpack_bf16(u.z); f[4] = t.x; f[5] = t.y;
  t = unpack_bf16(u.w); f[6] = t.x; f[7] = t.y;
}
__device__ __forceinline__ void cp_async16m(void* smem_dst, const void* gmem_src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_allm() { asm volatile("cp.async.wait_all;" ::: "memory"); }
// TMA bulk copy global -> this CTA's smem, completion counted in bytes on an mbarrier (16-byte aligned, size % 16 == 0)
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_add(unsigned* p, unsigned v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned atom_acq_rel_add(unsigned* p, unsigned v) {
  unsigned old;
  asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
  return old;
}
__device__ __forceinline__ long long global_ns() {
  long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

// W: rows of K elements of ESZ bytes (2: the engine's 16-bit type, 1: int8 codes)
template <int ESZ>
__device__ __forceinline__ void issue_rows(uint8_t* slab, uint64_t* bar, const uint8_t* W, int K, int R, int n, int N, int lane) {
  if (lane == 0) {
    const uint32_t row_bytes = (uint32_t)K * ESZ;
    mbar_arrive_expect_tx(bar, row_bytes * R);
    for (int r = 0; r < R; ++r) {
      const int row = min(n + r, N - 1);
      if constexpr (ESZ == 2) bulk_g2s(slab + (size_t)r * row_bytes, reinterpret_cast<const bf16*>(W) + (long long)row * K, row_bytes, bar);
      else bulk_g2s(slab + (size_t)r * row_bytes, W + (long long)row * K, row_bytes, bar);
    }
  }
}

// DRAM -> L2 only (no smem, no completion): the cross-attention K/V of a layer, ahead of its bulk load
__device__ __forceinline__ void l2_prefetch(const void* p, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}
// W8: int8 rows -- a lane reads 4 codes (4 B) at the same k0, so 32 lanes read 128 contiguous bytes (conflict-free)
template <int MB, int R, bool W8>
__device__ __forceinline__ void dot_chunk(const uint8_t* slab, const float* xs, int K, int k0, bool hi, float (&s)[R][MB]) {
  float4 x0[MB], x1[MB];
#pragma unroll
  for (int m = 0; m < MB; ++m) {
    x0[m] = *reinterpret_cast<const float4*>(&xs[m * K + k0]);
    x1[m] = hi ? *reinterpret_cast<const float4*>(&xs[m * K + k0 + 128]) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
#pragma unroll
  for (int r = 0; r < R; ++r) {
    float2 a0, a1, c0, c1;
    if constexpr (W8) {
      const uint32_t wa = *reinterpret_cast<const uint32_t*>(slab + (size_t)r * K + k0);
      const uint32_t wc = hi ? *reinterpret_cast<const uint32_t*>(slab + (size_t)r * K + k0 + 128) : 0u;
      float fa[4], fc[4];
      unpack_s8x4(wa, fa);
      unpack_s8x4(wc, fc);
      a0 = make_float2(fa[0], fa[1]); a1 = make_float2(fa[2], fa[3]); c0 = make_float2(fc[0], fc[1]); c1 = make_float2(fc[2], fc[3]);
    } else {
      const uint2 wa = *reinterpret_cast<const uint2*>(slab + ((size_t)r * K + k0) * 2);
      const uint2 wc = hi ? *reinterpret_cast<const uint2*>(slab + ((size_t)r * K + k0 + 128) * 2) : make_uint2(0u, 0u);
      a0 = unpack_bf16(wa.x); a1 = unpack_bf16(wa.y); c0 = unpack_bf16(wc.x); c1 = unpack_bf16(wc.y);
    }
#pragma unroll
    for (int m = 0; m < MB; ++m) {
      float t = s[r][m], u = 0.f;
      t = fmaf(a0.x, x0[m].x, t); u = fmaf(c0.x, x1[m].x, u);
      t = fmaf(a0.y, x0[m].y, t); u = fmaf(c0.y, x1[m].y, u);
      t = fmaf(a1.x, x0[m].z, t); u = fmaf(c1.x, x1[m].z, u);
      t = fmaf(a1.y, x0[m].w, t); u = fmaf(c1.y, x1[m].w, u);
      s[r][m] = t + u;
    }
  }
}

// The full 256-element chunks run branch-free (unrolled by 5 so the loads of several chunks are in flight together: with a
// guard per chunk the compiler serialised load -> convert -> FMA chunk by chunk, ~120 cycles each); a ragged tail
// (K % 256 != 0: only the small test models) takes the guarded path.
template <int MB, int R, bool W8>
__device__ __forceinline__ void dot_rows(const uint8_t* slab, const float* xs, int K, float (&acc)[RMAX][MB], int lane) {
  float s[R][MB];
#pragma unroll
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int m = 0; m < MB; ++m) s[r][m] = 0.f;
  const int nfull = K >> 8;
  int k0 = lane * 4;
#pragma unroll 5
  for (int c = 0; c < nfull; ++c, k0 += 256) dot_chunk<MB, R, W8>(slab, xs, K, k0, true, s);
  if (k0 < K) dot_chunk<MB, R, W8>(slab, xs, K, k0, (k0 + 128) < K, s);
#pragma unroll
  for (int r = 0; r < RMAX; ++r)
#pragma unroll
    for (int m = 0; m < MB; ++m) acc[r][m] = (r < R) ? warp_sum(s[r < R ? r : 0][m]) : 0.f;
}

// v[j] = this lane's partial sum of row j (NV = 4, 16 or 32 rows).  Halving stages with masks 16, 8, ...: a lane keeps the
// half of the rows selected by its own bit and hands the other half to its partner; the remaining stages are plain
// xor-sums.  Afterwards every lane holds the warp total of row (lane >> (5 - log2 NV)).
template <int NV>
__device__ __forceinline__ float treduce(float (&v)[NV], int lane) {
  int n = NV;
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) {
    if (n > 1) {
      const int h = n >> 1;
      const bool up = (lane & m) != 0;
#pragma unroll
      for (int j = 0; j < NV / 2; ++j) {
        if (j < h) {
          const float keep = up ? v[j + h] : v[j];
          const float send = up ? v[j] : v[j + h];
          v[j] = keep + __shfl_xor_sync(0xffffffffu, send, m);
        }
      }
      n = h;
    } else {
      v[0] += __shfl_xor_sync(0xffffffffu, v[0], m);
    }
  }
  return v[0];
}

// Scores, softmax numerators and the un-normalised P.V of one work item whose n <= NJ*KG keys sit in smem (rows of 128 B).
// Key group g (8 lanes, 8 dims each) owns keys g, g + KG, ...: its scores stay in registers, all smem reads of a pass are
// issued together (fully unrolled, predicated), and there are two CTA barriers in all: one for the maximum, one for the
// final fold of (sum, 64 outputs) across warps.  Returns max / sum / (threads < 64) the output sums.
// red: [2][MW] floats, redo: [MW][64 + 8] floats.
template <int NJ>
__device__ __forceinline__ void attend_smem(const uint8_t* sK, const uint8_t* sV, float* redo, float* red, const float (&qv)[8], int n,
                                            float* score_out, float& mx_out, float& sum_out, float& ov_out, long long* mk = nullptr) {
  const int grp = threadIdx.x >> 3, sub = threadIdx.x & 7;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // separate passes so that the NJ independent chains overlap: loads + FMAs of all keys, then the three shuffle stages
  // across all keys (one dependent shuffle chain per key cost ~150 cycles per key when interleaved with the FMAs)
  float d[NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int kk = grp + j * KG;
    float t0 = 0.f, t1 = 0.f;
    if (kk < n) {
      float kf[8];
      unpack8m(*reinterpret_cast<const uint4*>(sK + kk * 128 + sub * 16), kf);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        t0 = fmaf(qv[i], kf[i], t0);
        t1 = fmaf(qv[i + 4], kf[i + 4], t1);
      }
    }
    d[j] = t0 + t1;
  }
#pragma unroll
  for (int st = 1; st < 8; st <<= 1) {
#pragma unroll
    for (int j = 0; j < NJ; ++j) d[j] += __shfl_xor_sync(0xffffffffu, d[j], st);
  }
  float lmax = -INFINITY;
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int kk = grp + j * KG;
    if (kk < n) {
      lmax = fmaxf(lmax, d[j]);
      if (score_out && sub == 0) score_out[kk] = d[j];
    }
  }
  lmax = warp_max(lmax);
  if (mk && threadIdx.x == 0) { mk[1] = global_ns(); mk[3] = clock64(); }
  if (lane == 0) red[warp] = lmax;
  __syncthreads();
  float mx = red[0];
#pragma unroll
  for (int w = 1; w < MW; ++w) mx = fmaxf(mx, red[w]);
  float acc[8], lsum = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  {  // one exp per key (not one per lane): lane (j & 7) of the group exponentiates key j, the group shares it by shuffle
    float mine = 0.f, mine2 = 0.f;
#pragma unroll
    for (int j = 0; j < NJ; ++j)
      if ((j & 7) == sub) {
        if (j < 8) mine = d[j];
        else mine2 = d[j];
      }
    mine = __expf(mine - mx);
    if (NJ > 8) mine2 = __expf(mine2 - mx);
    const int gl = lane & 24;  // first lane of this group of 8
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const float e = __shfl_sync(0xffffffffu, j < 8 ? mine : mine2, gl + (j & 7));
      d[j] = (grp + j * KG < n) ? e : 0.f;
    }
  }
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int kk = grp + j * KG;
    if (kk < n) {
      lsum += d[j];
      float vf[8];
      unpack8m(*reinterpret_cast<const uint4*>(sV + kk * 128 + sub * 16), vf);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = fmaf(d[j], vf[i], acc[i]);
    }
  }
  // fold the 4 key groups of a warp with shuffles (lanes with equal sub), then the 12 warp partials through smem
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], 8);
    acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], 16);
  }
  lsum += __shfl_xor_sync(0xffffffffu, lsum, 8);  // (all 8 lanes of a group hold the same sum)
  lsum += __shfl_xor_sync(0xffffffffu, lsum, 16);
  if (lane < 8) {
#pragma unroll
    for (int i = 0; i < 8; ++i) redo[warp * 72 + lane * 8 + i] = acc[i];
    if (lane == 0) redo[warp * 72 + 64] = lsum;
  }
  __syncthreads();
  float ov = 0.f, ls = 0.f;
#pragma unroll
  for (int w = 0; w < MW; ++w) ls += redo[w * 72 + 64];
  if (threadIdx.x < 64) {
#pragma unroll
    for (int w = 0; w < MW; ++w) ov += redo[w * 72 + threadIdx.x];
  }
  mx_out = mx;
  sum_out = ls;
  ov_out = ov;
}

// smem plan: returns the dynamic smem bytes (0: does not fit in `limit`) and the offset of slab region 0 (0: single-buffered,
// everything at the pool's start).  limit = the device's opt-in shared memory per block less the kernel's static smem (layer
// table, barriers): on 132 SMs the double-buffered plan for large-v3 at Q = 1 fits with a few hundred bytes to spare, so the
// limit is taken from the device and the compiled kernel, not estimated.  esz: bytes per weight element (2, or 1 for int8).
// The overlap rule does not depend on esz: during an attention phase only the out-proj / cross out-proj slabs (K = D) of
// region 1 are live, and they stay below ATT_OFF (the launcher checks it for the element size); the attention scratch itself
// does not shrink with the weights, so with 1-byte rows it, not the slab regions, bounds the pool.
inline size_t mega_smem_plan(int mb, int D, int ffn, int num_sms, bool want_dbuf, size_t limit, int* p0_off, int esz = 2) {
  // rows of a CTA, rounded up to whole active warps: the unused rows of the last active warp are still read (and discarded)
  auto rc = [&](int n) {
    const int rows = (n + num_sms - 1) / num_sms, R = (rows + MW - 1) / MW;
    return (size_t)((rows + R - 1) / R * R);
  };
  const size_t attn = (size_t)MAXKEYS * 256 + (size_t)(MW * 72) * sizeof(float);
  const size_t xattn = (size_t)2 * XKMAX * 128 + (size_t)(MW * 72) * sizeof(float);
  const size_t att = ATT_OFF + (attn > xattn ? attn : xattn);
  const size_t lm = (size_t)MW * 2 * 2 * D * esz;  // LM head: 2 stages of row pairs per warp
  size_t r1 = rc(D) * ffn * esz;                   // region 1: out-proj / cross out-proj (K = D), fc2 (K = ffn)
  if (rc(D) * D * esz > r1) r1 = rc(D) * D * esz;
  size_t r0 = rc(3 * D) * D * esz;                 // region 0: QKV, cross-q, fc1
  if (rc(ffn) * D * esz > r0) r0 = rc(ffn) * D * esz;
  if (rc(D) * D * esz > r0) r0 = rc(D) * D * esz;
  const size_t fixed = 64 * sizeof(float) + (size_t)mb * ffn * sizeof(float) + 128;
  auto mx = [](size_t a, size_t b) { return a > b ? a : b; };
  const size_t off = (r1 + 127) / 128 * 128;
  const size_t pool_d = mx(mx(off + r0, att), lm);
  if (want_dbuf && fixed + pool_d <= limit) {
    *p0_off = (int)off;
    return fixed + pool_d;
  }
  *p0_off = 0;
  const size_t single = fixed + mx(mx(mx(r0, r1), att), lm);
  return single <= limit ? single : 0;
}

}  // namespace mega
}  // namespace bw
