// Encoder self-attention (non-causal, head_dim 64) as a wgmma flash kernel for sm_90a.
//
// Replaces SDPA / eager attention of TF/models/whisper/modeling_whisper.py:215-238,343-353 for the encoder
// (no mask, :637-641).  softmax(q k^T * dh^-1/2) v with fp32 scores/accumulators, bf16 operands.
//
// One CTA = 128 query rows of one (batch, head); 288 threads:
//   warps 0-7  two consumer warpgroups, 64 query rows each.  Per key tile of 128: S = Q K^T (4 x wgmma m64n128k16, Q and K from
//              smem) into registers, online max / sum over the rows (a row lives in the 4 lanes of a quad), P = exp2(...) packed to
//              bf16 in registers as the A operand of O += P V (8 x wgmma m64n64k16, A from registers); O stays in registers.
//   warp  8    TMA producer: Q once, then K / V tiles through a KV_STAGES-deep ring (mbarrier complete_tx)
// V is either the transposed copy vt [B, H, 64, Spad] (K-major operand) or, without a copy, the V columns of the qkv rows themselves
// (MN-major operand: row = key, 128 B = the head's 64 dims).
// Keys beyond S (tile overrun into the next audio's rows / TMA zero fill) are masked to -inf before the max.
#include "kernels.h"

namespace BW_NS {

namespace {

constexpr int TQ = 128;   // query rows per CTA
constexpr int TK = 128;   // keys per tile
constexpr int DH = 64;
constexpr int Q_BYTES = TQ * DH * 2;       // 16 KB
constexpr int K_BYTES = TK * DH * 2;       // 16 KB
constexpr int V_BYTES = DH * TK * 2;       // 16 KB  (V^T: two 8 KB atoms of 64 keys; direct: 128 rows of 128 B)
constexpr int KV_STAGES = 3;
constexpr int ATT_SMEM = Q_BYTES + KV_STAGES * (K_BYTES + V_BYTES) + 1024 /*align slack*/ + 256 /*barriers*/;
constexpr int THREADS = 288;
constexpr int CONSUMER_WARPS = 8;
constexpr float LOG2E = 1.4426950408889634f;

struct AttnParams {
  int B, S, H, D;
  float scale_log2e;  // dh^-1/2 * log2(e)
  bf16* out;
};

template <bool VDIRECT>
__global__ void __launch_bounds__(THREADS, 1)
attn_enc_kernel(const __grid_constant__ CUtensorMap tmQK, const __grid_constant__ CUtensorMap tmVT, const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + Q_BYTES;
  uint8_t* sV = sK + KV_STAGES * K_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + KV_STAGES * V_BYTES);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;              // [KV_STAGES]
  uint64_t* kv_empty = bars + 1 + KV_STAGES;  // [KV_STAGES]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * TQ, h = blockIdx.y, b = blockIdx.z;
  const int NT = (p.S + TK - 1) / TK;

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int i = 0; i < KV_STAGES; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], CONSUMER_WARPS);
    }
    fence_mbar_init();
  }
  if (warp == CONSUMER_WARPS && lane == 0) {
    tma_prefetch_desc(&tmQK);
    if (!VDIRECT) tma_prefetch_desc(&tmVT);
  }
  __syncthreads();
  pdl_wait();  // (programmatic dependent launch: the qkv rows are the predecessor's output)
  pdl_launch();

  if (warp == CONSUMER_WARPS) {
    // ---------------- TMA producer ----------------
    if (lane == 0) {
      const int row0 = b * p.S;
      mbar_arrive_expect_tx(q_full, Q_BYTES);
      tma_load_2d(sQ, &tmQK, q_full, h * DH, row0 + q0);
      const int vrow = (b * p.H + h) * DH;
      for (int j = 0; j < NT; ++j) {
        const int s = j % KV_STAGES;
        mbar_wait_wg(&kv_empty[s], ((j / KV_STAGES) & 1) ^ 1);
        mbar_arrive_expect_tx(&kv_full[s], K_BYTES + V_BYTES);
        tma_load_2d(sK + s * K_BYTES, &tmQK, &kv_full[s], p.D + h * DH, row0 + j * TK);
        if (VDIRECT) {
          tma_load_2d(sV + s * V_BYTES, &tmQK, &kv_full[s], 2 * p.D + h * DH, row0 + j * TK);
        } else {
          tma_load_2d(sV + s * V_BYTES, &tmVT, &kv_full[s], j * TK, vrow);
          tma_load_2d(sV + s * V_BYTES + V_BYTES / 2, &tmVT, &kv_full[s], j * TK + 64, vrow);
        }
      }
    }
    return;
  }

  // ---------------- consumer warpgroup g: query rows [q0 + 64 g, +64); this thread: rows r and r + 8 ----------------
  const int g = warp >> 2;
  const int r = g * 64 + (warp & 3) * 16 + (lane >> 2);
  const uint64_t qd = wg_desc_sw128(smem_u32(sQ + g * (Q_BYTES / 2)));
  float o[DH / 2];
#pragma unroll
  for (int i = 0; i < DH / 2; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};  // m in raw score units; l: this thread's share of the row sum
  mbar_wait_wg(q_full, 0);
  for (int j = 0; j < NT; ++j) {
    const int s = j % KV_STAGES;
    mbar_wait_wg(&kv_full[s], (j / KV_STAGES) & 1);
    float sc[TK / 2];
#pragma unroll
    for (int i = 0; i < TK / 2; ++i) sc[i] = 0.f;
    wg_fence();
    {
      const uint64_t kd = wg_desc_sw128(smem_u32(sK + s * K_BYTES));
#pragma unroll
      for (int k = 0; k < DH / 16; ++k) Wgmma<TK>::template ss<0>(sc, qd + 2 * k, kd + 2 * k, 1u);
    }
    wg_commit();
    wg_wait<0>();
    wg_pin(sc);
    const int key0 = j * TK;
    if (key0 + TK > p.S) {  // only the last key tile has keys beyond S
#pragma unroll
      for (int jj = 0; jj < TK / 8; ++jj)
#pragma unroll
        for (int c = 0; c < 2; ++c)
          if (key0 + 8 * jj + 2 * (lane & 3) + c >= p.S) sc[4 * jj + c] = sc[4 * jj + 2 + c] = -INFINITY;
    }
    float alpha[2], mb[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float t = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < TK / 8; ++jj) t = fmaxf(t, fmaxf(sc[4 * jj + 2 * hh], sc[4 * jj + 2 * hh + 1]));
      t = fmaxf(t, __shfl_xor_sync(0xffffffffu, t, 1));
      t = fmaxf(t, __shfl_xor_sync(0xffffffffu, t, 2));
      const float m_new = fmaxf(m[hh], t);                         // finite: every tile has >= 1 valid key
      alpha[hh] = ex2_approx((m[hh] - m_new) * p.scale_log2e);     // m = -inf on the first tile -> 0
      mb[hh] = m_new * p.scale_log2e;
      m[hh] = m_new;
    }
    // P = exp2(s c - m c) as the bf16 A fragments of the PV MMA: k-step kk covers keys [16 kk, 16 kk + 16) = chunks 2 kk, 2 kk + 1
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
    for (int kk = 0; kk < TK / 16; ++kk) {
      // MN-major V: 16 keys = 16 rows of 128 B;  K-major V^T: two 64-key atoms, 32 B per 16 keys inside one
      const uint64_t vd = VDIRECT ? wg_desc_sw128(smem_u32(sV + s * V_BYTES + kk * 2048))
                                  : wg_desc_sw128(smem_u32(sV + s * V_BYTES + (kk >> 2) * (V_BYTES / 2))) + 2 * (kk & 3);
      Wgmma<DH>::template rs<VDIRECT ? 1 : 0>(o, pa[kk], vd, 1u);
    }
    wg_commit();
    wg_wait<0>();
    wg_pin(o);
    if (lane == 0) mbar_arrive(&kv_empty[s]);  // this warp's reads of K(j) / V(j) are complete
  }
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float t = l[hh];
    t += __shfl_xor_sync(0xffffffffu, t, 1);
    t += __shfl_xor_sync(0xffffffffu, t, 2);
    const float inv = 1.0f / t;
    const int q = q0 + r + 8 * hh;
    if (q < p.S) {
      bf16* op = p.out + ((long long)(b * p.S + q) * p.D + h * DH);
#pragma unroll
      for (int jj = 0; jj < DH / 8; ++jj)
        *reinterpret_cast<uint32_t*>(op + 8 * jj + 2 * (lane & 3)) = pack_bf16(o[4 * jj + 2 * hh] * inv, o[4 * jj + 2 * hh + 1] * inv);
    }
  }
}

template <bool VDIRECT>
int launch_attn(cudaStream_t st, const CUtensorMap& tmQK, const CUtensorMap& tmVT, const AttnParams& p) {
  static bool attr_set = false;
  if (!attr_set) {
    BW_CUDA_OK(cudaFuncSetAttribute(attn_enc_kernel<VDIRECT>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_SMEM));
    attr_set = true;
  }
  dim3 grid((p.S + TQ - 1) / TQ, p.H, p.B);
  BW_CUDA_OK(launch_k(attn_enc_kernel<VDIRECT>, grid, dim3(THREADS), (size_t)ATT_SMEM, st, tmQK, tmVT, p));
  return 0;
}

// CUDA-core sibling: one block per (query, head, batch); scores staged in smem.  Comparator / bring-up only.
__global__ void attn_enc_simt_kernel(const bf16* __restrict__ qkv, bf16* __restrict__ out, int S, int H, int D, float scale) {
  extern __shared__ float sc[];  // S scores
  __shared__ float qs[DH];
  __shared__ float red[32];
  const int q = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const bf16* base = qkv + (long long)b * S * 3 * D;
  if (threadIdx.x < DH) qs[threadIdx.x] = e2f(base[(long long)q * 3 * D + h * DH + threadIdx.x]);
  __syncthreads();
  float lmax = -INFINITY;
  for (int k = threadIdx.x; k < S; k += blockDim.x) {
    const bf16* kp = base + (long long)k * 3 * D + D + h * DH;
    float a = 0.f;
    for (int d = 0; d < DH; ++d) a = fmaf(qs[d], e2f(kp[d]), a);
    a *= scale;
    sc[k] = a;
    lmax = fmaxf(lmax, a);
  }
  lmax = warp_max(lmax);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = lmax;
  __syncthreads();
  float mx = -INFINITY;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float lsum = 0.f;
  for (int k = threadIdx.x; k < S; k += blockDim.x) {
    const float e = expf(sc[k] - mx);
    sc[k] = e;
    lsum += e;
  }
  lsum = warp_sum(lsum);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = lsum;
  __syncthreads();
  float tot = 0.f;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) tot += red[i];
  if (threadIdx.x < DH) {
    float a = 0.f;
    for (int k = 0; k < S; ++k) a = fmaf(sc[k], e2f(base[(long long)k * 3 * D + 2 * D + h * DH + threadIdx.x]), a);
    out[((long long)(b * S + q)) * D + h * DH + threadIdx.x] = f2e(a / tot);
  }
}

// V slice of qkv [B*S, 3D] -> vt [B, H, 64, Spad] (keys contiguous): the K-major B operand of the PV MMA.
__global__ void transpose_v_kernel(const bf16* __restrict__ qkv, bf16* __restrict__ vt, int S, int Spad, int H, int D) {
  __shared__ bf16 tile[64][DH + 2];
  const int s0 = blockIdx.x * 64, h = blockIdx.y, b = blockIdx.z;
  for (int i = threadIdx.x; i < 64 * DH; i += blockDim.x) {
    const int s = i / DH, d = i % DH;
    tile[s][d] = (s0 + s < S) ? qkv[((long long)(b * S + s0 + s)) * 3 * D + 2 * D + h * DH + d] : f2e(0.f);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 64 * DH; i += blockDim.x) {
    const int d = i / 64, s = i % 64;
    if (s0 + s < Spad) vt[(((long long)b * H + h) * DH + d) * Spad + s0 + s] = tile[s][d];
  }
}

}  // namespace

// vt == nullptr: no transposed copy of V, the kernel reads V tiles from the qkv rows as an MN-major operand
int attn_enc_tc(cudaStream_t st, const bf16* qkv, const bf16* vt, bf16* out, int B, int S, int Spad, int H) {
  const int D = H * DH;
  BW_CHECK(vt == nullptr || (Spad % 8 == 0 && Spad >= S), "attn_enc: Spad=%d must be >= S and a multiple of 8", Spad);
  CUtensorMap tmQK, tmVT;
  if (int rc = make_tmap_2d_bf16(&tmQK, qkv, (uint64_t)B * S, (uint64_t)3 * D, (uint64_t)3 * D * 2, TQ, DH)) return rc;
  if (vt) {
    if (int rc = make_tmap_2d_bf16(&tmVT, vt, (uint64_t)B * H * DH, (uint64_t)Spad, (uint64_t)Spad * 2, DH, 64)) return rc;
  } else {
    tmVT = tmQK;
  }
  AttnParams p;
  p.B = B; p.S = S; p.H = H; p.D = D;
  p.scale_log2e = 0.125f * LOG2E;
  p.out = out;
  return vt ? launch_attn<false>(st, tmQK, tmVT, p) : launch_attn<true>(st, tmQK, tmVT, p);
}

int attn_enc_simt(cudaStream_t st, const bf16* qkv, bf16* out, int B, int S, int H) {
  const int D = H * DH;
  dim3 grid(S, H, B);
  attn_enc_simt_kernel<<<grid, 128, S * sizeof(float), st>>>(qkv, out, S, H, D, 0.125f);
  BW_CUDA_OK(cudaGetLastError());
  return 0;
}

int transpose_v(cudaStream_t st, const bf16* qkv, bf16* vt, int B, int S, int Spad, int H) {
  dim3 grid((Spad + 63) / 64, H, B);
  transpose_v_kernel<<<grid, 256, 0, st>>>(qkv, vt, S, Spad, H, H * DH);
  BW_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace bw
