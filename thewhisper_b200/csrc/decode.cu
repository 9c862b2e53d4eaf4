// Decoder-step kernels for sm_90a (q_len = 1): every one is a stream over weights or KV in HBM, so they are
// plain coalesced 16-byte-load kernels sized to cover all SMs; no tensor cores (SURVEY.md §8d: the step is
// HBM-bound, 1.60 GB of weights + 245.76 MB cross-KV per audio per token).
//
// Replaces, per generated token, TF/models/whisper/modeling_whisper.py:449-506 (decoder layer), :738-763
// (embeddings), :1081 (tied LM head) and the logits processors + argmax of TF/generation/logits_process.py:1812-2043
// and TF/generation/utils.py:2762-2797, which the reference runs as ~30 launches per layer plus Python loops.
#include <math.h>

#include "decode.cuh"
#include "kernels.h"

namespace BW_NS {

namespace {

// x[q, :] = E[token[q, pos], :] + P[pos, :]
__global__ void embed_kernel(const bf16* __restrict__ E, const float* __restrict__ P, const int* __restrict__ tokens,
                             const int* __restrict__ pos_ptr, float* __restrict__ x, int D, int Tmax) {
  const int q = blockIdx.x;
  pdl_wait();
  pdl_launch();
  const int pos = *pos_ptr;
  const int tok = tokens[q * Tmax + pos];
  for (int d = threadIdx.x; d < D; d += blockDim.x)
    x[(long long)q * D + d] = e2f(E[(long long)tok * D + d]) + P[(long long)pos * D + d];
}
// int8 embedding: x[q, :] = Es[t] * E[t, :] + P[pos, :], t = token[q, pos]
__global__ void embed_s8_kernel(const int8_t* __restrict__ E, const float* __restrict__ Es, const float* __restrict__ P,
                                const int* __restrict__ tokens, const int* __restrict__ pos_ptr, float* __restrict__ x, int D, int Tmax) {
  const int q = blockIdx.x;
  pdl_wait();
  pdl_launch();
  const int pos = *pos_ptr;
  const int tok = tokens[q * Tmax + pos];
  const float s = Es[tok];
  for (int d = threadIdx.x; d < D; d += blockDim.x)
    x[(long long)q * D + d] = s * (float)E[(long long)tok * D + d] + P[(long long)pos * D + d];
}

// ------------------------------------------------------------------------------------------------
// token selection: suppress masks + Whisper timestamp rules + greedy argmax, one block per sequence
// (SuppressTokens -> SuppressTokensAtBegin -> WhisperTimeStamp, the order observed in SURVEY.md §3.3)
// ------------------------------------------------------------------------------------------------
struct MaxIdx {
  float v;
  int i;
};
__device__ __forceinline__ MaxIdx better(MaxIdx a, MaxIdx b) {  // larger value, ties -> smaller index (torch.argmax)
  if (b.v > a.v || (b.v == a.v && b.i < a.i)) return b;
  return a;
}
__device__ __forceinline__ MaxIdx warp_best(MaxIdx m) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    MaxIdx t;
    t.v = __shfl_xor_sync(0xffffffffu, m.v, o);
    t.i = __shfl_xor_sync(0xffffffffu, m.i, o);
    m = better(m, t);
  }
  return m;
}

constexpr int SEL_THREADS = 1024;

__global__ void __launch_bounds__(SEL_THREADS) select_kernel(const SelectArgs a) {
  __shared__ MaxIdx s_text[32], s_ts[32];
  __shared__ float s_sum[32];
  __shared__ float s_f[4];
  __shared__ int s_i[8];
  const int q = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  pdl_wait();
  pdl_launch();
  const int pos = *a.pos;          // index of the token just consumed
  const int cur_len = pos + 1;     // tokens present; the new token goes to index cur_len
  const bool generating = cur_len >= a.begin_index && cur_len < a.Tmax;
  const bool want_nsp = a.out_lp && pos == a.nsp_cfg[0];
  if (!generating && want_nsp) {
    // a forced step whose input is <|startoftranscript|> (a prompt or history before it): only the raw lse, for the no-speech prob
    const float* lg = a.logits + (long long)q * a.ldl;
    float m = -INFINITY;
    for (int v = threadIdx.x; v < a.V; v += SEL_THREADS) m = fmaxf(m, lg[v]);
    m = warp_max(m);
    if (lane == 0) s_sum[warp] = m;
    __syncthreads();
    if (warp == 0) {
      const float r = warp_max(s_sum[lane]);
      if (lane == 0) s_f[0] = r;
    }
    __syncthreads();
    m = s_f[0];
    __syncthreads();
    float sum = 0.f;
    for (int v = threadIdx.x; v < a.V; v += SEL_THREADS) sum += __expf(lg[v] - m);
    sum = warp_sum(sum);
    if (lane == 0) s_sum[warp] = sum;
    __syncthreads();
    if (threadIdx.x == 0) {
      float rsum = 0.f;
      for (int w = 0; w < SEL_THREADS / 32; ++w) rsum += s_sum[w];
      a.out_nsp[q] = expf(lg[a.nsp_cfg[1]] - (m + logf(rsum)));
    }
  }
  if (generating) {
    const float* lg = a.logits + (long long)q * a.ldl;
    const int* seq = a.tokens + q * a.Tmax;
    // ---- mask ranges from the token history (WhisperTimeStampLogitsProcessor, logits_process.py:1995-2033)
    if (threadIdx.x == 0) {
      int block_ts_all = 0, block_text_below_eos = 0, ts_lo_block_end = a.ts_begin, first_step = 0;
      if (a.ts_rules) {
        const int ngen = cur_len - a.begin_index;
        const bool last_ts = ngen >= 1 && seq[cur_len - 1] >= a.ts_begin;
        const bool penult_ts = ngen < 2 || seq[cur_len - 2] >= a.ts_begin;
        if (last_ts) {
          if (penult_ts) block_ts_all = 1;
          else block_text_below_eos = 1;
        }
        int last_tsv = -1;
        for (int i = cur_len - 1; i >= a.begin_index; --i)
          if (seq[i] >= a.ts_begin) { last_tsv = seq[i]; break; }
        if (last_tsv >= 0) ts_lo_block_end = (last_ts && !penult_ts) ? last_tsv : last_tsv + 1;
        first_step = (cur_len == a.begin_index);
      }
      s_i[0] = block_ts_all; s_i[1] = block_text_below_eos; s_i[2] = ts_lo_block_end; s_i[3] = first_step;
    }
    __syncthreads();
    const int block_ts_all = s_i[0], block_text_below_eos = s_i[1], ts_lo_end = s_i[2], first_step = s_i[3];
    const bool at_begin = (cur_len == a.begin_index);
    const int last_allowed = (a.max_initial_ts >= 0) ? a.ts_begin + a.max_initial_ts : a.V;
    auto masked = [&](int v) -> bool {
      if (a.suppress_bits[v >> 5] >> (v & 31) & 1u) return true;
      if (at_begin && a.begin_suppress_bits && (a.begin_suppress_bits[v >> 5] >> (v & 31) & 1u)) return true;
      if (a.ts_rules) {
        if (v == a.no_ts) return true;
        if (v >= a.ts_begin) {
          if (block_ts_all) return true;
          if (v < ts_lo_end) return true;
          if (first_step && v > last_allowed) return true;
        } else {
          if (block_text_below_eos && v < a.eos) return true;
          if (first_step) return true;
        }
      }
      return false;
    };
    // ---- pass 1: masked max / argmax of the text range and of the timestamp range; raw max for the lse
    MaxIdx bt{-INFINITY, 0x7fffffff}, bs{-INFINITY, 0x7fffffff};
    float rawmax = -INFINITY;
    const int tsb = a.ts_rules ? a.ts_begin : a.V;
    for (int v = threadIdx.x; v < a.V; v += SEL_THREADS) {
      const float x = lg[v];
      rawmax = fmaxf(rawmax, x);
      if (!masked(v)) {
        MaxIdx c{x, v};
        if (v < tsb) bt = better(bt, c);
        else bs = better(bs, c);
      }
    }
    bt = warp_best(bt);
    bs = warp_best(bs);
    rawmax = warp_max(rawmax);
    if (lane == 0) { s_text[warp] = bt; s_ts[warp] = bs; s_sum[warp] = rawmax; }
    __syncthreads();
    if (warp == 0) {
      MaxIdx t = s_text[lane], s = s_ts[lane];
      float r = s_sum[lane];
      t = warp_best(t); s = warp_best(s); r = warp_max(r);
      if (lane == 0) { s_text[0] = t; s_ts[0] = s; s_f[0] = r; }
    }
    __syncthreads();
    bt = s_text[0];
    bs = s_ts[0];
    rawmax = s_f[0];
    __syncthreads();
    // ---- pass 2: sum exp over unmasked timestamps (relative to their max) and over all raw logits
    //      (+ with scores on: over unmasked text, relative to its max -- the allowed mass)
    const bool scores = a.out_lp != nullptr;
    float ts_sum = 0.f, raw_sum = 0.f, text_sum = 0.f;
    for (int v = threadIdx.x; v < a.V; v += SEL_THREADS) {
      const float x = lg[v];
      raw_sum += __expf(x - rawmax);
      if (v >= tsb && !masked(v)) ts_sum += __expf(x - bs.v);
      if (scores && v < tsb && !masked(v)) text_sum += __expf(x - bt.v);
    }
    ts_sum = warp_sum(ts_sum);
    raw_sum = warp_sum(raw_sum);
    if (scores) text_sum = warp_sum(text_sum);
    if (lane == 0) { s_sum[warp] = ts_sum; s_text[warp].v = raw_sum; s_ts[warp].v = text_sum; }
    __syncthreads();
    if (threadIdx.x == 0) {
      float tsum = 0.f, rsum = 0.f;
      for (int w = 0; w < SEL_THREADS / 32; ++w) { tsum += s_sum[w]; rsum += s_text[w].v; }
      if (a.out_lse) a.out_lse[q] = rawmax + logf(rsum);
      int choice;
      if (a.ts_rules) {
        // "sum of timestamp probability > max text probability -> sample a timestamp" (logits_process.py:2036-2041);
        // both sides share the log-softmax normaliser, so compare logsumexp(ts logits) with max(text logits)
        const float ts_lse = (bs.v == -INFINITY) ? -INFINITY : bs.v + logf(tsum);
        const bool force_ts = ts_lse > bt.v;
        if (force_ts) choice = bs.i;
        else choice = better(bt, bs).i;
      } else {
        choice = bt.i;
      }
      const bool was_finished = a.finished[q] != 0;
      if (scores) {
        // log-softmax of the processed scores: the allowed set is the unmasked timestamps alone when a timestamp is forced
        float xsum = 0.f;
        for (int w = 0; w < SEL_THREADS / 32; ++w) xsum += s_ts[w].v;
        const float raw_lse = rawmax + logf(rsum);
        const float ts_lse = (bs.v == -INFINITY) ? -INFINITY : bs.v + logf(tsum);
        const float text_lse = (bt.v == -INFINITY) ? -INFINITY : bt.v + logf(xsum);
        const bool forced = a.ts_rules && ts_lse > bt.v;
        float allowed = ts_lse;
        if (!forced && text_lse != -INFINITY) {
          const float hi = fmaxf(text_lse, ts_lse), lo = fminf(text_lse, ts_lse);
          allowed = (lo == -INFINITY) ? hi : hi + log1pf(expf(lo - hi));
        }
        a.out_lmass[q * a.Tmax + cur_len] = allowed - raw_lse;
        a.out_lp[q * a.Tmax + cur_len] = was_finished ? 0.f : (choice < a.V ? lg[choice] - allowed : -INFINITY);  // (none allowed)
        if (want_nsp) a.out_nsp[q] = expf(lg[a.nsp_cfg[1]] - raw_lse);
      }
      if (was_finished) choice = a.pad;
      else if (choice == a.eos) a.finished[q] = 1;
      a.tokens[q * a.Tmax + cur_len] = choice;
      s_f[1] = rawmax + logf(rsum);
      s_i[4] = (a.ts_rules && ((bs.v == -INFINITY) ? -INFINITY : bs.v + logf(tsum)) > bt.v) ? 1 : 0;
    }
    if (a.n_cand > 0) {
      // ---- beam search: this sequence's best n_cand continuations, score = running score + log-softmax(raw)[v] with
      //      the processors' masks (HF: log_softmax first, then processors, utils.py:3256-3257); the host merges the
      //      per-beam lists into the per-audio top 2*num_beams (ties -> smaller token id)
      __shared__ int s_sel[16];
      __syncthreads();
      const float lse = s_f[1];
      const int force_ts = s_i[4];
      const float run = a.run_scores[q];
      for (int k = 0; k < a.n_cand; ++k) {
        MaxIdx best{-INFINITY, 0x7fffffff};
        for (int v = threadIdx.x; v < a.V; v += SEL_THREADS) {
          if (masked(v) || (force_ts && v < tsb)) continue;
          bool taken = false;
          for (int j = 0; j < k; ++j) taken |= (s_sel[j] == v);
          if (taken) continue;
          best = better(best, MaxIdx{lg[v], v});
        }
        best = warp_best(best);
        if (lane == 0) s_text[warp] = best;
        __syncthreads();
        if (warp == 0) {
          MaxIdx t = warp_best(s_text[lane]);
          if (lane == 0) {
            s_sel[k] = t.i;
            const bool none = (t.i == 0x7fffffff);
            a.cand_scores[q * a.n_cand + k] = none ? -INFINITY : (t.v - lse + run);
            a.cand_tokens[q * a.n_cand + k] = none ? -1 : t.i;
          }
        }
        __syncthreads();
      }
    }
  }
  // ---- last block advances the shared position counter
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned prev = atomicAdd(a.done_ctr, 1u);
    if (prev == (unsigned)(a.Q - 1)) {
      *a.done_ctr = 0u;
      *a.pos = pos + 1;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm over rows (encoder): fp32 in, bf16 (GEMM operand) or fp32 out.  One warp per row.
// ------------------------------------------------------------------------------------------------
template <typename OutT>
__global__ void layernorm_rows_kernel(const float* __restrict__ x, const float* __restrict__ g, const float* __restrict__ b,
                                      OutT* __restrict__ y, int rows, int D) {
  pdl_wait();
  pdl_launch();
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* xr = x + (long long)row * D;
  float s = 0.f;
  for (int k = lane * 4; k < D; k += 128) {
    const float4 v = *reinterpret_cast<const float4*>(xr + k);
    s += v.x + v.y + v.z + v.w;
  }
  const float mean = warp_sum(s) / (float)D;
  float ss = 0.f;
  for (int k = lane * 4; k < D; k += 128) {
    const float4 v = *reinterpret_cast<const float4*>(xr + k);
    const float a0 = v.x - mean, a1 = v.y - mean, a2 = v.z - mean, a3 = v.w - mean;
    ss += a0 * a0 + a1 * a1 + a2 * a2 + a3 * a3;
  }
  const float rstd = rsqrtf(warp_sum(ss) / (float)D + 1e-5f);
  for (int k = lane * 4; k < D; k += 128) {
    const float4 v = *reinterpret_cast<const float4*>(xr + k);
    const float4 gg = *reinterpret_cast<const float4*>(g + k);
    const float4 bb = *reinterpret_cast<const float4*>(b + k);
    const float o0 = (v.x - mean) * rstd * gg.x + bb.x, o1 = (v.y - mean) * rstd * gg.y + bb.y;
    const float o2 = (v.z - mean) * rstd * gg.z + bb.z, o3 = (v.w - mean) * rstd * gg.w + bb.w;
    if constexpr (sizeof(OutT) == 2) {
      uint2 w;
      w.x = pack_bf16(o0, o1);
      w.y = pack_bf16(o2, o3);
      *reinterpret_cast<uint2*>(reinterpret_cast<bf16*>(y) + (long long)row * D + k) = w;
    } else {
      *reinterpret_cast<float4*>(reinterpret_cast<float*>(y) + (long long)row * D + k) = make_float4(o0, o1, o2, o3);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// batched decoder step: residual update from split-K partial sums fused with the LayerNorm that follows it.
// One CTA per sequence row, values held in registers (D <= 8 * RL_THREADS).
// ------------------------------------------------------------------------------------------------
constexpr int RL_THREADS = 256;
__device__ __forceinline__ float block_sum_rl(float v, float* red) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int w = 0; w < RL_THREADS / 32; ++w) s += red[w];
  __syncthreads();
  return s;
}
__global__ void __launch_bounds__(RL_THREADS) resid_ln_kernel(float* __restrict__ x, const float* __restrict__ part, int nsplit,
                                                              long long split_stride, const float* __restrict__ bias,
                                                              const float* __restrict__ g, const float* __restrict__ b,
                                                              bf16* __restrict__ y, int D) {
  __shared__ float red[RL_THREADS / 32];
  const int q = blockIdx.x;
  pdl_wait();
  pdl_launch();
  float* xr = x + (long long)q * D;
  float4 v[2];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int k = (threadIdx.x + i * RL_THREADS) * 4;
    v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (k < D) {
      v[i] = *reinterpret_cast<const float4*>(xr + k);
      if (nsplit > 0) {
        if (bias) {
          const float4 bb = *reinterpret_cast<const float4*>(bias + k);
          v[i].x += bb.x; v[i].y += bb.y; v[i].z += bb.z; v[i].w += bb.w;
        }
        const float* pq = part + (long long)q * D + k;
        int sp = 0;
        for (; sp + 3 < nsplit; sp += 4) {  // four splits' loads in flight together, added in split order
          float4 pp[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) pp[u] = *reinterpret_cast<const float4*>(pq + (long long)(sp + u) * split_stride);
#pragma unroll
          for (int u = 0; u < 4; ++u) { v[i].x += pp[u].x; v[i].y += pp[u].y; v[i].z += pp[u].z; v[i].w += pp[u].w; }
        }
        for (; sp < nsplit; ++sp) {
          const float4 pp = *reinterpret_cast<const float4*>(pq + (long long)sp * split_stride);
          v[i].x += pp.x; v[i].y += pp.y; v[i].z += pp.z; v[i].w += pp.w;
        }
        *reinterpret_cast<float4*>(xr + k) = v[i];
      }
      s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
  }
  if (!y) return;
  const float mean = block_sum_rl(s, red) / (float)D;
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int k = (threadIdx.x + i * RL_THREADS) * 4;
    if (k < D) {
      const float a0 = v[i].x - mean, a1 = v[i].y - mean, a2 = v[i].z - mean, a3 = v[i].w - mean;
      ss += (a0 * a0 + a1 * a1) + (a2 * a2 + a3 * a3);
    }
  }
  const float rstd = rsqrtf(block_sum_rl(ss, red) / (float)D + 1e-5f);
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int k = (threadIdx.x + i * RL_THREADS) * 4;
    if (k < D) {
      const float4 gg = *reinterpret_cast<const float4*>(g + k);
      const float4 bb = *reinterpret_cast<const float4*>(b + k);
      uint2 w;
      w.x = pack_bf16((v[i].x - mean) * rstd * gg.x + bb.x, (v[i].y - mean) * rstd * gg.y + bb.y);
      w.y = pack_bf16((v[i].z - mean) * rstd * gg.z + bb.z, (v[i].w - mean) * rstd * gg.w + bb.w);
      *reinterpret_cast<uint2*>(y + (long long)q * D + k) = w;
    }
  }
}

}  // namespace

int launch_resid_ln(cudaStream_t st, float* x, const float* part, int nsplit, long long split_stride, const float* bias, const float* g,
                    const float* b, bf16* y, int Q, int D) {
  BW_CHECK(D % 4 == 0 && D <= 8 * RL_THREADS, "resid_ln: D=%d must be a multiple of 4 and <= %d", D, 8 * RL_THREADS);
  BW_CUDA_OK(launch_k(resid_ln_kernel, dim3(Q), dim3(RL_THREADS), 0, st, x, part, nsplit, split_stride, bias, g, b, y, D));
  return 0;
}

int launch_embed(cudaStream_t st, const void* E, const float* Es, const float* P, const int* tokens, const int* pos, float* x, int Q, int D,
                 int Tmax) {
  if (Es) BW_CUDA_OK(launch_k(embed_s8_kernel, dim3(Q), dim3(256), 0, st, static_cast<const int8_t*>(E), Es, P, tokens, pos, x, D, Tmax));
  else BW_CUDA_OK(launch_k(embed_kernel, dim3(Q), dim3(256), 0, st, static_cast<const bf16*>(E), P, tokens, pos, x, D, Tmax));
  return 0;
}

int launch_select(cudaStream_t st, const SelectArgs& a0) {
  SelectArgs a = a0;
  if (a.ldl < a.V) a.ldl = a.V;
  BW_CUDA_OK(launch_k(select_kernel, dim3(a.Q), dim3(SEL_THREADS), 0, st, a));
  return 0;
}

int layernorm_bf16(cudaStream_t st, const float* x, const float* g, const float* b, bf16* y, int rows, int D) {
  BW_CHECK(D % 4 == 0, "layernorm: D=%d must be a multiple of 4", D);
  BW_CUDA_OK(launch_k(layernorm_rows_kernel<bf16>, dim3((rows + 7) / 8), dim3(256), 0, st, x, g, b, y, rows, D));
  return 0;
}

int layernorm_f32(cudaStream_t st, const float* x, const float* g, const float* b, float* y, int rows, int D) {
  BW_CHECK(D % 4 == 0, "layernorm: D=%d must be a multiple of 4", D);
  BW_CUDA_OK(launch_k(layernorm_rows_kernel<float>, dim3((rows + 7) / 8), dim3(256), 0, st, x, g, b, y, rows, D));
  return 0;
}

}  // namespace bw
