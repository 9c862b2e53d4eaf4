// One persistent kernel per decoder step (q_len = 1, one beam per audio, up to 2 sequences).
//
// Why: with one kernel per op the step is 259 launches and every op pays its own chain of dependent global round
// trips, several times the time its bytes take at HBM bandwidth.  Here the whole step -- embedding, 32 x (LN1+QKV, self-attention, out-proj,
// LN2+cross-q, cross-attention, out-proj, LN3+fc1+GELU, fc2), final LN + tied LM head -- runs in ONE kernel of one CTA
// per SM, phases separated by a grid barrier.
//
// What the barrier timelines and ncu captures of the earlier versions taught:
//   * a phase is only as fast as its chain of *dependent* L2/DRAM round trips (~0.6-1 us each), not its bytes: everything
//     that does not depend on the previous phase is requested BEFORE the barrier that precedes a phase -- the weight rows
//     of the phase (TMA bulk copies into a per-warp smem slab, one instruction per row: issuing the same bytes as 16-byte
//     cp.async pieces cost ~1 us of LSU issue time per phase), bias values, LayerNorm gamma/beta, the attention K/V rows
//     that are already final;
//   * the barrier is one red.release + ld.acquire polling loop (no membar.sc / L1 invalidation; activations that cross
//     CTAs are read with ld.global.cg);
//   * the GEMV inner loop is bound by the 128 B/clk shared-memory port: x is LayerNormed once per CTA (not on the fly in
//     every warp), and lanes read contiguous 16-byte (x) / 8-byte (w) pieces so no LDS has bank conflicts;
//   * 31% of the non-barrier stall samples were instruction-cache misses: the fully inlined version was 15k SASS
//     instructions (245 KB) walked once per layer against a 32 KB L1.5 I-cache.  The six GEMV phases of a layer are
//     therefore ONE loop body driven by a small descriptor (make_desc), not six inlined copies;
//   * the two slab regions (double buffering, see the kernel body) must fit: the smem limit is the device's opt-in limit
//     less the kernel's static smem as compiled.  On 132 SMs large-v3 at Q = 1 fits with 640 B to spare; an estimated
//     8 KB margin had made every step single-buffered (H100 SXM at 700 W: 1.27 ms per step, 1.19 ms double-buffered);
//   * more lookahead is not better: a per-CTA byte ring that requested the rows of every later phase as far ahead as
//     ~200 KB of smem allowed, right after each barrier arrival, left no slab exposed but roughly tripled the latency of
//     the barriers behind those ~26 MB of copies (1.41 ms per step);
//   * weight rows are NOT prefetched into L2.  A DRAM -> L2 prefetch of each phase's rows two phases ahead (~13 MB for fc1
//     and for fc2) kept the slabs from ever being exposed (0.13 us), but every barrier that ran while it was in flight slowed
//     down: cross-q 4.0 us and cross out-proj 4.8 us instead of ~1 us (layer averages).  Keeping the prefetch W bytes ahead
//     of the copies with a per-CTA cursor, or capping it per hand-over to even out the DRAM load, only moved that cost into
//     other phases (1.18-1.33 ms per step for W = 8-48 MB, H100 SXM at 700 W).  With no weight prefetch the slab copy, issued a whole phase ahead
//     into the second slab region, reads DRAM itself: the cross-q barrier falls to 1.0 us and the step from 1.19-1.20 to
//     1.13-1.16 ms (H100 80GB HBM3, 400 W power limit).  Only the cross-attention K/V, read by a bulk load three phases
//     later, are still prefetched: without that the cross-attention phase took 6.7 us instead of 5.9 us (the step times of the
//     two were within each other's spread);
//   * the cross-attention key splits are merged by their consumer: each CTA's cross out-projection staging reads the partials
//     of every split (merge_xattn, one round of independent L2 loads).  When the last-arriving split of each head merged them in
//     phase E, behind an acq_rel counter and a second dependent round trip, every CTA waited for that at the barrier.  The DMA
//     warp queues the fc1 slab copy (~100 KB per SM) only once the merge loads are issued: queued first, it held them back.
//     H100 80GB HBM3 at 700 W, bench.py: 849-850 tok/s instead of 812-814 (829-830 with the copy queued first).  The traced
//     instantiation does not show it: E's work falls from 5.9-6.2 to 4.5 us, but F's rises from 1.7 to 4.1 us and fc2's
//     x staging from 0.6 to 3.4 us, and its step span is not shorter -- take step times from the untraced kernel.
// After a barrier only the x row (and the residual values of the rows a warp owns) have to be fetched.
//
// Work split: 12 warps per CTA, global warp id gw; a GEMV phase gives warp gw the R rows starting at gw*R (one pass:
// the launcher checks 12 * SMs * R >= N); attention phases hand (sequence, head[, key split]) items to CTAs round-robin.
// Token selection stays a separate small kernel.
#include "decode_mega_common.cuh"

namespace BW_NS {

namespace {

using namespace mega;


// Template parameter VAR: bit 0 (V_NOTRACE) compiles the barrier-timeline instrumentation out.  The launcher picks it whenever no
// trace buffer is attached.  Round 1 left five more hand-over variants
// here (relaxed barriers over tagged activations, per-head readiness counters, a 4-way sharded barrier counter, producer-only
// arrival, several steps per launch) and a third-generation kernel (attention fused with its out-projection); measured in round 2
// they were bit-exact and no faster than this one, so they are gone (history: commit c3ab1ae).
constexpr unsigned V_NOTRACE = 1;

__device__ __noinline__ void wait_timeout(const char* what, unsigned a0, unsigned a1) {
  printf("[bw] decode_mega: %s timed out (block %d thread %d: %u %u)\n", what, blockIdx.x, threadIdx.x, a0, a1);
  __trap();
}
// grid barrier: monotonically increasing arrival counter (zeroed by a memset node before the kernel).  bar.sync orders
// the CTA's writes before thread 0's release; the acquire poll + bar.sync orders the other CTAs' writes before our reads.
template <unsigned VAR>
struct GridBar {
  static constexpr bool TRACE = !(VAR & V_NOTRACE);
  unsigned* ctr;
  unsigned nblocks;
  unsigned epoch;
  long long* trace;  // optional [nblocks][2*MEGA_TRACE_N]: arrival / release time of every barrier (BW_MEGA_TRACE=1)
  // Two lessons from the timelines: (1) as a real (noinline) call the compiler waited for every in-flight prefetch load that
  // is live across it (~1 us per phase); (2) the release fence of the arriving thread waits for that thread's OWN outstanding
  // loads -- so the arriving thread is the CTA's last one, which never has a prefetch load in flight (it owns no LayerNorm
  // slice for D <= 1280 and never finishes a row, see prefetch_phase).
  // arrive() right after the CTA's own __syncthreads, wait() after whatever can be requested for the next phase: the arrival
  // is not delayed by the prefetch issue, and the ~700 read requests of a slab copy queue behind the arrival, not before it.
  __device__ __forceinline__ void arrive() {
    if (threadIdx.x == MT - 1) {
      if (TRACE && trace && epoch < MEGA_TRACE_N) trace[((long long)blockIdx.x * MEGA_TRACE_N + epoch) * 2] = global_ns();
      red_release_add(ctr, 1u);
    }
  }
  // (a per-CTA flag array polled by one warp instead of the single counter was tried: 3+ us per barrier)
  __device__ __forceinline__ void wait() {
    if (threadIdx.x == MT - 1) {
      const unsigned target = (epoch + 1) * nblocks;
      if (ld_acquire_u32(ctr) < target) {
        const long long t0 = clock64();
        while (ld_acquire_u32(ctr) < target) {
          if (clock64() - t0 > (1ll << 32)) {
            printf("[bw] decode_mega: grid barrier %u timed out (block %d)\n", epoch, blockIdx.x);
            __trap();
          }
        }
      }
      if (TRACE && trace && epoch < MEGA_TRACE_N) trace[((long long)blockIdx.x * MEGA_TRACE_N + epoch) * 2 + 1] = global_ns();
    }
    ++epoch;
    __syncthreads();
  }
  __device__ __forceinline__ void sync() {
    __syncthreads();
    arrive();
    wait();
  }
};

// One GEMV phase: out[m][n] = epi(sum_k W[n][k] * LN?(src[m])[k] + bias[n]).
struct GemvDesc {
  const uint8_t* W;       // rows of K elements: 16-bit, or int8 codes (W8 instantiation)
  const float* scale;     // W8: fp32 scale per row, applied to the finished dot product before the bias
  const float* bias;
  int N, K, R;            // R rows per warp (1 .. RMAX)
  int n0, nend;           // rows of this CTA: [n0, nend), contiguous, ceil(N / CTAs) each (the LM head streams: [0, N))
  bool lm;
  const float* src;       // [M][K] fp32 activations written by an earlier phase
  const float *lng, *lnb; // LayerNorm applied to src while staging (nullptr: none)
  float* out;
  int ldo;
  const float* residual;  // may alias out
  int act;                // 1: GELU
  float alpha;            // rows < alpha_cols are scaled (q * 1/sqrt(dh))
  int alpha_cols;
  bf16 *kc, *vc;          // optional self-KV append (fused QKV): rows [D, 2D) -> kc, [2D, 3D) -> vc at position pos
};

// g: 0 LN1+QKV | 1 self out-proj | 2 LN2+cross q | 3 cross out-proj | 4 LN3+fc1+GELU | 5 fc2; l == a.L: final LN + LM head
__device__ __forceinline__ void split_rows(GemvDesc& d) {
  const int rc = (d.N + (int)gridDim.x - 1) / (int)gridDim.x;
  d.R = (rc + MW - 1) / MW;
  d.n0 = min(d.N, (int)blockIdx.x * rc);
  d.nend = min(d.N, d.n0 + rc);
}
template <unsigned VAR, bool W8>
__device__ __forceinline__ GemvDesc make_desc(const MegaArgs& a, const MegaLayer* layers, int l, int g, int pos) {
  GemvDesc d;
  d.scale = nullptr;
  if constexpr (W8) d.scale = l >= a.L ? a.embed_scale : a.wscale[l * 6 + g];
  d.lng = d.lnb = nullptr;
  d.residual = nullptr;
  d.act = 0;
  d.alpha = 1.f;
  d.alpha_cols = 0;
  d.kc = d.vc = nullptr;
  d.N = d.K = d.ldo = a.D;
  d.lm = false;
  if (l >= a.L) {
    d.W = static_cast<const uint8_t*>(a.embed); d.bias = nullptr; d.N = a.V; d.R = 2; d.n0 = 0; d.nend = a.V; d.lm = true; d.src = a.dx; d.lng = a.lnf_g; d.lnb = a.lnf_b; d.out = a.logits; d.ldo = a.ldl;
    return d;
  }
  const MegaLayer& L = layers[l];
  switch (g) {
    case 0:
      d.W = static_cast<const uint8_t*>(L.wqkv); d.bias = L.bqkv; d.N = 3 * a.D; d.src = a.dx; d.lng = L.ln1g; d.lnb = L.ln1b; d.out = a.dqkv; d.ldo = 3 * a.D;
      d.alpha = 0.125f; d.alpha_cols = a.D; d.kc = L.self_k; d.vc = L.self_v;
      break;
    case 1:
      d.W = static_cast<const uint8_t*>(L.wo); d.bias = L.bo; d.src = a.dattn; d.out = a.dx; d.residual = a.dx;
      break;
    case 2:
      d.W = static_cast<const uint8_t*>(L.xwq); d.bias = L.xbq; d.src = a.dx; d.lng = L.ln2g; d.lnb = L.ln2b; d.out = a.dq; d.alpha = 0.125f; d.alpha_cols = a.D;
      break;
    case 3:
      d.W = static_cast<const uint8_t*>(L.xwo); d.bias = L.xbo; d.src = a.part_o; d.out = a.dx; d.residual = a.dx;  // x: merge_xattn
      break;
    case 4:
      d.W = static_cast<const uint8_t*>(L.w1); d.bias = L.b1; d.N = a.ffn; d.src = a.dx; d.lng = L.ln3g; d.lnb = L.ln3b; d.out = a.dh; d.ldo = a.ffn; d.act = 1;
      break;
    default:
      d.W = static_cast<const uint8_t*>(L.w2); d.bias = L.b2; d.K = a.ffn; d.src = a.dh; d.out = a.dx; d.residual = a.dx;
      break;
  }
  split_rows(d);
  return d;
}

// What a warp requests before the barrier that precedes a GEMV phase: its weight rows (lane 0: one TMA bulk copy per
// row into the warp's slab, completion on the warp's mbarrier), the bias values and this thread's LayerNorm slice.
struct Pre {
  float bias;   // of the row this lane finishes (lanes [8r, 8r + MB) finish row n + r)
  float scale;  // W8: the scale of that row
  float4 g, b;  // gamma / beta of elements [4*tid, 4*tid + 4)
};

// The CTA's weight rows of a layer phase: one bulk copy into a slab region, completion on that region's mbarrier.  The rows
// of a CTA's 12 warps are contiguous in memory (rows [blockIdx*12*R, +12*R)) and so are their slabs in smem: one TMA
// operation per CTA and phase.  (Per-row operations cost ~10 ns of TMA issue each -- 36 of them per SM and phase were
// 0.35 us on the critical path.)
template <int ESZ>
__device__ __forceinline__ void issue_slabs(const GemvDesc& d, uint8_t* region, uint64_t* cbar) {
  if (threadIdx.x == DMA_T && d.n0 < d.nend) {
    const uint32_t bytes = (uint32_t)(d.nend - d.n0) * d.K * ESZ;
    mbar_arrive_expect_tx(cbar, bytes);
    if constexpr (ESZ == 2) bulk_g2s(region, reinterpret_cast<const bf16*>(d.W) + (long long)d.n0 * d.K, bytes, cbar);
    else bulk_g2s(region, d.W + (long long)d.n0 * d.K, bytes, cbar);
  }
}

// What is requested before the barrier that precedes a GEMV phase (besides the slabs): the bias of the row a lane will
// finish and this thread's LayerNorm slice.  The LM head (many passes) uses per-warp slabs and barriers: its passes are
// refilled warp by warp; its first pass is requested here.
template <bool W8>
__device__ __forceinline__ void prefetch_phase(const GemvDesc& d, Pre& p, uint8_t* pool, uint64_t* wbar, int gw, int warp, int lane) {
  constexpr int ESZ = W8 ? 1 : 2;
  int n;
  if (d.lm) {
    n = gw * d.R;
    if (n < d.N) issue_rows<ESZ>(pool + (size_t)warp * d.R * d.K * ESZ, wbar, d.W, d.K, d.R, n, d.N, lane);
  } else {
    n = d.n0 + warp * d.R;
  }
  const int r_sel = lane >> 3;
  p.bias = (d.bias && (lane & 7) < 2 && r_sel < d.R && n + r_sel < d.nend) ? d.bias[n + r_sel] : 0.f;
  if constexpr (W8) p.scale = (!d.lm && (lane & 7) < 2 && r_sel < d.R && n + r_sel < d.nend) ? d.scale[n + r_sel] : 1.f;
  const int k = threadIdx.x * 4;
  if (d.lng && k < d.K) {
    p.g = *reinterpret_cast<const float4*>(d.lng + k);
    p.b = *reinterpret_cast<const float4*>(d.lnb + k);
  }
}

// The cross out-projection's x: the cross-attention output of each sequence, merged here from the partials of its nsplit key
// splits (part_o [Q][H][nsplit][64], part_ml [..][2] = (max, sum)) that phase E left, so that phase E ends at its barrier arrival.
// Thread t stages elements [4t, 4t + 4) of a sequence: lane j of a 16-lane group (one head) reads split j's (max, sum) and the
// group shares them by shuffle; the loads of the first XC splits are issued before any is used, so for nsplit <= XC a
// sequence costs one round of L2 reads, queued before the DMA warp's slab copy of the next phase.  (At Q = 2 the sequences go
// one after the other: both rounds in flight together would need ~50 more registers than the kernel's peak.)  The arithmetic (the pl > 0 predicate, the maximum, __expf weights,
// fmaf sums in split order, one division) is fixed, so every CTA stages the same x bit for bit.  The CTA also stores its own
// rows [n0, nend) of x to dattn: nothing in the step reads them, but after the step dattn holds the last layer's
// cross-attention output as on the other step paths.
template <int MB>
__device__ __forceinline__ void merge_xattn(float* xs, const GemvDesc& d, const MegaArgs& a, int M) {
  constexpr int XC = 6;  // splits per round of loads (large-v3 on 132 SMs: nsplit = 6)
  static_assert(MAXD <= (MT - 32) * 4 && XSPLIT <= 16, "one float4 per staging thread and sequence; one lane per split");
  const int K = d.K, nsplit = a.nsplit;
  const int k = threadIdx.x * 4, sp_l = threadIdx.x & 15;
  const bool have = k < K;
#pragma unroll 1
  for (int m = 0; m < MB; ++m) {
    const int hb = (m * a.H + (k >> 6)) * nsplit;  // (sequence, head) of this thread's elements
    const float* po_base = a.part_o + hb * 64 + (k & 63);
    const bool live = have && m < M;
    float pm = -INFINITY, pl = 0.f;
    float4 po[XC];
    if (live && sp_l < nsplit) {
      const float2 v = __ldcg(reinterpret_cast<const float2*>(a.part_ml) + hb + sp_l);
      pm = v.x;
      pl = v.y;
    }
#pragma unroll
    for (int sp = 0; sp < XC; ++sp) {
      po[sp] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (live && sp < nsplit) po[sp] = __ldcg(reinterpret_cast<const float4*>(po_base + sp * 64));
    }
    if (m == 0) asm volatile("bar.arrive 2, %0;" ::"n"(MT) : "memory");  // loads issued: the DMA warp may queue its copies
    float mx = pl > 0.f ? pm : -INFINITY;  // fmaxf is exact: the tree gives the split-order maximum
#pragma unroll
    for (int s = 8; s >= 1; s >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, s));
    float lsum = 0.f;
    float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int sp0 = 0;;) {
#pragma unroll
      for (int sp = 0; sp < XC; ++sp) {
        const float sm = __shfl_sync(0xffffffffu, pm, sp0 + sp, 16), sl = __shfl_sync(0xffffffffu, pl, sp0 + sp, 16);
        if (sp0 + sp < nsplit && sl > 0.f) {
          const float w = __expf(sm - mx);
          lsum = fmaf(sl, w, lsum);
          o.x = fmaf(po[sp].x, w, o.x);
          o.y = fmaf(po[sp].y, w, o.y);
          o.z = fmaf(po[sp].z, w, o.z);
          o.w = fmaf(po[sp].w, w, o.w);
        }
      }
      sp0 += XC;
      if (sp0 >= nsplit) break;
#pragma unroll
      for (int sp = 0; sp < XC; ++sp)
        if (live && sp0 + sp < nsplit) po[sp] = __ldcg(reinterpret_cast<const float4*>(po_base + (sp0 + sp) * 64));
    }
    if (!have) continue;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (m < M) {
      v = make_float4(o.x / lsum, o.y / lsum, o.z / lsum, o.w / lsum);
      float* row = a.dattn + m * K;
      if (k >= d.n0 && k < d.nend) row[k] = v.x;
      if (k + 1 >= d.n0 && k + 1 < d.nend) row[k + 1] = v.y;
      if (k + 2 >= d.n0 && k + 2 < d.nend) row[k + 2] = v.z;
      if (k + 3 >= d.n0 && k + 3 < d.nend) row[k + 3] = v.w;
    }
    *reinterpret_cast<float4*>(xs + m * K + k) = v;
  }
}

// stage M rows of K floats into smem (ld.global.cg), LayerNormed when the phase has one; xattn (the cross out-projection):
// x is merged from the cross-attention partials instead (merge_xattn).
// The last warp takes no part in the staging: it runs `dma` (the TMA requests of the coming phases, ~0.25 us of issue
// time) meanwhile and only joins the final CTA barrier.  The staging warps synchronise among themselves on named barrier 1.
__device__ __forceinline__ void stage_sync() { asm volatile("bar.sync 1, %0;" ::"n"(MT - 32) : "memory"); }
// End of the staging: the staging warps synchronise among themselves and only SIGNAL the DMA warp (bar.arrive), which
// waits for x (bar.sync on the same barrier) after it has issued its TMA requests -- the ~0.5 us of descriptor arithmetic
// and TMA issue in `dma` run beside the dot products of the other warps instead of in front of them (r1_v8: the
// K-parallel kernel, which has this property, gained 0.3 us on the phases without LayerNorm).
__device__ __forceinline__ void stage_done_stagers() {
  asm volatile("bar.sync 1, %0;" ::"n"(MT - 32) : "memory");
  asm volatile("bar.arrive 3, %0;" ::"n"(MT) : "memory");
}
__device__ __forceinline__ void stage_done_dma() { asm volatile("bar.sync 3, %0;" ::"n"(MT) : "memory"); }

template <int MB, unsigned VAR, class Dma>
__device__ __forceinline__ void stage_x(float* xs, float* red, const GemvDesc& d, const Pre& p, int M, bool split_end, const MegaArgs& a,
                                        bool xattn, Dma&& dma) {
  const int K = d.K;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == MW - 1) {
    if (xattn) asm volatile("bar.sync 2, %0;" ::"n"(MT) : "memory");  // after the merge loads (merge_xattn)
    dma();
    if (split_end) stage_done_dma();
    else __syncthreads();
    return;
  }
  if (xattn) {
    merge_xattn<MB>(xs, d, a, M);
    if (split_end) stage_done_stagers();
    else __syncthreads();
    return;
  }
  constexpr int ST = MT - 32;  // staging threads
  if (!d.lng) {
    constexpr int U = 4;
    for (int base = threadIdx.x * 4; base < MB * K; base += ST * 4 * U) {
      float4 v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int i = base + u * ST * 4;
        const int m = (MB > 1 && i >= K) ? 1 : 0;
        v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (i < MB * K && m < M) v[u] = __ldcg(reinterpret_cast<const float4*>(d.src + (long long)m * K + (i - m * K)));
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int i = base + u * ST * 4;
        if (i < MB * K) *reinterpret_cast<float4*>(xs + i) = v[u];
      }
    }
    if (split_end) stage_done_stagers();
    else __syncthreads();
    return;
  }
  // LayerNorm (K <= 4 * ST): one float4 per thread and row, two-pass statistics through two reductions on register values
  const int k = threadIdx.x * 4;
  const bool have = k < K;
  float4 v[MB];
#pragma unroll
  for (int m = 0; m < MB; ++m) {
    v[m] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (have && m < M) v[m] = __ldcg(reinterpret_cast<const float4*>(d.src + (long long)m * K + k));
  }
#pragma unroll
  for (int m = 0; m < MB; ++m) {
    const float s = warp_sum((v[m].x + v[m].y) + (v[m].z + v[m].w));
    if (lane == 0) red[m * MW + warp] = s;
  }
  stage_sync();
  float mean[MB];
#pragma unroll
  for (int m = 0; m < MB; ++m) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < MW - 1; ++w) s += red[m * MW + w];
    mean[m] = s / (float)K;
    float ss = 0.f;
    if (have) {
      const float a0 = v[m].x - mean[m], a1 = v[m].y - mean[m], a2 = v[m].z - mean[m], a3 = v[m].w - mean[m];
      ss = (a0 * a0 + a1 * a1) + (a2 * a2 + a3 * a3);
    }
    ss = warp_sum(ss);
    if (lane == 0) red[(MB + m) * MW + warp] = ss;
  }
  stage_sync();
#pragma unroll
  for (int m = 0; m < MB; ++m) {
    float ss = 0.f;
#pragma unroll
    for (int w = 0; w < MW - 1; ++w) ss += red[(MB + m) * MW + w];
    const float rstd = rsqrtf(ss / (float)K + 1e-5f);
    if (have) {
      float4 o;
      o.x = (v[m].x - mean[m]) * rstd * p.g.x + p.b.x;
      o.y = (v[m].y - mean[m]) * rstd * p.g.y + p.b.y;
      o.z = (v[m].z - mean[m]) * rstd * p.g.z + p.b.z;
      o.w = (v[m].w - mean[m]) * rstd * p.g.w + p.b.w;
      *reinterpret_cast<float4*>(xs + m * K + k) = o;
    }
  }
  if (split_end) stage_done_stagers();
  else __syncthreads();
}

// lanes [8r, 8r + MB) finish row n + r  (R <= RMAX = 4, MB <= 8); W8: the row's scale multiplies the dot product first
template <int MB, unsigned VAR, bool W8>
__device__ __forceinline__ void finish_rows(const GemvDesc& d, const float (&acc)[RMAX][MB], float scale, float bias, int n, int M,
                                            float res, bool res_valid, int D, int Tmax, int pos, int lane) {
  const int m = lane & 7, r_sel = lane >> 3;
  const int nn = n + r_sel;
  if (r_sel < d.R && m < MB && m < M && nn < d.nend) {
    float v = 0.f;
#pragma unroll
    for (int r = 0; r < RMAX; ++r) {
#pragma unroll
      for (int mm = 0; mm < MB; ++mm)
        if (r == r_sel && mm == m) v = acc[r][mm];
    }
    if (W8) v *= scale;
    v += bias;
    if (nn < d.alpha_cols) v *= d.alpha;
    if (d.act == 1) v = gelu_erf(v);
    if (d.residual) v += res_valid ? res : __ldcg(d.residual + (long long)m * d.ldo + nn);
    d.out[(long long)m * d.ldo + nn] = v;
    if (d.kc && nn >= D) {
      const long long row = ((long long)m * Tmax + pos) * D;
      if (nn < 2 * D) d.kc[row + nn - D] = f2e(v);
      else d.vc[row + nn - 2 * D] = f2e(v);
    }
  }
}

// smem carve-up (dynamic): red [64] | xs [MB*ffn] | pool: weight slabs from 0, attention scratch from ATT_OFF
// W8: int8 decoder weights (1-byte slab rows, a scale per output row); the static smem is the same in both instantiations
template <int MB, unsigned VAR, bool W8>
__global__ void __launch_bounds__(MT, 1) decode_mega_kernel(const __grid_constant__ MegaArgs a) {
  constexpr bool TRACE = !(VAR & V_NOTRACE);
  constexpr int ESZ = W8 ? 1 : 2;
  extern __shared__ __align__(128) uint8_t dyn[];
  float* red = reinterpret_cast<float*>(dyn);
  float* xs = red + 64;
  uint8_t* pool = reinterpret_cast<uint8_t*>(xs + (size_t)MB * a.ffn);
  uint8_t* att = pool + ATT_OFF;  // only R=1 slabs (<= 30 KB) are live while an attention phase runs
  __shared__ __align__(8) uint64_t wbar[2 * MW];  // per warp: slab barrier (+ second stage for the LM head)
  __shared__ __align__(8) uint64_t xbar;          // cross-attention K/V item
  __shared__ __align__(8) uint64_t cbar[2];       // the CTA's weight slabs of a layer phase (one per slab region)
  __shared__ long long wts[MW][2];                // trace only: per warp, slab landed / rows finished
  // the per-layer pointer table, copied out of the kernel parameter bank once: dynamically indexed constant loads at every
  // phase boundary missed the constant cache (it shares the 32 KB L1.5 with the instruction stream) -- ~1 us per phase
  __shared__ __align__(16) MegaLayer sl[MEGA_MAXL];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gw = blockIdx.x * MW + warp, GW = gridDim.x * MW;
  const int D = a.D, H = a.H, Q = a.Q;
  const int pos0 = *a.pos;
  GridBar<VAR> bar{a.bar, gridDim.x, 0u, a.trace};
  const bool split_end = (a.flags & 64) != 0;  // the DMA warp does not hold up the end of the x staging
  long long* const mkbase = (TRACE && a.trace) ? a.trace + (long long)gridDim.x * MEGA_TRACE_N * 2 + (long long)blockIdx.x * MEGA_TRACE_N * 4 : nullptr;
  auto mark = [&](int j) {
    if (mkbase && threadIdx.x == 0 && bar.epoch < MEGA_TRACE_N) mkbase[bar.epoch * 4 + j] = global_ns();
  };

  const int nsplit = a.nsplit;
  const int ks = (a.S + nsplit - 1) / nsplit;
  const int grp = threadIdx.x >> 3, sub = threadIdx.x & 7;  // KG key groups x 8 lanes
  uint32_t wpar = 0, wpar1 = 0, xpar = 0, cpar0 = 0, cpar1 = 0;                    // mbarrier phase parities

  {
    static_assert(sizeof(MegaLayer) % 8 == 0, "MegaLayer is copied in 8-byte words");
    const unsigned long long* src = reinterpret_cast<const unsigned long long*>(a.layers);
    unsigned long long* dst = reinterpret_cast<unsigned long long*>(sl);
    for (int i = threadIdx.x; i < a.L * (int)(sizeof(MegaLayer) / 8); i += MT) dst[i] = src[i];
  }
  if (threadIdx.x == 0) {
    for (int i = 0; i < 2 * MW; ++i) mbar_init(&wbar[i], 1);
    mbar_init(&xbar, 1);
    mbar_init(&cbar[0], 1);
    mbar_init(&cbar[1], 1);
    fence_mbar_init();
  }
  __syncthreads();

  const int pos = pos0;
  // ---- phase 0: embedding (CTA 0 writes the residual stream); first QKV rows + LN1 params requested meanwhile
  GemvDesc cur = make_desc<VAR, W8>(a, sl, 0, 0, pos);
  Pre pre;
  // Slab regions: GEMV phase ph (= 6*layer + g) lives in region ph & 1 -- region 1 at the pool's start (out-proj, cross
  // out-proj, fc2), region 0 at p0_off (QKV, cross-q, fc1).  Double-buffered (p0_off > 0), the copy for phase ph + 1 is
  // requested at the START of phase ph: it has landed long before its barrier, which then runs at its ~1.1 us floor (a copy
  // requested just before the barrier left 0.3-1.3 us of L2 -> smem transfer exposed behind it).  Attention scratch starts
  // at ATT_OFF, above the small region-1 slabs that are live during the attention phases, and overlays region 0.
  const bool dbuf = a.p0_off > 0;
  issue_slabs<ESZ>(cur, pool + a.p0_off, &cbar[0]);
  prefetch_phase<W8>(cur, pre, pool, &wbar[warp], gw, warp, lane);
  if (blockIdx.x == 0) {
    for (int i = threadIdx.x; i < Q * D; i += MT) {
      const int q = i / D, d = i - q * D;
      const int tok = a.tokens[q * a.Tmax + pos];
      if constexpr (W8)
        a.dx[i] = a.embed_scale[tok] * (float)static_cast<const int8_t*>(a.embed)[(long long)tok * D + d] + a.dec_pos[(long long)pos * D + d];
      else
        a.dx[i] = e2f(static_cast<const bf16*>(a.embed)[(long long)tok * D + d]) + a.dec_pos[(long long)pos * D + d];
    }
  }
  bar.sync();

  const int nph = a.L * 6;
  for (int ph = 0; ph < nph; ++ph) {
    const int l = ph / 6, g = ph - l * 6;
    const MegaLayer& L = sl[l];
    // ---------------- GEMV phase g of layer l ----------------
    {
      const int n = cur.n0 + warp * cur.R;
      const bool active = n < cur.nend;
      float res = 0.f;
      {
        const int m = lane & 7, r_sel = lane >> 3;
        if (cur.residual && active && r_sel < cur.R && m < MB && m < Q && n + r_sel < cur.nend)
          res = __ldcg(cur.residual + (long long)m * cur.ldo + n + r_sel);
      }
      // the DMA warp's turn while x is staged, when the TMA queue is empty: the slab copy of the next phase, and in the QKV
      // phase the L2 prefetch of this layer's cross-attention K/V (DRAM -> L2, three phases before its bulk load)
      auto ahead = [&]() {
        if (dbuf && ph + 1 < nph) {
          const GemvDesc d1 = make_desc<VAR, W8>(a, sl, (ph + 1) / 6, (ph + 1) % 6, pos);
          issue_slabs<ESZ>(d1, pool + (((ph + 1) & 1) ? 0 : a.p0_off), &cbar[(ph + 1) & 1]);
        }
        if (g == 0 && threadIdx.x == DMA_T + 1 && blockIdx.x < Q * H * nsplit) {  // this layer's cross-attention item
          const int item = blockIdx.x;
          const int split = item % nsplit, h = (item / nsplit) % H, q = item / (nsplit * H);
          const int s0 = split * ks;
          const int n = max(0, min(a.S, s0 + ks) - s0);
          if (n > 0) {
            l2_prefetch(L.cross_k + (((long long)q * H + h) * a.S + s0) * 64, (uint32_t)n * 128);
            l2_prefetch(L.cross_v + (((long long)q * H + h) * a.S + s0) * 64, (uint32_t)n * 128);
          }
        }
      };
      stage_x<MB, VAR>(xs, red, cur, pre, Q, split_end, a, g == 3, ahead);
      mark(2);
      if (mkbase && lane == 0) wts[warp][0] = wts[warp][1] = 0;
      if (active) {
        mbar_wait(&cbar[ph & 1], (ph & 1) ? cpar1 : cpar0);
        if (mkbase && lane == 0) wts[warp][0] = global_ns();
        const uint8_t* slab = pool + ((ph & 1) ? 0 : a.p0_off) + (size_t)warp * cur.R * cur.K * ESZ;
        float acc[RMAX][MB];
        if (cur.R == 4) dot_rows<MB, 4, W8>(slab, xs, cur.K, acc, lane);
        else if (cur.R == 3) dot_rows<MB, 3, W8>(slab, xs, cur.K, acc, lane);
        else if (cur.R == 2) dot_rows<MB, 2, W8>(slab, xs, cur.K, acc, lane);
        else dot_rows<MB, 1, W8>(slab, xs, cur.K, acc, lane);
        finish_rows<MB, VAR, W8>(cur, acc, pre.scale, pre.bias, n, Q, res, true, D, a.Tmax, pos, lane);
        if (mkbase && lane == 0) wts[warp][1] = global_ns();
      }
      mark(3);
      if (cur.n0 < cur.nend) {  // (uniform per CTA: the phase's copy was issued iff the CTA owns rows)
        if (ph & 1) cpar1 ^= 1u;
        else cpar0 ^= 1u;
      }
    }
    __syncthreads();  // every warp is done with its slab and with xs: the pool can be re-carved
    bar.arrive();
    if (mkbase && threadIdx.x == 0 && bar.epoch < MEGA_TRACE_N) {
      long long t0 = 0, t1 = 0;
      for (int w = 0; w < MW; ++w) {
        t0 = wts[w][0] > t0 ? wts[w][0] : t0;
        t1 = wts[w][1] > t1 ? wts[w][1] : t1;
      }
      mkbase[bar.epoch * 4 + 0] = t0;
      mkbase[bar.epoch * 4 + 1] = t1;
    }
    cur = make_desc<VAR, W8>(a, sl, ph + 1 < nph ? (ph + 1) / 6 : a.L, (ph + 1) % 6, pos);
    if (!dbuf && !cur.lm) issue_slabs<ESZ>(cur, pool, &cbar[(ph + 1) & 1]);
    prefetch_phase<W8>(cur, pre, pool, &wbar[warp], gw, warp, lane);

    if (g == 0) {
      // past K/V rows of this CTA's self-attention item do not depend on this step: request them now
      if (blockIdx.x < Q * H) {
        const int q = blockIdx.x / H, h = blockIdx.x - q * H;
        uint8_t* sK = att;
        uint8_t* sV = att + (size_t)MAXKEYS * 128;
        for (int s = grp; s < pos; s += KG) {
          const long long off = ((long long)q * a.Tmax + s) * D + h * 64 + sub * 8;
          cp_async16m(sK + s * 128 + sub * 16, L.self_k + off);
          cp_async16m(sV + s * 128 + sub * 16, L.self_v + off);
        }
      }
      bar.wait();
      // ---------------- B: causal self-attention, one (sequence, head) per CTA ----------------
      for (int item = blockIdx.x; item < Q * H; item += gridDim.x) {
        const int q = item / H, h = item - q * H;
        const int n = pos + 1;
        uint8_t* sK = att;
        uint8_t* sV = att + (size_t)MAXKEYS * 128;
        float* redo = reinterpret_cast<float*>(att + (size_t)MAXKEYS * 256);  // [MW][72]
        const int s_first = (item == blockIdx.x) ? pos : 0;  // rows < pos of the first item were prefetched
        for (int s = s_first + grp; s < n; s += KG) {
          const long long off = ((long long)q * a.Tmax + s) * D + h * 64 + sub * 8;
          cp_async16m(sK + s * 128 + sub * 16, L.self_k + off);
          cp_async16m(sV + s * 128 + sub * 16, L.self_v + off);
        }
        float qv[8];
        {
          const float4 q0 = __ldcg(reinterpret_cast<const float4*>(a.dqkv + (long long)q * 3 * D + h * 64 + sub * 8));
          const float4 q1 = __ldcg(reinterpret_cast<const float4*>(a.dqkv + (long long)q * 3 * D + h * 64 + sub * 8 + 4));
          qv[0] = q0.x; qv[1] = q0.y; qv[2] = q0.z; qv[3] = q0.w; qv[4] = q1.x; qv[5] = q1.y; qv[6] = q1.z; qv[7] = q1.w;
        }
        cp_async_wait_allm();
        __syncthreads();  // the row of position `pos` was copied by group 0, whatever group reads it below
        float mx, sum, ov;
        if (n <= 3 * KG) attend_smem<3>(sK, sV, redo, red, qv, n, nullptr, mx, sum, ov);
        else attend_smem<(MAXKEYS + KG - 1) / KG>(sK, sV, redo, red, qv, n, nullptr, mx, sum, ov);
        if (threadIdx.x < 64) a.dattn[(long long)q * D + h * 64 + threadIdx.x] = ov / sum;
        fence_proxy_async_smem();  // this thread's scratch writes (generic proxy) before later TMA writes to the same bytes
        __syncthreads();
      }
      bar.sync();
    } else if (g == 2) {
      // the encoder K/V slice of this CTA's first cross-attention item is constant during decoding: request it now
      // (contiguous in the head-major cross cache: one bulk copy each)
      if (threadIdx.x == 0 && blockIdx.x < Q * H * nsplit) {
        const int item = blockIdx.x;
        const int split = item % nsplit, h = (item / nsplit) % H, q = item / (nsplit * H);
        const int s0 = split * ks;
        const int n = max(0, min(a.S, s0 + ks) - s0);
        mbar_arrive_expect_tx(&xbar, (uint32_t)n * 256);
        if (n > 0) {
          bulk_g2s(att, L.cross_k + (((long long)q * H + h) * a.S + s0) * 64, (uint32_t)n * 128, &xbar);
          bulk_g2s(att + XKMAX * 128, L.cross_v + (((long long)q * H + h) * a.S + s0) * 64, (uint32_t)n * 128, &xbar);
        }
      }
      bar.wait();
      // ---------------- E: cross-attention, (audio, head, key split) items; phase F merges the splits ----------------
      {
        uint8_t* sK = att;
        uint8_t* sV = att + XKMAX * 128;
        float* redo = reinterpret_cast<float*>(att + 2 * XKMAX * 128);  // [MW][72]
        for (int item = blockIdx.x; item < Q * H * nsplit; item += gridDim.x) {
          const int split = item % nsplit;
          const int h = (item / nsplit) % H;
          const int q = item / (nsplit * H);
          const int s0 = split * ks;
          const int n = max(0, min(a.S, s0 + ks) - s0);
          if (item != blockIdx.x && threadIdx.x == 0) {  // later items of this CTA were not prefetched
            mbar_arrive_expect_tx(&xbar, (uint32_t)n * 256);
            if (n > 0) {
              bulk_g2s(sK, L.cross_k + (((long long)q * H + h) * a.S + s0) * 64, (uint32_t)n * 128, &xbar);
              bulk_g2s(sV, L.cross_v + (((long long)q * H + h) * a.S + s0) * 64, (uint32_t)n * 128, &xbar);
            }
          }
          float qv[8];
          {
            const float4 q0 = __ldcg(reinterpret_cast<const float4*>(a.dq + (long long)q * D + h * 64 + sub * 8));
            const float4 q1 = __ldcg(reinterpret_cast<const float4*>(a.dq + (long long)q * D + h * 64 + sub * 8 + 4));
            qv[0] = q0.x; qv[1] = q0.y; qv[2] = q0.z; qv[3] = q0.w; qv[4] = q1.x; qv[5] = q1.y; qv[6] = q1.z; qv[7] = q1.w;
          }
          float* align_row = nullptr;
          if (a.align && L.head_slots) {
            const int slot = L.head_slots[h];
            const int step = pos - a.step_base;
            if (slot >= 0 && step >= 0 && step < a.Tcap) align_row = a.align + (((long long)q * a.Ha + slot) * a.Tcap + step) * a.S + s0;
          }
          mbar_wait(&xbar, xpar);
          xpar ^= 1u;
          mark(0);
          if (mkbase && threadIdx.x == 0 && bar.epoch < MEGA_TRACE_N) mkbase[bar.epoch * 4 + 2] = clock64();
          float mx, sum, ov;
          attend_smem<(XKMAX + KG - 1) / KG>(sK, sV, redo, red, qv, n, align_row, mx, sum, ov,
                                             (mkbase && bar.epoch < MEGA_TRACE_N) ? mkbase + bar.epoch * 4 : nullptr);
          // the split's partials: every CTA's cross out-projection staging merges them after the barrier (merge_xattn)
          const long long pb = ((long long)q * H + h) * nsplit + split;
          if (threadIdx.x < 64) a.part_o[pb * 64 + threadIdx.x] = ov;
          if (threadIdx.x == 0) {
            a.part_ml[pb * 2 + 0] = mx;
            a.part_ml[pb * 2 + 1] = sum;
          }
          fence_proxy_async_smem();
          __syncthreads();
        }
      }
      bar.sync();
    } else {
      bar.wait();
    }
  }

  // ---------------- final LayerNorm + tied LM head: row pairs, two slab stages per warp ----------------
  stage_x<MB, VAR>(xs, red, cur, pre, Q, split_end, a, false, [] {});
  unsigned long long best = 0ull;  // of the logits this lane finished: (order-preserving value bits << 32) | ~token
  {
    const int K = cur.K, N = cur.N;
    const size_t slab_bytes = (size_t)2 * K * ESZ;
    const size_t set_bytes = slab_bytes * MW;
    int buf = 0;
    const bool at_begin = (pos + 1 == a.begin_index) && a.begin_suppress_bits;
    for (int n = gw * 2; n < N; n += GW * 2) {
      const int n2 = n + GW * 2;
      if (n2 < N) {
        __syncwarp();  // every lane is done reading the stage that is refilled now
        issue_rows<ESZ>(pool + (buf ^ 1) * set_bytes + (size_t)warp * slab_bytes, &wbar[(buf ^ 1) * MW + warp], cur.W, K, 2, n2, N, lane);
      }
      float sc = 1.f;  // W8: scale of the row this lane finishes (requested before the slab wait)
      if constexpr (W8) sc = cur.scale[min(n + (lane >> 3), N - 1)];
      if (buf == 0) {
        mbar_wait(&wbar[warp], wpar);
        wpar ^= 1u;
      } else {
        mbar_wait(&wbar[MW + warp], wpar1);
        wpar1 ^= 1u;
      }
      float acc[RMAX][MB];
      dot_rows<MB, 2, W8>(pool + buf * set_bytes + (size_t)warp * slab_bytes, xs, K, acc, lane);
      finish_rows<MB, VAR, W8>(cur, acc, sc, 0.f, n, Q, 0.f, true, D, a.Tmax, pos, lane);
      if (a.fuse_select) {
        const int m = lane & 7, r_sel = lane >> 3, nn = n + r_sel;
        if (r_sel < 2 && m < MB && m < Q && nn < N) {
          float v = 0.f;
#pragma unroll
          for (int r = 0; r < 2; ++r)
#pragma unroll
            for (int mm = 0; mm < MB; ++mm)
              if (r == r_sel && mm == m) v = acc[r][mm];
          if (W8) v *= sc;
          bool masked = (a.suppress_bits[nn >> 5] >> (nn & 31)) & 1u;
          if (at_begin) masked = masked || ((a.begin_suppress_bits[nn >> 5] >> (nn & 31)) & 1u);
          if (!masked) {
            unsigned u = __float_as_uint(v);
            u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
            const unsigned long long key = ((unsigned long long)u << 32) | (unsigned long long)(0xffffffffu - (unsigned)nn);
            best = key > best ? key : best;
          }
        }
      }
      buf ^= 1;
    }
  }
  if (a.fuse_select) {
    // lanes m and 8 + m hold sequence m's candidates; fold per warp, per CTA, then one atomicMax per CTA and sequence
    {
      const unsigned long long o = __shfl_xor_sync(0xffffffffu, best, 8);
      best = o > best ? o : best;
    }
    unsigned long long* sb = reinterpret_cast<unsigned long long*>(xs);  // x is no longer needed: [MB][MW]
    __syncthreads();
    if (lane < MB) sb[lane * MW + warp] = best;
    __syncthreads();
    if (threadIdx.x < MB && threadIdx.x < Q) {
      unsigned long long b = 0ull;
      for (int w = 0; w < MW; ++w) b = sb[threadIdx.x * MW + w] > b ? sb[threadIdx.x * MW + w] : b;
      if (b) atomicMax(a.sel_best + threadIdx.x, b);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      const unsigned prev = atom_acq_rel_add(a.sel_ctr, 1u);
      if (prev == gridDim.x - 1) {  // every CTA's maxima are in: this is SelectArgs' greedy branch (decode.cu select_kernel)
        const int cur_len = pos + 1;
        const bool generating = cur_len >= a.begin_index && cur_len < a.Tmax;
        for (int q = 0; q < Q; ++q) {
          const unsigned long long b = __ldcg(a.sel_best + q);
          a.sel_best[q] = 0ull;
          if (generating) {
            int choice = (int)(0xffffffffu - (unsigned)(b & 0xffffffffull));
            if (a.finished[q]) choice = a.pad;
            else if (choice == a.eos) a.finished[q] = 1;
            a.tokens_rw[q * a.Tmax + cur_len] = choice;
          }
        }
        *a.sel_ctr = 0u;
        *a.pos_rw = pos + 1;
      }
    }
  }
  if (TRACE && a.trace && bar.epoch < MEGA_TRACE_N) {  // end of this CTA's LM-head share
    __syncthreads();
    if (threadIdx.x == 0) a.trace[((long long)blockIdx.x * MEGA_TRACE_N + bar.epoch) * 2] = global_ns();
  }
}

}  // namespace

int g_mega_coop = -1;  // -1: read BW_MEGA_COOP on first use; the engine clears it if a cooperative launch cannot be captured

namespace {

template <int MB, unsigned VAR, bool W8>
int launch_mega(cudaStream_t st, const MegaArgs& a, int num_sms, int coop) {
  // the shared-memory budget: the device's opt-in limit per block less this instantiation's static smem, read once
  static size_t limit = 0, attr = 0;
  if (!limit) {
    int dev = 0, optin = 0;
    BW_CUDA_OK(cudaGetDevice(&dev));
    BW_CUDA_OK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    cudaFuncAttributes fa{};
    BW_CUDA_OK(cudaFuncGetAttributes(&fa, decode_mega_kernel<MB, VAR, W8>));
    limit = (size_t)optin - fa.sharedSizeBytes;
  }
  MegaArgs b = a;
  const size_t smem = mega_smem_plan(MB, a.D, a.ffn, num_sms, !(a.flags & 2), limit, &b.p0_off, W8 ? 1 : 2);
  if (!smem) return -3;
  if (smem > attr) {
    BW_CUDA_OK(cudaFuncSetAttribute(decode_mega_kernel<MB, VAR, W8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    BW_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, decode_mega_kernel<MB, VAR, W8>, MT, smem));
    if (per_sm < 1) return -3;
    attr = smem;
  }
  BW_CUDA_OK(cudaMemsetAsync(a.bar, 0, 1024 * sizeof(unsigned), st));
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(num_sms); cfg.blockDim = dim3(MT); cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeCooperative; at[0].val.cooperative = 1;
  cfg.attrs = at; cfg.numAttrs = coop ? 1 : 0;
  BW_CUDA_OK(cudaLaunchKernelEx(&cfg, decode_mega_kernel<MB, VAR, W8>, b));
  return 0;
}

}  // namespace

// Launches the persistent step kernel on `st`.  Returns -3 when the configuration is outside what it supports
// (the caller then uses the per-op path).
int launch_decode_mega(cudaStream_t st, const MegaArgs& a, int num_sms) {
  const int Q = a.Q;
  const bool w8 = a.embed_scale != nullptr;
  const size_t esz = w8 ? 1 : 2;
  if (a.L > MEGA_MAXL || Q > 2 || a.D > MAXD || a.ffn > 5120 || a.D % 8 != 0 || a.ffn % 8 != 0 || a.Tmax > MAXKEYS) return -3;
  if ((size_t)MW * a.D * esz > (size_t)ATT_OFF) return -3;  // R=1 slabs must stay below the attention scratch
  {  // every layer GEMV is one pass of at most RMAX rows per warp
    const int nmax = 3 * a.D > a.ffn ? 3 * a.D : a.ffn;
    if (((nmax + num_sms - 1) / num_sms + MW - 1) / MW > RMAX) return -3;
  }
  if (a.nsplit > XSPLIT) return -3;
  if ((size_t)((a.D + num_sms - 1) / num_sms) * a.D * esz > (size_t)ATT_OFF) return -3;  // region-1 slabs live under the attention scratch
  const int ks = (a.S + a.nsplit - 1) / a.nsplit;
  if (ks > XKMAX) return -3;
  // Co-residency of the CTAs (one per SM) (round-1 advisor): the grid barriers spin, so a CTA that is not scheduled deadlocks the rest until
  // the 2^32-cycle timeout traps.  (1) the occupancy calculator must promise one CTA per SM, else -3 (per-op path); (2) the launch is
  // cooperative, so the driver either runs the whole grid at once or fails the launch (another kernel holding SMs: an error code at
  // the C-ABI, not a poisoned context).  BW_MEGA_COOP=0 falls back to the plain launch of round 1.
  int& coop = g_mega_coop;
  if (coop < 0) {
    const char* ev = getenv("BW_MEGA_COOP");
    coop = (ev && ev[0] == '0') ? 0 : 1;
  }
  // the instrumented instantiation only when a trace buffer is attached (BW_MEGA_TRACE=1)
  int rc;
  if (w8) {
    if (Q <= 1) rc = a.trace ? launch_mega<1, 0u, true>(st, a, num_sms, coop) : launch_mega<1, V_NOTRACE, true>(st, a, num_sms, coop);
    else rc = a.trace ? launch_mega<2, 0u, true>(st, a, num_sms, coop) : launch_mega<2, V_NOTRACE, true>(st, a, num_sms, coop);
  } else {
    if (Q <= 1) rc = a.trace ? launch_mega<1, 0u, false>(st, a, num_sms, coop) : launch_mega<1, V_NOTRACE, false>(st, a, num_sms, coop);
    else rc = a.trace ? launch_mega<2, 0u, false>(st, a, num_sms, coop) : launch_mega<2, V_NOTRACE, false>(st, a, num_sms, coop);
  }
  if (rc) return rc;
  BW_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace bw
