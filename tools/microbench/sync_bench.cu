// Microbenchmarks of the synchronisation / hand-over primitives a persistent one-CTA-per-SM decoder step is built from.
// Every test runs a grid of one 384-thread CTA per SM through N rounds and reports ns per round (globaltimer of CTA 0).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o sync_bench sync_bench.cu && ./sync_bench
// The numbers decide which hand-over the decoder-step kernel should use (profiles/r1_v8_sync_microbench.md).
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(1); } } while (0)

constexpr int MT = 384;
constexpr int NV = 1280;   // values handed from all CTAs to all CTAs per round
constexpr int XT = 320;    // consumer threads (4 values each)

__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) { unsigned v; asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ unsigned ld_relaxed(const unsigned* p) { unsigned v; asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ void red_release(unsigned* p, unsigned v) { asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void red_relaxed(unsigned* p, unsigned v) { asm volatile("red.relaxed.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void st_relaxed64(unsigned long long* p, unsigned long long v) { asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ void ld_relaxed64x2(const unsigned long long* p, unsigned long long& a, unsigned long long& b) {
  asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}
__device__ __forceinline__ long long gns() { long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t; }
__device__ __forceinline__ void guard(long long t0, int what) {
  if (clock64() - t0 > (1ll << 31)) { printf("timeout in test %d block %d thread %d\n", what, blockIdx.x, threadIdx.x); __trap(); }
}

struct Args {
  unsigned* ctr;              // barrier counter(s)
  float* x;                   // [2][NV] plain values
  unsigned long long* ll;     // [2][NV] tagged words, or mailboxes [grid][2][NV]
  long long* out_ns;          // [0] total ns
  float* sink;
  int rounds;
  int mode;
};

// grid barrier: last thread arrives (red.release) and polls (ld.acquire)
__device__ __forceinline__ void grid_barrier(unsigned* ctr, unsigned& epoch, int mode) {
  __syncthreads();
  if (threadIdx.x == MT - 1) {
    if (mode == 1) { __threadfence(); red_relaxed(ctr, 1u); }
    else red_release(ctr, 1u);
    const unsigned target = (epoch + 1) * gridDim.x;
    const long long t0 = clock64();
    while (ld_acquire(ctr) < target) guard(t0, 1);
  }
  ++epoch;
  __syncthreads();
}

// test 0/1: barrier only (mode 1: __threadfence + relaxed red).  test 2: barrier + every CTA writes its share of x, then all read x.
__global__ void __launch_bounds__(MT, 1) k_barrier(Args a) {
  extern __shared__ unsigned char dyn[];
  unsigned epoch = 0;
  const int per = (NV + gridDim.x - 1) / gridDim.x;
  float acc = 0.f;
  grid_barrier(a.ctr, epoch, 0);
  const long long t0 = gns();
  for (int it = 0; it < a.rounds; ++it) {
    if (a.mode == 2) {
      float* xb = a.x + (it & 1) * NV;
      const int i = blockIdx.x * per + threadIdx.x;
      if ((int)threadIdx.x < per && i < NV) xb[i] = acc * 1e-9f + (float)it;
    }
    grid_barrier(a.ctr, epoch, a.mode == 1 ? 1 : 0);
    if (a.mode == 2 && threadIdx.x < XT) {
      const float4 v = __ldcg(reinterpret_cast<const float4*>(a.x + (it & 1) * NV) + threadIdx.x);
      acc += v.x + v.y + v.z + v.w;
    }
  }
  const long long t1 = gns();
  if (blockIdx.x == 0 && threadIdx.x == 0) a.out_ns[0] = t1 - t0;
  if (acc == 123.456f) a.sink[0] = acc;
}

// test 3/4/5: flag-in-data all-to-all: every CTA publishes its share as {tag, value} words, every CTA polls all NV words.
// mode 3: 320 threads poll 4 words each, spinning; mode 4: same with __nanosleep(40) between rounds;
// mode 5: push -- every producer writes its share into EVERY consumer's private mailbox, consumers poll only their own lines
__global__ void __launch_bounds__(MT, 1) k_ll(Args a) {
  extern __shared__ unsigned char dyn[];
  unsigned epoch = 0;
  const int per = (NV + gridDim.x - 1) / gridDim.x;
  float acc = 0.f;
  grid_barrier(a.ctr, epoch, 0);
  const long long t0 = gns();
  for (int it = 0; it < a.rounds; ++it) {
    const unsigned tag = (unsigned)it + 1u;
    if (a.mode == 5) {
      // per values x gridDim mailboxes, spread over the CTA's threads
      for (int j = threadIdx.x; j < per * (int)gridDim.x; j += MT) {
        const int dst = j / per, r = j - dst * per;
        const int i = blockIdx.x * per + r;
        if (i < NV) st_relaxed64(a.ll + ((size_t)dst * 2 + (it & 1)) * NV + i, ((unsigned long long)tag << 32) | __float_as_uint(acc * 1e-9f + (float)it));
      }
    } else {
      const int i = blockIdx.x * per + threadIdx.x;
      if ((int)threadIdx.x < per && i < NV) st_relaxed64(a.ll + (size_t)(it & 1) * NV + i, ((unsigned long long)tag << 32) | __float_as_uint(acc * 1e-9f + (float)it));
    }
    if (threadIdx.x < XT) {
      const unsigned long long* p = (a.mode == 5 ? a.ll + ((size_t)blockIdx.x * 2 + (it & 1)) * NV : a.ll + (size_t)(it & 1) * NV) + threadIdx.x * 4;
      unsigned long long w0, w1, w2, w3;
      const long long tt = clock64();
      for (;;) {
        ld_relaxed64x2(p, w0, w1);
        ld_relaxed64x2(p + 2, w2, w3);
        if ((unsigned)(w0 >> 32) >= tag && (unsigned)(w1 >> 32) >= tag && (unsigned)(w2 >> 32) >= tag && (unsigned)(w3 >> 32) >= tag) break;
        if (a.mode == 4) __nanosleep(40);
        guard(tt, 3);
      }
      acc += __uint_as_float((unsigned)w0) + __uint_as_float((unsigned)w1) + __uint_as_float((unsigned)w2) + __uint_as_float((unsigned)w3);
    }
    __syncthreads();  // (a phase of the real kernel ends with a CTA barrier too)
  }
  const long long t1 = gns();
  if (blockIdx.x == 0 && threadIdx.x == 0) a.out_ns[0] = t1 - t0;
  if (acc == 123.456f) a.sink[0] = acc;
}

// test 6: ping-pong between CTA 0 and CTA (grid-1): one-way latency of a relaxed 64-bit store seen by a relaxed poll
__global__ void __launch_bounds__(MT, 1) k_pingpong(Args a) {
  if (threadIdx.x != 0) return;
  const int peer = gridDim.x - 1;
  if (blockIdx.x != 0 && (int)blockIdx.x != peer) return;
  unsigned long long* mine = a.ll + (blockIdx.x == 0 ? 0 : 64);
  unsigned long long* theirs = a.ll + (blockIdx.x == 0 ? 64 : 0);
  const long long t0 = gns();
  for (int it = 1; it <= a.rounds; ++it) {
    if (blockIdx.x == 0) st_relaxed64(theirs, (unsigned long long)it);
    const long long tt = clock64();
    unsigned long long v;
    do { asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(mine) : "memory"); guard(tt, 6); } while (v < (unsigned long long)it);
    if (blockIdx.x != 0) st_relaxed64(theirs, (unsigned long long)it);
  }
  const long long t1 = gns();
  if (blockIdx.x == 0) a.out_ns[0] = t1 - t0;
}

// test 7: CTA-local costs: __syncthreads with 384 threads, and a dependent chain of L2 loads (ld.cg) by one warp
__global__ void __launch_bounds__(MT, 1) k_local(Args a) {
  __shared__ float s[MT];
  float acc = 0.f;
  long long t0 = clock64();
  for (int it = 0; it < a.rounds; ++it) { s[threadIdx.x] = acc; __syncthreads(); acc += s[(threadIdx.x + 1) % MT]; __syncthreads(); }
  long long t1 = clock64();
  if (blockIdx.x == 0 && threadIdx.x == 0) a.out_ns[0] = (t1 - t0);
  // dependent L2 loads: pointer chase through a.x (indices stored as floats), all CTAs at once (contended) 
  int idx = (threadIdx.x * 4 + blockIdx.x * 16) % NV;
  t0 = clock64();
  for (int it = 0; it < a.rounds; ++it) { const float v = __ldcg(a.x + idx); idx = ((int)v + idx + 64) % NV; }
  t1 = clock64();
  if (blockIdx.x == 0 && threadIdx.x == 0) a.out_ns[1] = (t1 - t0);
  if (acc == 123.456f || idx < 0) a.sink[0] = acc;
}

// test 8/9/10: grid barrier variants.  mode 8: no atomics -- CTA b stores its epoch into slot b of a packed array (148 x 4 B),
// lanes 0..36 of the last warp poll the whole array with 16-byte loads; mode 9 / 10: the counter sharded 8 / 4 ways
// (128 bytes apart), 8 / 4 lanes poll.
__global__ void __launch_bounds__(MT, 1) k_barrier2(Args a) {
  extern __shared__ unsigned char dyn[];
  float acc = 0.f;
  unsigned epoch = 0;
  grid_barrier(a.ctr + 1024 - 32, epoch, 0);
  epoch = 0;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long t0 = gns();
  for (int it = 0; it < a.rounds; ++it) {
    __syncthreads();
    if (a.mode == 8) {
      if (warp == MT / 32 - 1) {
        if (lane == 31) { __threadfence(); asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(a.ctr + blockIdx.x), "r"(epoch + 1) : "memory"); }
        const int nq = ((int)gridDim.x + 3) / 4;  // 16-byte groups
        const long long tt = clock64();
        for (;;) {
          bool ok = true;
          for (int q = lane; q < nq; q += 32) {
            uint4 v;
            asm volatile("ld.relaxed.gpu.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(a.ctr + q * 4) : "memory");
            const int b = q * 4;
            ok = ok && v.x > epoch && (b + 1 >= (int)gridDim.x || v.y > epoch) && (b + 2 >= (int)gridDim.x || v.z > epoch) && (b + 3 >= (int)gridDim.x || v.w > epoch);
          }
          if (__all_sync(0xffffffffu, ok)) break;
          guard(tt, 8);
        }
        __threadfence();
      }
    } else {
      const int ng = a.mode == 9 ? 8 : 4;
      if (threadIdx.x == MT - 1) red_release(a.ctr + (blockIdx.x % ng) * 32, 1u);
      if (warp == MT / 32 - 1 && lane < ng) {
        const unsigned cnt = (gridDim.x - lane + ng - 1) / ng;
        const unsigned target = (epoch + 1) * cnt;
        const long long tt = clock64();
        for (;;) {
          const bool ok = ld_acquire(a.ctr + lane * 32) >= target;
          if (__all_sync((1u << ng) - 1u, ok)) break;
          guard(tt, 9);
        }
      }
    }
    ++epoch;
    __syncthreads();
  }
  const long long t1 = gns();
  if (blockIdx.x == 0 && threadIdx.x == 0) a.out_ns[0] = t1 - t0;
  if (acc == 123.456f) a.sink[0] = acc;
}

// test 11: flag-in-data WITH A HINT.  Producers store their share as {tag, value} words (relaxed), then -- no fence -- one thread
// stores the tag into the CTA's slot of a packed hint array.  Consumers: the last warp polls the 592-byte hint array (cheap),
// then the 320 consumer threads read their 4 words ONCE and verify the tags (re-polling only if a word is late: correctness
// never depends on the hint).  mode 12: same, but the consumers skip the hint and the data is read after a plain grid barrier
// whose arrival has NO release fence (red.relaxed) -- data validity again by tags.
__global__ void __launch_bounds__(MT, 1) k_hint(Args a) {
  extern __shared__ unsigned char dyn[];
  unsigned epoch = 0;
  const int per = (NV + gridDim.x - 1) / gridDim.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float acc = 0.f;
  grid_barrier(a.ctr + 1024 - 32, epoch, 0);
  epoch = 0;
  unsigned retries = 0;
  const long long t0 = gns();
  for (int it = 0; it < a.rounds; ++it) {
    const unsigned tag = (unsigned)it + 1u;
    {
      const int i = blockIdx.x * per + threadIdx.x;
      if ((int)threadIdx.x < per && i < NV) st_relaxed64(a.ll + (size_t)(it & 1) * NV + i, ((unsigned long long)tag << 32) | __float_as_uint(acc * 1e-9f + (float)it));
    }
    __syncthreads();
    if (a.mode == 11) {
      if (warp == MT / 32 - 1) {
        if (lane == 31) asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(a.ctr + blockIdx.x), "r"(tag) : "memory");
        const int nq = ((int)gridDim.x + 3) / 4;
        const long long tt = clock64();
        for (;;) {
          bool ok = true;
          for (int q = lane; q < nq; q += 32) {
            uint4 v;
            asm volatile("ld.relaxed.gpu.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(a.ctr + q * 4) : "memory");
            const int b = q * 4;
            ok = ok && v.x >= tag && (b + 1 >= (int)gridDim.x || v.y >= tag) && (b + 2 >= (int)gridDim.x || v.z >= tag) && (b + 3 >= (int)gridDim.x || v.w >= tag);
          }
          if (__all_sync(0xffffffffu, ok)) break;
          guard(tt, 11);
        }
      }
    } else {
      if (threadIdx.x == MT - 1) {
        red_relaxed(a.ctr, 1u);
        const unsigned target = (epoch + 1) * gridDim.x;
        const long long tt = clock64();
        while (ld_relaxed(a.ctr) < target) guard(tt, 12);
      }
      ++epoch;
    }
    __syncthreads();
    if (threadIdx.x < XT) {
      const unsigned long long* p = a.ll + (size_t)(it & 1) * NV + threadIdx.x * 4;
      unsigned long long w0, w1, w2, w3;
      const long long tt = clock64();
      for (;;) {
        ld_relaxed64x2(p, w0, w1);
        ld_relaxed64x2(p + 2, w2, w3);
        if ((unsigned)(w0 >> 32) >= tag && (unsigned)(w1 >> 32) >= tag && (unsigned)(w2 >> 32) >= tag && (unsigned)(w3 >> 32) >= tag) break;
        ++retries;
        guard(tt, 13);
      }
      acc += __uint_as_float((unsigned)w0) + __uint_as_float((unsigned)w1) + __uint_as_float((unsigned)w2) + __uint_as_float((unsigned)w3);
    }
    __syncthreads();
  }
  const long long t1 = gns();
  if (blockIdx.x == 0 && threadIdx.x == 0) a.out_ns[0] = t1 - t0;
  if (retries) atomicAdd(reinterpret_cast<unsigned long long*>(a.out_ns + 2), (unsigned long long)retries);
  if (acc == 123.456f) a.sink[0] = acc;
}

// test 13: partial barrier -- only `nprod` CTAs arrive (red.release), every CTA polls (what stands between an attention phase
// with 20 producer CTAs and the out-projection that needs all heads).  test 14: point-to-point -- 20 counters, counter h gets
// 8 arrivals (the CTAs that produce head h's rows) and is polled by 7 CTAs (the key splits of head h); the other CTAs idle.
__global__ void __launch_bounds__(MT, 1) k_partial(Args a) {
  extern __shared__ unsigned char dyn[];
  unsigned epoch = 0;
  grid_barrier(a.ctr + 1024 - 32, epoch, 0);
  const long long t0 = gns();
  for (int it = 0; it < a.rounds; ++it) {
    __syncthreads();
    if (a.mode == 13) {
      const int nprod = 20;
      if (threadIdx.x == MT - 1) {
        if ((int)blockIdx.x < nprod) red_release(a.ctr, 1u);
        const unsigned target = (unsigned)(it + 1) * nprod;
        const long long tt = clock64();
        while (ld_acquire(a.ctr) < target) guard(tt, 13);
      }
    } else {
      // producers: CTA b signals head (b * 20 / gridDim) -- about gridDim/20 arrivals per head; pollers: CTA b < 140 polls head b / 7
      const int H = 20;
      const int hp = (int)((long long)blockIdx.x * H / gridDim.x);
      if (threadIdx.x == MT - 1) {
        red_release(a.ctr + 32 * hp, 1u);
        if ((int)blockIdx.x < H * 7) {
          const int hc = blockIdx.x / 7;
          unsigned cnt = 0;
          for (int b = 0; b < (int)gridDim.x; ++b) cnt += ((int)((long long)b * H / gridDim.x) == hc);
          const unsigned target = (unsigned)(it + 1) * cnt;
          const long long tt = clock64();
          while (ld_acquire(a.ctr + 32 * hc) < target) guard(tt, 14);
        }
      }
      // (a full barrier every 64 rounds keeps the non-polling CTAs from running ahead without bound)
      if ((it & 63) == 63) grid_barrier(a.ctr + 1024 - 32, epoch, 0);
    }
    __syncthreads();
  }
  const long long t1 = gns();
  if (blockIdx.x == 0 && threadIdx.x == 0) a.out_ns[0] = t1 - t0;
}

// test 16: fp32 reductions through L2: 140 CTAs each add 64 partial values into each of ... -- the pattern of an out-projection
// fused into the attention phase: CTA (h, j) adds its 183-row slice of head h's contribution: 1280 addresses x 20 contributions.
// Reports ns per round including the grid barrier that follows (compare with test 0).
__global__ void __launch_bounds__(MT, 1) k_redf32(Args a) {
  extern __shared__ unsigned char dyn[];
  unsigned epoch = 0;
  grid_barrier(a.ctr, epoch, 0);
  const long long t0 = gns();
  for (int it = 0; it < a.rounds; ++it) {
    if (blockIdx.x < 140) {
      const int j = blockIdx.x % 7;          // row slice of this CTA
      const int r0 = j * 183;
      for (int r = threadIdx.x; r < 183 && r0 + r < NV; r += MT) atomicAdd(a.x + (it & 1) * NV + r0 + r, 1.0f);
    }
    grid_barrier(a.ctr, epoch, 0);
  }
  const long long t1 = gns();
  if (blockIdx.x == 0 && threadIdx.x == 0) a.out_ns[0] = t1 - t0;
}

// test 15: hand-over inside a thread-block cluster through distributed shared memory: every CTA writes 16 floats into the smem
// of every CTA of its cluster (st.shared::cluster), then barrier.cluster arrive.release / wait.acquire; ns per round.
template <int CS>
__global__ void __launch_bounds__(MT, 1) k_cluster(Args a) {
  __shared__ float box[8][16];
  unsigned rank, nctas;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
  asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(nctas));
  float acc = 0.f;
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
  const long long t0 = gns();
  for (int it = 0; it < a.rounds; ++it) {
    if (threadIdx.x < 16 * nctas) {
      const unsigned dst = threadIdx.x / 16, i = threadIdx.x % 16;
      unsigned local = (unsigned)__cvta_generic_to_shared(&box[rank][i]);
      unsigned remote;
      asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local), "r"(dst));
      asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(remote), "f"(acc + (float)it) : "memory");
    }
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
    if (threadIdx.x < 16 * nctas) acc += box[threadIdx.x / 16][threadIdx.x % 16] * 1e-9f;
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
  }
  const long long t1 = gns();
  if (blockIdx.x == 0 && threadIdx.x == 0) a.out_ns[0] = t1 - t0;
  if (acc == 123.456f) a.sink[0] = acc;
}

__global__ void k_empty(Args a) {
  if (a.rounds == -1) a.sink[0] = 1.f;
}

int main() {
  int dev = 0, sms = 0, khz = 0;
  CK(cudaSetDevice(dev));
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  CK(cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, dev));
  printf("SMs %d, max clock %.0f MHz\n", sms, khz / 1e3);
  Args a{};
  CK(cudaMalloc(&a.ctr, 4096));
  CK(cudaMalloc(&a.x, 2 * NV * sizeof(float)));
  const size_t ll_words = (size_t)sms * 2 * NV;
  CK(cudaMalloc(&a.ll, ll_words * 8));
  CK(cudaMalloc(&a.out_ns, 64));
  CK(cudaMalloc(&a.sink, 64));
  CK(cudaMemset(a.x, 0, 2 * NV * sizeof(float)));
  const int smem = 200 * 1024;
  CK(cudaFuncSetAttribute(k_barrier, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  CK(cudaFuncSetAttribute(k_ll, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  CK(cudaFuncSetAttribute(k_empty, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const char* names[] = {"grid barrier (red.release + ld.acquire poll)", "grid barrier (__threadfence + red.relaxed)",
                         "barrier + all-to-all of 1280 floats (write share, barrier, every CTA reads 5 KB)",
                         "flag-in-data all-to-all, 320 pollers per CTA spinning", "flag-in-data all-to-all, pollers with nanosleep(40)",
                         "flag-in-data PUSH into per-consumer mailboxes (148 x 1280 words), pollers read private lines"};
  for (int rep = 0; rep < 2; ++rep) {
    for (int mode = 0; mode < 6; ++mode) {
      a.mode = mode;
      a.rounds = 2000;
      CK(cudaMemset(a.ctr, 0, 4096));
      CK(cudaMemset(a.ll, 0, ll_words * 8));
      if (mode <= 2) k_barrier<<<sms, MT, smem>>>(a);
      else k_ll<<<sms, MT, smem>>>(a);
      CK(cudaGetLastError());
      CK(cudaDeviceSynchronize());
      long long ns = 0;
      CK(cudaMemcpy(&ns, a.out_ns, 8, cudaMemcpyDeviceToHost));
      if (rep == 1) printf("test %d: %7.1f ns / round   %s\n", mode, (double)ns / a.rounds, names[mode]);
    }
  }
  CK(cudaFuncSetAttribute(k_barrier2, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  CK(cudaFuncSetAttribute(k_hint, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const char* names2[] = {"grid barrier without atomics: per-CTA epoch slots (592 B), one warp polls with 16-byte loads",
                          "grid barrier, counter sharded 8 ways (8 polling lanes)", "grid barrier, counter sharded 4 ways",
                          "flag-in-data all-to-all WITH HINT array (no fence): poll 592 B, then read + verify 10 KB once",
                          "flag-in-data all-to-all after a fence-less barrier (red.relaxed + ld.relaxed), tags verify"};
  for (int rep = 0; rep < 2; ++rep) {
    for (int mode = 8; mode <= 12; ++mode) {
      a.mode = mode;
      a.rounds = 2000;
      CK(cudaMemset(a.ctr, 0, 4096));
      CK(cudaMemset(a.ll, 0, ll_words * 8));
      CK(cudaMemset(a.out_ns, 0, 64));
      if (mode <= 10) k_barrier2<<<sms, MT, smem>>>(a);
      else k_hint<<<sms, MT, smem>>>(a);
      CK(cudaGetLastError());
      CK(cudaDeviceSynchronize());
      long long ns[3] = {0, 0, 0};
      CK(cudaMemcpy(ns, a.out_ns, 24, cudaMemcpyDeviceToHost));
      if (rep == 1) printf("test %d: %7.1f ns / round   %s%s\n", mode, (double)ns[0] / a.rounds, names2[mode - 8],
                           mode >= 11 ? (ns[2] ? "  [some words were late: re-polled]" : "  [no re-polls]") : "");
      if (rep == 1 && mode >= 11) printf("         late-word re-polls: %lld over %d rounds x %d threads\n", ns[2], a.rounds, sms * XT);
    }
  }
  CK(cudaFuncSetAttribute(k_partial, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  CK(cudaFuncSetAttribute(k_redf32, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  for (int mode : {13, 14, 16}) {
    for (int rep = 0; rep < 2; ++rep) {
      a.mode = mode;
      a.rounds = 2000;
      CK(cudaMemset(a.ctr, 0, 4096));
      CK(cudaMemset(a.x, 0, 2 * NV * sizeof(float)));
      if (mode == 16) k_redf32<<<sms, MT, smem>>>(a);
      else k_partial<<<sms, MT, smem>>>(a);
      CK(cudaGetLastError());
      CK(cudaDeviceSynchronize());
      long long ns = 0;
      CK(cudaMemcpy(&ns, a.out_ns, 8, cudaMemcpyDeviceToHost));
      if (rep == 1)
        printf("test %d: %7.1f ns / round   %s\n", mode, (double)ns / a.rounds,
               mode == 13 ? "partial barrier: 20 CTAs arrive, all 148 poll"
                          : (mode == 14 ? "point-to-point: 20 counters, ~7 arrivals and 7 pollers each"
                                        : "25.6 k fp32 atomicAdd into 1280 addresses (20 per address) + grid barrier"));
    }
  }
  {  // test 15: cluster hand-over through DSMEM
    a.rounds = 2000;
    auto run_cluster = [&](int cs) {
      cudaLaunchConfig_t cfg = {};
      const int grid = sms / cs * cs;
      cfg.gridDim = dim3(grid);
      cfg.blockDim = dim3(MT);
      cfg.dynamicSmemBytes = 0;
      cudaLaunchAttribute at[1];
      at[0].id = cudaLaunchAttributeClusterDimension;
      at[0].val.clusterDim.x = cs;
      at[0].val.clusterDim.y = 1;
      at[0].val.clusterDim.z = 1;
      cfg.attrs = at;
      cfg.numAttrs = 1;
      cudaError_t e = cudaSuccess;
      for (int rep = 0; rep < 2 && e == cudaSuccess; ++rep) {
        if (cs == 2) e = cudaLaunchKernelEx(&cfg, k_cluster<2>, a);
        else if (cs == 4) e = cudaLaunchKernelEx(&cfg, k_cluster<4>, a);
        else e = cudaLaunchKernelEx(&cfg, k_cluster<8>, a);
        if (e == cudaSuccess) e = cudaDeviceSynchronize();
      }
      if (e != cudaSuccess) { printf("test 15: cluster size %d: %s\n", cs, cudaGetErrorString(e)); cudaGetLastError(); return; }
      long long ns = 0;
      CK(cudaMemcpy(&ns, a.out_ns, 8, cudaMemcpyDeviceToHost));
      printf("test 15: %7.1f ns / round   cluster of %d: DSMEM all-to-all of 16 floats + 2 cluster barriers (grid %d)\n", (double)ns / a.rounds, cs, grid);
    };
    run_cluster(2);
    run_cluster(4);
    run_cluster(8);
  }
  {  // test 17: what a launch boundary costs: back-to-back launches of an empty kernel, and of a memset + kernel graph
    a.rounds = 0;
    cudaStream_t st;
    CK(cudaStreamCreate(&st));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    const int n = 2000;
    for (int rep = 0; rep < 2; ++rep) {
      CK(cudaEventRecord(e0, st));
      for (int i = 0; i < n; ++i) k_empty<<<sms, MT, 0, st>>>(a);
      CK(cudaEventRecord(e1, st));
      CK(cudaStreamSynchronize(st));
    }
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    printf("test 17: %7.2f us per back-to-back launch of an empty %d x %d kernel\n", ms * 1e3 / n, sms, MT);
    cudaGraph_t g;
    cudaGraphExec_t ge;
    CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    CK(cudaMemsetAsync(a.ctr, 0, 4096, st));
    k_empty<<<sms, MT, smem, st>>>(a);
    CK(cudaStreamEndCapture(st, &g));
    CK(cudaGraphInstantiate(&ge, g, 0));
    for (int rep = 0; rep < 2; ++rep) {
      CK(cudaEventRecord(e0, st));
      for (int i = 0; i < n; ++i) CK(cudaGraphLaunch(ge, st));
      CK(cudaEventRecord(e1, st));
      CK(cudaStreamSynchronize(st));
    }
    CK(cudaEventElapsedTime(&ms, e0, e1));
    printf("test 17: %7.2f us per launch of a (4 KB memset + empty kernel with 200 KB smem) graph -- the per-token boundary of the decoder\n", ms * 1e3 / n);
  }
  for (int grid : {2, sms}) {
    a.rounds = 2000;
    CK(cudaMemset(a.ll, 0, ll_words * 8));
    k_pingpong<<<grid, MT>>>(a);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    long long ns = 0;
    CK(cudaMemcpy(&ns, a.out_ns, 8, cudaMemcpyDeviceToHost));
    printf("test 6: %7.1f ns one-way (store -> visible to a polling thread), CTA 0 <-> CTA %d\n", (double)ns / a.rounds / 2, grid - 1);
  }
  {
    a.rounds = 1000;
    k_local<<<sms, MT>>>(a);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    long long c[2];
    CK(cudaMemcpy(c, a.out_ns, 16, cudaMemcpyDeviceToHost));
    printf("test 7: %.1f cycles per (smem write, __syncthreads, smem read, __syncthreads) with 384 threads; %.1f cycles per dependent ld.global.cg (all CTAs loading)\n",
           (double)c[0] / a.rounds, (double)c[1] / a.rounds);
  }
  return 0;
}
