// Fused log-mel front end for sm_90a: reflect-pad framing + periodic Hann window + 400-point FFT + |.|^2 +
// sparse slaney mel filter bank + log10, then the per-sample dynamic-range clamp and (x+4)/4.
//
// Replaces WhisperFeatureExtractor._torch_extract_fbank_features, which the reference runs with torch.stft on the
// CPU (TF/models/whisper/feature_extraction_whisper.py:135-164; frame layout of torch.stft(center=True,
// pad_mode="reflect"), n_fft=400, hop=160, last frame dropped :150).
//
// Kernel 1 (logmel_frames): one warp per frame, 6 warps per CTA.  The 400-point complex FFT is a mixed-radix
// Stockham autosort (radices 4,4,5,5) that ping-pongs between two per-warp smem buffers; twiddles come from an
// exact fp64-computed table.  Power spectrum -> 128 mel filters from a CSR copy of the (sparse, <= ~24 nnz/filter)
// bank -> log10(max(.,1e-10)) written time-major, plus an atomicMax per audio for the "max - 8" clamp.
// Kernel 2 (logmel_finalize): clamp, (x+4)/4, bf16 time-major output with a zero row either side (the conv
// stem reads it as an im2col view through TMA), optionally the fp32 [mel, frame] layout of the reference.
// HBM-bound by design: 1.92 MB PCM in + 0.77 MB bf16 out per 30 s chunk (SURVEY.md §8d).
#include <math.h>

#include <vector>

#include "kernels.h"

namespace BW_NS {

namespace {
constexpr int NFFT = 400;
constexpr int HOP = 160;
constexpr int NBINS = 201;
constexpr int WARPS = 6;  // 6 x 6.4 KB FFT ping-pong buffers + tables < 48 KB static smem
constexpr int MAXW = 32;  // max non-zeros per mel filter supported
}  // namespace

struct LogmelPlan {
  int n_mels = 0;
  float2* tw = nullptr;     // [400] exp(-2*pi*i*k/400)
  float* window = nullptr;  // [400] periodic hann
  int* fstart = nullptr;    // [n_mels]
  int* flen = nullptr;      // [n_mels]
  float* fw = nullptr;      // [n_mels][MAXW]
};

namespace {

__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }

template <int R>
__device__ __forceinline__ void small_dft(float2 (&v)[R]);

template <>
__device__ __forceinline__ void small_dft<4>(float2 (&v)[4]) {
  const float2 a = make_float2(v[0].x + v[2].x, v[0].y + v[2].y);
  const float2 b = make_float2(v[0].x - v[2].x, v[0].y - v[2].y);
  const float2 c = make_float2(v[1].x + v[3].x, v[1].y + v[3].y);
  const float2 d = make_float2(v[1].x - v[3].x, v[1].y - v[3].y);  // times -i below
  v[0] = make_float2(a.x + c.x, a.y + c.y);
  v[2] = make_float2(a.x - c.x, a.y - c.y);
  v[1] = make_float2(b.x + d.y, b.y - d.x);  // b - i d
  v[3] = make_float2(b.x - d.y, b.y + d.x);  // b + i d
}

template <>
__device__ __forceinline__ void small_dft<5>(float2 (&v)[5]) {
  // w^k = exp(-2*pi*i*k/5)
  const float c1 = 0.30901699437494742f, s1 = 0.95105651629515357f;
  const float c2 = -0.80901699437494742f, s2 = 0.58778525229247313f;
  const float2 a1 = make_float2(v[1].x + v[4].x, v[1].y + v[4].y), b1 = make_float2(v[1].x - v[4].x, v[1].y - v[4].y);
  const float2 a2 = make_float2(v[2].x + v[3].x, v[2].y + v[3].y), b2 = make_float2(v[2].x - v[3].x, v[2].y - v[3].y);
  const float2 x0 = v[0];
  v[0] = make_float2(x0.x + a1.x + a2.x, x0.y + a1.y + a2.y);
  const float2 t1 = make_float2(x0.x + c1 * a1.x + c2 * a2.x, x0.y + c1 * a1.y + c2 * a2.y);
  const float2 t2 = make_float2(x0.x + c2 * a1.x + c1 * a2.x, x0.y + c2 * a1.y + c1 * a2.y);
  // -i * (s1 b1 + s2 b2) and -i * (s2 b1 - s1 b2)
  const float2 u1 = make_float2(s1 * b1.x + s2 * b2.x, s1 * b1.y + s2 * b2.y);
  const float2 u2 = make_float2(s2 * b1.x - s1 * b2.x, s2 * b1.y - s1 * b2.y);
  v[1] = make_float2(t1.x + u1.y, t1.y - u1.x);
  v[4] = make_float2(t1.x - u1.y, t1.y + u1.x);
  v[2] = make_float2(t2.x + u2.y, t2.y - u2.x);
  v[3] = make_float2(t2.x - u2.y, t2.y + u2.x);
}

// one Stockham stage over the whole warp: N/R butterflies, lane-strided
template <int R>
__device__ __forceinline__ void fft_stage(const float2* __restrict__ src, float2* __restrict__ dst, const float2* __restrict__ tw,
                                          int Ns, int lane) {
  constexpr int NB = NFFT / R;
  const int tstep = NFFT / (Ns * R);
  for (int j = lane; j < NB; j += 32) {
    const int k = j % Ns;
    float2 v[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      v[r] = src[j + r * NB];
      if (r > 0 && k > 0) v[r] = cmul(v[r], tw[(r * k * tstep) % NFFT]);
    }
    small_dft<R>(v);
    const int d = (j / Ns) * Ns * R + k;
#pragma unroll
    for (int r = 0; r < R; ++r) dst[d + r * Ns] = v[r];
  }
}

__device__ __forceinline__ unsigned f2ord(float f) {
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(unsigned o) {
  const unsigned u = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
  return __uint_as_float(u);
}

__global__ void __launch_bounds__(WARPS * 32)
logmel_frames_kernel(LogmelPlan plan, const float* __restrict__ pcm, int n_samples, int frames, float* __restrict__ scratch,
                     long long f_stride, long long m_stride, unsigned* __restrict__ smax) {
  __shared__ float2 s_tw[NFFT];
  __shared__ float s_win[NFFT];
  __shared__ float2 s_buf[WARPS][2][NFFT];
  __shared__ float s_wmax[WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.y;
  for (int i = threadIdx.x; i < NFFT; i += blockDim.x) {
    s_tw[i] = plan.tw[i];
    s_win[i] = plan.window[i];
  }
  __syncthreads();
  const float* x = pcm + (long long)b * n_samples;
  float2* b0 = s_buf[warp][0];
  float2* b1 = s_buf[warp][1];
  float wmax = -INFINITY;
  const int f = blockIdx.x * WARPS + warp;
  if (f < frames) {
    // frame f covers samples [f*160 - 200, f*160 + 200) of the reflect-padded signal
    const int start = f * HOP - NFFT / 2;
    for (int i = lane; i < NFFT; i += 32) {
      int idx = start + i;
      if (idx < 0) idx = -idx;
      if (idx >= n_samples) idx = 2 * (n_samples - 1) - idx;
      b0[i] = make_float2(x[idx] * s_win[i], 0.f);
    }
    __syncwarp();
    fft_stage<4>(b0, b1, s_tw, 1, lane);
    __syncwarp();
    fft_stage<4>(b1, b0, s_tw, 4, lane);
    __syncwarp();
    fft_stage<5>(b0, b1, s_tw, 16, lane);
    __syncwarp();
    fft_stage<5>(b1, b0, s_tw, 80, lane);
    __syncwarp();
    // power spectrum of bins 0..200 into b1 (as floats)
    float* pw = reinterpret_cast<float*>(b1);
    for (int i = lane; i < NBINS; i += 32) pw[i] = b0[i].x * b0[i].x + b0[i].y * b0[i].y;
    __syncwarp();
    // log10 of (audio b, frame f, mel m) goes to scratch[b * frames * n_mels + f * f_stride + m * m_stride]: time-major rows
    // (f_stride = n_mels, m_stride = 1) on the chunk path, the reference's [mel][frame] layout (f_stride = 1, m_stride = frames)
    // on the long path, which then finalizes in place
    float* orow = scratch + (long long)b * frames * plan.n_mels + f * f_stride;
    for (int mth = lane; mth < plan.n_mels; mth += 32) {
      const int s = plan.fstart[mth], n = plan.flen[mth];
      const float* w = plan.fw + mth * MAXW;
      float acc = 0.f;
      for (int i = 0; i < n; ++i) acc = fmaf(w[i], pw[s + i], acc);
      const float lv = log10f(fmaxf(acc, 1e-10f));
      orow[mth * m_stride] = lv;
      wmax = fmaxf(wmax, lv);
    }
  }
  wmax = warp_max(wmax);
  if (lane == 0) s_wmax[warp] = wmax;
  __syncthreads();
  if (threadIdx.x == 0) {
    float mx = s_wmax[0];
    for (int i = 1; i < WARPS; ++i) mx = fmaxf(mx, s_wmax[i]);
    if (mx > -INFINITY) atomicMax(&smax[b], f2ord(mx));
  }
}

// scratch [B][frames][n_mels] fp32 -> out_tm [B][frames+2][n_mels] bf16 (+ optional out_f32 [B][n_mels][frames])
__global__ void logmel_finalize_kernel(const float* __restrict__ scratch, const unsigned* __restrict__ smax, int frames, int n_mels,
                                       bf16* __restrict__ out_tm, float* __restrict__ out_f32) {
  __shared__ float tile[32][129];
  const int b = blockIdx.y;
  const int f0 = blockIdx.x * 32;
  const float floor_v = ord2f(smax[b]) - 8.0f;
  for (int i = threadIdx.x; i < 32 * n_mels; i += blockDim.x) {
    const int ff = i / n_mels, mth = i % n_mels;
    const int f = f0 + ff;
    float v = 0.f;
    if (f < frames) {
      v = scratch[((long long)b * frames + f) * n_mels + mth];
      v = (fmaxf(v, floor_v) + 4.0f) / 4.0f;
      out_tm[((long long)b * (frames + 2) + f + 1) * n_mels + mth] = f2e(v);
    }
    if (mth < 128) tile[ff][mth] = v;
  }
  if (blockIdx.x == 0) {  // zero the two padding rows
    for (int i = threadIdx.x; i < n_mels; i += blockDim.x) {
      out_tm[((long long)b * (frames + 2)) * n_mels + i] = f2e(0.f);
      out_tm[((long long)b * (frames + 2) + frames + 1) * n_mels + i] = f2e(0.f);
    }
  }
  if (out_f32) {
    __syncthreads();
    for (int i = threadIdx.x; i < 32 * n_mels; i += blockDim.x) {
      const int mth = i / 32, ff = i % 32;
      if (f0 + ff < frames) out_f32[((long long)b * n_mels + mth) * frames + f0 + ff] = tile[ff][mth];
    }
  }
}

// long path: x [B][n_mels][frames] fp32 in place -> (max(x, max_b - 8) + 4) / 4, the arithmetic of logmel_finalize_kernel
__global__ void logmel_finalize_inplace_kernel(float* __restrict__ x, const unsigned* __restrict__ smax, long long per_audio) {
  const int b = blockIdx.y;
  const float floor_v = ord2f(smax[b]) - 8.0f;
  float* xb = x + (long long)b * per_audio;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < per_audio; i += (long long)gridDim.x * blockDim.x)
    xb[i] = (fmaxf(xb[i], floor_v) + 4.0f) / 4.0f;
}

}  // namespace

int logmel_plan_create_from_bank(LogmelPlan** out, const float* bank /*[201][n_mels] row-major*/, int n_mels) {
  BW_CHECK(n_mels > 0 && n_mels <= 128, "logmel: n_mels=%d unsupported (1..128)", n_mels);
  LogmelPlan* p = new LogmelPlan();
  p->n_mels = n_mels;
  std::vector<float2> tw(NFFT);
  std::vector<float> win(NFFT);
  for (int k = 0; k < NFFT; ++k) {
    const double a = -2.0 * M_PI * (double)k / NFFT;
    tw[k] = make_float2((float)cos(a), (float)sin(a));
    win[k] = (float)(0.5 - 0.5 * cos(2.0 * M_PI * (double)k / NFFT));  // torch.hann_window(400) (periodic)
  }
  std::vector<int> fs(n_mels), fl(n_mels);
  std::vector<float> fw((size_t)n_mels * MAXW, 0.f);
  for (int m = 0; m < n_mels; ++m) {
    int lo = NBINS, hi = -1;
    for (int k = 0; k < NBINS; ++k)
      if (bank[(size_t)k * n_mels + m] != 0.f) {
        if (k < lo) lo = k;
        hi = k;
      }
    if (hi < 0) { lo = 0; hi = -1; }
    const int n = hi - lo + 1;
    if (n > MAXW) {
      delete p;
      BW_CHECK(false, "logmel: mel filter %d spans %d bins (> %d)", m, n, MAXW);
    }
    fs[m] = lo;
    fl[m] = n;
    for (int i = 0; i < n; ++i) fw[(size_t)m * MAXW + i] = bank[(size_t)(lo + i) * n_mels + m];
  }
  BW_CUDA_OK(cudaMalloc(&p->tw, sizeof(float2) * NFFT));
  BW_CUDA_OK(cudaMalloc(&p->window, sizeof(float) * NFFT));
  BW_CUDA_OK(cudaMalloc(&p->fstart, sizeof(int) * n_mels));
  BW_CUDA_OK(cudaMalloc(&p->flen, sizeof(int) * n_mels));
  BW_CUDA_OK(cudaMalloc(&p->fw, sizeof(float) * n_mels * MAXW));
  BW_CUDA_OK(cudaMemcpy(p->tw, tw.data(), sizeof(float2) * NFFT, cudaMemcpyHostToDevice));
  BW_CUDA_OK(cudaMemcpy(p->window, win.data(), sizeof(float) * NFFT, cudaMemcpyHostToDevice));
  BW_CUDA_OK(cudaMemcpy(p->fstart, fs.data(), sizeof(int) * n_mels, cudaMemcpyHostToDevice));
  BW_CUDA_OK(cudaMemcpy(p->flen, fl.data(), sizeof(int) * n_mels, cudaMemcpyHostToDevice));
  BW_CUDA_OK(cudaMemcpy(p->fw, fw.data(), sizeof(float) * n_mels * MAXW, cudaMemcpyHostToDevice));
  *out = p;
  return 0;
}

void logmel_plan_destroy(LogmelPlan* p) {
  if (!p) return;
  cudaFree(p->tw);
  cudaFree(p->window);
  cudaFree(p->fstart);
  cudaFree(p->flen);
  cudaFree(p->fw);
  delete p;
}

int logmel(cudaStream_t st, const LogmelPlan* plan, const float* pcm, int B, int n_samples, int frames, bf16* out_tm,
           float* out_f32, float* scratch, unsigned* scratch_max) {
  BW_CHECK(plan != nullptr, "logmel: null plan");
  BW_CHECK(n_samples >= NFFT, "logmel: n_samples=%d too short", n_samples);
  BW_CHECK(frames * HOP <= n_samples, "logmel: frames=%d exceeds n_samples/160", frames);
  BW_CUDA_OK(cudaMemsetAsync(scratch_max, 0, sizeof(unsigned) * B, st));
  dim3 g1((frames + WARPS - 1) / WARPS, B);
  logmel_frames_kernel<<<g1, WARPS * 32, 0, st>>>(*plan, pcm, n_samples, frames, scratch, plan->n_mels, 1, scratch_max);
  BW_CUDA_OK(cudaGetLastError());
  dim3 g2((frames + 31) / 32, B);
  logmel_finalize_kernel<<<g2, 256, 0, st>>>(scratch, scratch_max, frames, plan->n_mels, out_tm, out_f32);
  BW_CUDA_OK(cudaGetLastError());
  return 0;
}

int logmel_long(cudaStream_t st, const LogmelPlan* plan, const float* pcm, int B, int n_samples, float* out_f32, unsigned* scratch_max) {
  BW_CHECK(plan != nullptr && out_f32 != nullptr, "logmel_long: null plan or output");
  BW_CHECK(n_samples >= NFFT, "logmel_long: n_samples=%d too short", n_samples);
  const int frames = n_samples / HOP;
  BW_CUDA_OK(cudaMemsetAsync(scratch_max, 0, sizeof(unsigned) * B, st));
  dim3 g1((frames + WARPS - 1) / WARPS, B);
  logmel_frames_kernel<<<g1, WARPS * 32, 0, st>>>(*plan, pcm, n_samples, frames, out_f32, 1, frames, scratch_max);
  BW_CUDA_OK(cudaGetLastError());
  const long long per_audio = (long long)plan->n_mels * frames;
  const long long blocks = (per_audio + 255) / 256;
  dim3 g2((unsigned)(blocks < 1024 ? blocks : 1024), B);
  logmel_finalize_inplace_kernel<<<g2, 256, 0, st>>>(out_f32, scratch_max, per_audio);
  BW_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace bw
