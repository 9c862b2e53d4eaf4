// Internal launcher declarations (host side).  The public C-ABI is include/thewhisper_b200.h.
#pragma once
#include "common.cuh"

namespace BW_NS {

// ---------------------------------------------------------------------------------------------
// wgmma GEMM: C[b,t,n] = epilogue( sum_k A(b,t,k) * W[n,k] ), bf16 operands, fp32 accumulate in registers
// ---------------------------------------------------------------------------------------------
// A operand view.  Element (b, t, k) lives at base[b*batch_stride + (t + k / kwrap) * pitch + (k % kwrap)].
//   plain row-major activations : kwrap >= K, pitch = row length
//   conv1 (k=3, s=1) im2col     : base = time-major padded mel [B][T+2][128], pitch = 128,  kwrap = 128
//   conv2 (k=3, s=2) im2col     : base = padded h1 viewed as [B][(T+2)/2][2*D], pitch = 2*D, kwrap = 2*D
// so the convolutions are plain GEMMs whose TMA coordinates wrap; nothing is materialised.
struct GemmA {
  const bf16* base = nullptr;
  long long batch_stride = 0;  // elements
  long long pitch = 0;         // elements, multiple of 8
  int rows_base = 0;           // rows per item that exist in memory (TMA bound; beyond -> zero fill)
  int kwrap = 0x7fffffff;      // multiple of 64 when < K
};

struct GemmEpi {
  const float* bias = nullptr;      // [N] fp32 or null
  float alpha = 1.0f;               // (acc + bias) * alpha for columns n < alpha_cols (q-projection scaling; alpha_cols % 32 == 0)
  int alpha_cols = 0x7fffffff;
  int act = 0;                      // 0 none, 1 exact-erf GELU
  const float* residual = nullptr;  // fp32, same addressing as the output; may alias out_f32 (in-place x += ...)
  const float* pos = nullptr;       // fp32 [rows, N] added after the activation (encoder positional table)
  float* out_f32 = nullptr;         // exactly one of out_f32 / out_bf16
  bf16* out_bf16 = nullptr;
  // element offset of (b, t, n): b*batch_stride + t*row_stride + (n / 64)*head_stride + (n % 64)
  // plain row-major [B*rows, ld]: batch_stride = rows*ld, row_stride = ld, head_stride = 64.
  long long batch_stride = 0;
  long long row_stride = 0;
  long long head_stride = 64;
  int n_valid = 0;  // rows of W that exist in memory (0 = N); rows beyond are zero-filled by TMA (tied LM head: V = 51866 of N = 51872)
};

// W: [N, K] bf16 row-major (torch Linear layout).  K % 64 == 0, N % 32 == 0.  rows = output rows per item.
int gemm_tc(cudaStream_t st, const GemmA& a, const bf16* W, int B, int rows, int N, int K, const GemmEpi& epi,
            int force_bn /*0 = auto, else 32/64/128/256*/);
// Split-K form for the decoder's residual GEMMs (K >> N / SM-count tiles): grid.z = ksplit, split z writes raw fp32 partial sums at
// out_f32 + z * split_stride; the consumer (resid_ln) adds them in a fixed order.  ksplit is clamped so that every split owns a k-block (gemm_tc_ksplit gives the count used).
int gemm_tc_split(cudaStream_t st, const GemmA& a, const bf16* W, int B, int rows, int N, int K, const GemmEpi& epi, int force_bn,
                  int ksplit, long long split_stride);
int gemm_tc_ksplit(int K, int ksplit);
// Encoder GEMM over flat rows (the gemm_tc kernel, B = 1): 128 x BN tiles across item boundaries, epilogues specialised per use.
// A [M, K] plain row-major; the epilogue address map splits the flat row r as b = r / rows_per_item, t = r % rows_per_item
// (rows_per_item <= 0: one item).  No conv wrap, no positional table.  force_bn: 0 auto, 128, 256 (+ 1000: generic epilogue, tests).
bool gemm_tc2_supported(int M, int N, int K);
int gemm_tc2(cudaStream_t st, const bf16* A, const bf16* W, int M, int N, int K, int rows_per_item, const GemmEpi& epi, int force_bn);
// CUDA-core sibling with identical semantics: on-device comparator for the tests and the bring-up fallback
// selected by BW_GEMM_IMPL=simt (never the default).
int gemm_simt(cudaStream_t st, const GemmA& a, const bf16* W, int B, int rows, int N, int K, const GemmEpi& epi);

// ---------------------------------------------------------------------------------------------
// decoder-step projections (gemm_dec.cu): weights are the 128-row MMA operand, the Q activation rows the N operand, K split
// across CTAs so that one launch is one DRAM round trip.  ksplit > 1: raw fp32 partial sums at out_f32 + z * split_stride
// ([split][q][n], row pitch epi.row_stride); ksplit == 1: bias / alpha (columns < alpha_cols) / GELU applied, fp32 or bf16 out.
// ---------------------------------------------------------------------------------------------
struct DecGemmPlan {
  int QB = 16, q_tiles = 1, stages = 2, kper = 1, ksplit = 1;
  size_t smem = 0;
};
DecGemmPlan gemm_dec_plan(int Q, int N, int K, int num_sms, bool want_split, bool w8 = false);
// W: [N, K] 16-bit, or int8 codes with a scale per row (wscale != nullptr; plan with w8 = true)
int gemm_dec(cudaStream_t st, const bf16* X, const void* W, const float* wscale, int Q, int N, int K, int n_valid, const GemmEpi& epi,
             const DecGemmPlan& pl, long long split_stride);
// h[q, n] = bf16(GELU(sum_s part[s][q][n] + bias[n]))
int launch_gelu_bias(cudaStream_t st, const float* part, int nsplit, long long split_stride, const float* bias, bf16* h, int Q, int N);

// ---------------------------------------------------------------------------------------------
// encoder attention (non-causal).  qkv: [B*S, 3*D] bf16 (q pre-scaled by dh^-1/2), vt: [B, H, 64, Spad] bf16
// (zero beyond S), out: [B*S, D] bf16.  head_dim is 64 for every Whisper size.
// ---------------------------------------------------------------------------------------------
// same kernel; vt == nullptr reads V straight from the qkv rows (MN-major operand) instead of the transposed copy
int attn_enc_tc(cudaStream_t st, const bf16* qkv, const bf16* vt, bf16* out, int B, int S, int Spad, int H);
int attn_enc_simt(cudaStream_t st, const bf16* qkv, bf16* out, int B, int S, int H);
int transpose_v(cudaStream_t st, const bf16* qkv, bf16* vt, int B, int S, int Spad, int H);

// ---------------------------------------------------------------------------------------------
// small / memory-bound kernels
// ---------------------------------------------------------------------------------------------
int layernorm_bf16(cudaStream_t st, const float* x, const float* g, const float* b, bf16* y, int rows, int D);
int layernorm_f32(cudaStream_t st, const float* x, const float* g, const float* b, float* y, int rows, int D);

struct LogmelPlan;  // opaque: filter bank + twiddles on device
int logmel_plan_create_from_bank(LogmelPlan** out, const float* bank /*[201][n_mels]*/, int n_mels);
void logmel_plan_destroy(LogmelPlan* p);
// pcm: [B, n_samples] fp32 on device (already padded/truncated to the chunk); out_tm: [B, frames+2, n_mels]
// bf16 time-major with one zero row of padding each side (the conv stem's im2col view);
// out_f32 (optional): [B, n_mels, frames] fp32 in the reference layout for parity tests.
// scratch: B*(n_mels*frames) floats + B uints.
int logmel(cudaStream_t st, const LogmelPlan* plan, const float* pcm, int B, int n_samples, int frames, bf16* out_tm,
           float* out_f32, float* scratch, unsigned* scratch_max);
// any sample count: pcm [B, n_samples] (rows zero-padded to the longest) -> out_f32 [B, n_mels, n_samples / 160] fp32 only (the
// reference layout; log10 values are written there and finalized in place, no scratch).  scratch_max: B uints.
int logmel_long(cudaStream_t st, const LogmelPlan* plan, const float* pcm, int B, int n_samples, float* out_f32, unsigned* scratch_max);

}  // namespace bw
