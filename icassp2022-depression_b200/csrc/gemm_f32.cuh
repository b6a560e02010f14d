// gemm_f32.cuh — interface of the fp32 time-parallel GEMMs (input projection K1, wgrad/dgrad K6).
#pragma once
#include "common.cuh"

namespace b200rnn {

// C(m,n) (+)= sum_k A(m,k) * B(k,n) + bias1[n] + (n < bias2_n ? bias2[n] : 0)
struct GemmParams {
  const float* A;
  RowMap a_rows;  // a_kcontig: row index = m (k contiguous); else row index = k (m contiguous)
  int a_kcontig;
  const float* B;
  RowMap b_rows;  // b_kcontig: row index = n (k contiguous); else row index = k (n contiguous)
  int b_kcontig;
  float* C;
  RowMap c_rows;  // row index = m, n contiguous
  int M, N, K;
  const float* bias1;
  const float* bias2;
  int bias2_n;
  int accumulate;
  // optional workspace for the tensor-core 3xTF32 path (gemm_tc.cu); NULL => fp32 FFMA path
  void* tc_ws;
  size_t tc_ws_bytes;
  int tc_a_presplit;  // the A operand's hi/lo halves already sit at tc_ws (see tc_a_hi / tc_a_lo)
  // optional: the B operand (a weight matrix) already split into dense [N,K] hi / lo matrices by an earlier call
  // (b200rnn_prepare_weights: frozen encoders split their W_ih once, not once per step)
  const float* tc_b_hi;
  const float* tc_b_lo;
};

// where launch_gemm_tc expects / puts the split A operand inside its workspace
float* tc_a_hi(void* ws);
float* tc_a_lo(void* ws, int M, int K);
// LayerNorm over the last dimension fused with the TF32 split: hi/lo <- split(LN(src row) * gamma + beta)
// `out` (optional): dense [R][Cc] copy of LN(src) kept for the backward pass (layer-0 wgrad operand)
int tc_layernorm_split(const float* src, const RowMap& rows, int R, int Cc, const float* gamma, const float* beta,
                       float eps, float* hi, float* lo, cudaStream_t stream, float* out = nullptr);
// backward of that prologue: dx (strided like x) from dy = d/dLN(x) (dense), dgamma / dbeta (+)=; part = scratch of
// layernorm_bwd_scratch_floats(Cc) floats
size_t layernorm_bwd_scratch_floats(int Cc);
int launch_layernorm_bwd(const float* x, const RowMap& x_rows, const float* dy, int R, int Cc, const float* gamma,
                         float eps, float* dx, const RowMap& dx_rows, float* dgamma, float* dbeta, int accumulate,
                         float* part, cudaStream_t stream);

// tensor-core (wgmma) 3xTF32 path: C = A[M,K] * B[N,K]^T + biases (both operands k-contiguous, K % 32 == 0, N % 128 == 0)
size_t gemm_tc_scratch_bytes(int M, int N, int K);
bool gemm_tc_eligible(const GemmParams& p, size_t ws_bytes);
int launch_gemm_tc(const GemmParams& p, void* ws, size_t ws_bytes, cudaStream_t stream);

// Building blocks of the tensor-core path for callers that manage the split operands themselves (backward pass).
struct TcOperand {
  const float* hi;
  const float* lo;
  long long ld;  // floats between consecutive rows (multiple of 4)
  bool mn = false;  // false: K-major, dense [M or N rows][K]; true: MN-major, dense [K rows][M or N] (no transpose needed
                    // for operands whose contraction index is their row index: dG, X, h_prev in the wgrad GEMMs)
};
bool tc_available();
int tc_split(const float* src, const RowMap& rows, int R, int Cc, float* hi, float* lo, cudaStream_t stream);
int tc_gemm_presplit(const TcOperand& A, const TcOperand& B, int M, int N, int K, float* C, const RowMap& c_rows,
                     const float* bias1, const float* bias2, int bias2_n, int accumulate, void* splitk_ws,
                     size_t splitk_ws_bytes, cudaStream_t stream);
// C(m,n) (+)= sum_z partial[z][m][n] (+ biases), fixed order (deterministic)
int launch_splitk_reduce(const float* partial, int splitk, int M, int N, float* C, const RowMap& c_rows,
                         const float* bias1, const float* bias2, int bias2_n, int accumulate, cudaStream_t stream);

// bytes of scratch launch_gemm may use for split-K partials for this problem (0 if none wanted)
size_t gemm_scratch_bytes(int M, int N, int K);

// Enqueue on `stream`. `scratch` may be NULL (then no split-K). Returns B200RNN_* code.
int launch_gemm(const GemmParams& p, void* scratch, size_t scratch_bytes, cudaStream_t stream);

}  // namespace b200rnn
