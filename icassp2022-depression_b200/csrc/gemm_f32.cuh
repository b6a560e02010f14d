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
  int tc_a_f32;  // A (k-contiguous) is read in fp32 through a_rows and split on chip; needs tc_a_f32_in_place
  // optional: the B operand (a weight matrix) already split into dense [N,K] hi / lo matrices by an earlier call
  // (b200rnn_prepare_weights: frozen encoders split their W_ih once, not once per step)
  const float* tc_b_hi;
  const float* tc_b_lo;
  // optional, tensor-core path only: streamed launch. ready[m] counts the finished n-tiles of row tile m (TC_TILE_M
  // rows); the tiles are walked time-major by tc_stream_clusters 4-CTA clusters, and the launch lets the next kernel
  // in the stream start early (the forward recurrence, which waits on these counters). The counters must be zero on
  // entry.
  int* tc_ready;
  int tc_stream_clusters;
  // tensor-core path only: single-pass TF32 (one MMA per k-step on operands rounded to TF32; B200RNN_FLAG_TF32)
  // instead of 3xTF32. Only tc_b_hi of a presplit weight is read, and a per-call split writes hi only.
  int tc_tf32;
  // tensor-core fp32-A path only: fp16 pairs (gemm_f16x3_kernel, the no-grad forward of b200rnn_forward_fused) when the
  // shape allows (g16::shape_ok), else 3xTF32. tc_b_h16 (optional): W already split into fp16 pairs
  // (gemm_h16_layout.cuh, b200rnn_prepare_weights); else the call splits W into its workspace.
  int tc_h16;
  const void* tc_b_h16;
  // the forward input projection only (else NULL): where its A operand comes from, named on the B200RNN_DEBUG line.
  // "tma" (read in place through a_rows), "gather" (dense copy), "ln" (the LayerNorm prologue's output), "widen" (fp32
  // copy of a 16-bit operand). Host side only.
  const char* a_route;
};

// where launch_gemm_tc puts the split A operand inside its workspace (tc_a_hi: also room for a dense fp32 [M][K] A)
float* tc_a_hi(void* ws);
float* tc_a_lo(void* ws, int M, int K);
// whether the fp32-A GEMM can read A[M][K] in place through `rows` (dense, or a [T][B] view with B dividing 128 or a
// multiple of it; 16-byte aligned base and strides)
bool tc_a_f32_in_place(const float* A, const RowMap& rows, int M, int K);
// dense fp32 copy dst[R][Cc] <- rows of src, for an A operand that cannot be read in place
// `clear` (optional): nclear ints zeroed by the same launch (the ready counters of a streamed GEMM that reads dst)
int tc_gather_rows(const float* src, const RowMap& rows, int R, int Cc, float* dst, cudaStream_t stream,
                   int* clear = nullptr, int nclear = 0);
// LayerNorm over the last dimension: out[R][Cc] <- LN(src row) * gamma + beta (dense fp32: the A operand of the
// input projection, and when kept, the layer-0 wgrad operand of the backward pass)
// `clear` (optional): nclear ints zeroed by the same launch (the ready counters of a streamed GEMM that reads out)
// `lengths` (optional, ragged batch; rows r = t*B + b): the rows with t >= lengths[b] are written as 0, x is not read
int tc_layernorm(const float* src, const RowMap& rows, int R, int Cc, const float* gamma, const float* beta, float eps,
                 float* out, cudaStream_t stream, int* clear = nullptr, int nclear = 0, const int* lengths = nullptr,
                 int B = 1);
// backward of that prologue: dx (strided like x) from dy = d/dLN(x) (dense), dgamma / dbeta (+)=; part = scratch of
// layernorm_bwd_scratch_floats(Cc) floats. `lengths` as above: padded rows get dx = 0 and add nothing to dgamma / dbeta
size_t layernorm_bwd_scratch_floats(int Cc);
int launch_layernorm_bwd(const float* x, const RowMap& x_rows, const float* dy, int R, int Cc, const float* gamma,
                         float eps, float* dx, const RowMap& dx_rows, float* dgamma, float* dbeta, int accumulate,
                         float* part, cudaStream_t stream, const int* lengths = nullptr, int B = 1);

// tensor-core (wgmma) 3xTF32 path: C = A[M,K] * B[N,K]^T + biases (both operands k-contiguous, K % 32 == 0, N % 128 == 0)
size_t gemm_tc_scratch_bytes(int M, int N, int K);
bool gemm_tc_eligible(const GemmParams& p, size_t ws_bytes);
int launch_gemm_tc(const GemmParams& p, void* ws, size_t ws_bytes, cudaStream_t stream);

// Building blocks of the tensor-core path for callers that manage the split operands themselves (backward pass).
struct TcOperand {
  const float* hi;
  const float* lo;  // NULL for the operands of a single-pass TF32 GEMM
  long long ld;  // floats between consecutive rows (multiple of 4)
  bool mn = false;  // false: K-major, dense [M or N rows][K]; true: MN-major, dense [K rows][M or N] (no transpose needed
                    // for operands whose contraction index is their row index: dG, X, h_prev in the wgrad GEMMs)
};
bool tc_available();
// lo == NULL: hi only (the operand of a single-pass TF32 GEMM)
int tc_split(const float* src, const RowMap& rows, int R, int Cc, float* hi, float* lo, cudaStream_t stream);
// ready: streamed launch of stream_clusters 4-CTA clusters (GemmParams::tc_ready); needs splitk_ws == NULL
// tf32: single-pass TF32 (GemmParams::tc_tf32), only the hi parts of A and B are read
int tc_gemm_presplit(const TcOperand& A, const TcOperand& B, int M, int N, int K, float* C, const RowMap& c_rows,
                     const float* bias1, const float* bias2, int bias2_n, int accumulate, void* splitk_ws,
                     size_t splitk_ws_bytes, cudaStream_t stream, int* ready = nullptr, int stream_clusters = 0,
                     bool tf32 = false);
// C = A[M,K] * B[N,K]^T + biases, A fp32 read in place through a_rows (tc_a_f32_in_place) and split in registers,
// B K-major presplit; bit-identical to tc_gemm_presplit on the split of A. ready / stream_clusters as above.
int tc_gemm_f32a(const float* A, const RowMap& a_rows, const TcOperand& B, int M, int N, int K, float* C,
                 const RowMap& c_rows, const float* bias1, const float* bias2, int bias2_n, cudaStream_t stream,
                 int* ready = nullptr, int stream_clusters = 0, bool tf32 = false);
// W[N][K] (rows through `rows`) -> fp16 pairs and row exponents at w16 (256-byte aligned, g16::w16_layout(N, K) bytes)
int tc_split_w16(const float* W, const RowMap& rows, int N, int K, void* w16, cudaStream_t stream);
// C = A[M,K] * W[N,K]^T + biases, A fp32 read in place (tc_a_f32_in_place) and split into fp16 pairs on chip, W the
// fp16 pairs at w16 (tc_split_w16); N % 128 == 0, K % 64 == 0. ready / stream_clusters as above.
int tc_gemm_f16a(const float* A, const RowMap& a_rows, const void* w16, int M, int N, int K, float* C,
                 const RowMap& c_rows, const float* bias1, const float* bias2, int bias2_n, cudaStream_t stream,
                 int* ready = nullptr, int stream_clusters = 0);
// C(m,n) (+)= sum_z partial[z][m][n] (+ biases), fixed order (deterministic)
int launch_splitk_reduce(const float* partial, int splitk, int M, int N, float* C, const RowMap& c_rows,
                         const float* bias1, const float* bias2, int bias2_n, int accumulate, cudaStream_t stream);

// bytes of scratch launch_gemm may use for split-K partials for this problem (0 if none wanted)
size_t gemm_scratch_bytes(int M, int N, int K);
// the K splits launch_gemm's FFMA path runs with this scratch, and the K range of each (the last may be shorter)
void gemm_splitk_plan(int M, int N, int K, void* scratch, size_t scratch_bytes, int* splitk, int* k_chunk);
// the K splits tc_gemm_presplit runs (a workspace of ws_bytes when have_ws), and the k-blocks of 32 in each
void tc_splitk_plan(int M, int N, int K, bool have_ws, size_t ws_bytes, int* splitk, int* kb_per_split);

// Enqueue on `stream`. `scratch` may be NULL (then no split-K). Returns B200RNN_* code.
int launch_gemm(const GemmParams& p, void* scratch, size_t scratch_bytes, cudaStream_t stream);

}  // namespace b200rnn
