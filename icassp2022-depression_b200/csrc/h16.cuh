// h16.cuh — 16-bit (fp16 / bf16) modules, B200RNN_FLAG_F16 / B200RNN_FLAG_BF16: the conversions around the fp32
// kernels and the native 16-bit input projection (gemm_n16_kernel, gemm_tc.cu). DESIGN.md "16-bit modules".
//
// Every widening is exact (a 16-bit value is an fp32 value), every narrowing rounds to nearest even once.
#pragma once
#include "common.cuh"

namespace b200rnn {

// storage type of the user-visible tensors of one call (the reserve and the scratch stay fp32)
enum : int { DT_F32 = 0, DT_F16 = 1, DT_BF16 = 2 };

// dst[r * C + c] = (float) src[rows.off(r) + c], src 16-bit of type dt; dst dense
int launch_widen16(const void* src, const RowMap& rows, int R, int C, int dt, float* dst, cudaStream_t stream);

// v = src[src_rows.off(r) + c] (+ the value already at dst when accumulate); dst[dst_rows.off(r) + c] = round_dt(v);
// wb (optional, dense [R][C]) = the rounded value widened back to fp32
int launch_narrow16(const float* src, const RowMap& src_rows, int R, int C, int dt, void* dst, const RowMap& dst_rows,
                    bool accumulate, float* wb, cudaStream_t stream);

// ---- fp32 master parameters (B200RNN_FLAG_F32_PARAMS): one launch over every parameter tensor of a call ----------------
// Per segment, element i: r = round_dt(src[i]) (nearest even, as narrow16 rounds), then
//   ROUND16_IMAGES:   d16[i] = r, d32[i] = widen(r)      (either target may be NULL)
//   ROUND16_GRAD_SET: d32[i] = widen(r)                  (a gradient into its fp32 target)
//   ROUND16_GRAD_ADD: d32[i] = d32[i] + widen(r)         (the same, accumulated in fp32)
enum : int { ROUND16_IMAGES = 0, ROUND16_GRAD_SET = 1, ROUND16_GRAD_ADD = 2 };
constexpr int ROUND16_MAX_SEGS = 8 * 2 * 4;  // L * D * 4 parameters, L <= 8, D <= 2
struct Round16Seg {
  const float* src;
  uint16_t* d16;
  float* d32;
  long long n;
};
int launch_round16_multi(const Round16Seg* segs, int nseg, int dt, int mode, cudaStream_t stream);

// 16-bit rows gathered into a dense [R][C] 16-bit copy (an A operand the TMA cannot read in place)
int launch_copy16(const void* src, const RowMap& rows, int R, int C, void* dst, cudaStream_t stream);

// C[M,N] = A[M,K] W[N,K]^T + bias1 + bias2 (columns < bias2_n) on wgmma m64n128k16 with f16 or bf16 operands (dt)
// and fp32 accumulation: every product is exact, each k-block of 64 is summed by the tensor core and added into an
// fp32 total. A is read in place through a_rows by a 3-D TMA, W [N][K] dense. tc_gemm_n16_ok: whether the shape and
// the operands' alignment allow it (N % 128 == 0, K % 8 == 0, 16-byte aligned rows; A's rows as tc_a_f32_in_place
// requires of an fp32 A).
bool tc_gemm_n16_ok(const void* A, const RowMap& a_rows, const void* W, int M, int N, int K);
// a_route: where A comes from ("tma": the caller's tensor or the previous layer's output, "copy16": a dense copy of x),
// named on the B200RNN_DEBUG line
int tc_gemm_n16(const void* A, const RowMap& a_rows, const void* W, int M, int N, int K, int dt, float* C,
                const RowMap& c_rows, const float* bias1, const float* bias2, int bias2_n, cudaStream_t stream,
                const char* a_route = "tma");

}  // namespace b200rnn
