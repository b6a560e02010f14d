// misc_kernels.cuh — small time-parallel helpers around the recurrence (K7 dropout, transposes, bias sums).
#pragma once
#include "common.cuh"

namespace b200rnn {

// Resolve the dropout RNG state of one forward call on the device, so the call is CUDA-graph replayable:
//   hdr[0] = seed, hdr[1] = offset   taken from `state_dev` ([seed, offset], then offset += consume) if it is
//   non-NULL, else from the by-value arguments. skip: hdr[1] = offset + skip (one of several models drawing from
//   one state as consecutive calls would)
int launch_rng_setup(uint64_t* hdr, uint64_t seed, uint64_t offset, uint64_t* state_dev, uint64_t consume,
                     cudaStream_t stream, uint64_t skip = 0);

// out[i] = in[i] * mask(i) / (1-p) over n dense elements; mask is Philox4x32-10 keyed by hdr = {seed, offset}
// and the per-layer stream id; in == out is allowed (in place).
// `clear` (optional): nclear ints zeroed by the same launch (the ready counters of a streamed GEMM that reads out).
int launch_dropout(const float* in, float* out, size_t n, float p, const uint64_t* hdr, uint32_t stream_id,
                   cudaStream_t stream, int* clear = nullptr, int nclear = 0);

// Batch-slot order of a ragged batch: order[slot] = the row of rank `slot` when the B rows are sorted by descending
// lengths[row], ties by row index (a stable sort: non-increasing lengths give the identity). One CTA.
int launch_length_order(const int* lengths, int B, int* order, cudaStream_t stream);

// The recurrent-side gate gradient of each row's first scanned step, the rows the initial state's dW_hh term pairs
// with h_0: out[b][c] = dGh[t_first(b)][b][c] over c < G*H, where dGh is dgates [T,B,G*H] (the GRU's n columns come
// from dghn [T,B,H] instead; an Elman row is its H dpre columns). t_first = 0 forward; reverse: T - 1, or lengths[b] - 1 (a row of length 0: zeros).
int launch_initial_state_rows(const float* dgates, const float* dghn, int mode, int B, int T, int H, bool reverse,
                              const int* lengths, float* out, cudaStream_t stream);

// Dense copy dst[T*B][C] of the rows r = t*B + b of src (read through `rows`), with the rows past each sequence's end
// (t >= lengths[b]) written as 0 instead of read: the layer-0 operand of a ragged backward's dW_ih GEMM, so that
// whatever the caller left in the padding (NaN, Inf) meets the zero gate gradients of those steps as a 0, not as 0 * NaN.
int launch_valid_rows(const float* src, const RowMap& rows, int T, int B, int C, const int* lengths, float* dst,
                      cudaStream_t stream);

// db_ih / db_hh from the per-slice partial sums written by the backward recurrence:
//   part [nslices][(G+1)*H]  (first G*H: sum of dGi columns; tail H: GRU sum of dn*r)
//   GRU : db_ih = sum(part[:, :3H]);  db_hh = (sum part[:, :2H], sum part[:, 3H:4H])
//   LSTM: db_ih = db_hh = sum(part[:, :4H])
//   Elman: part [nslices][H] (sum of dpre); db_ih = db_hh = sum(part)
int launch_bias_reduce(const float* part, int nslices, int mode, int H, float* db_ih, float* db_hh,
                       int accumulate, cudaStream_t stream);

// ---- one Adam / AdamW rule for every kernel that applies it (adam_kernel, the fuse head and its deferred finish) ----
// torch.optim.Adam / AdamW without amsgrad at step t (1-based): the same code everywhere, so that the fused head's
// update and b200rnn_adamw's are bit-identical from the same gradient.
struct AdamCoef {
  float step_size;     // lr / (1 - beta1^t)
  float inv_sqrt_bc2;  // 1 / sqrt(1 - beta2^t)
  float decay;         // 1 - lr * weight_decay (decoupled, AdamW); exactly 1 for Adam
};
// 1 - beta^t = -expm1(t * log1p(-(1 - beta))): 1 - beta is exact in fp32 for beta in [0.5, 1], and no step cancels.
// 1 - powf(beta, t) loses up to ~110 ulp of bc2 at beta2 = 0.999 and t = 2..5, because beta^t is close to 1 there.
__device__ __forceinline__ float adam_bias_correction(float beta, float t) {
  return -expm1f(t * log1pf(-(1.f - beta)));
}
__device__ __forceinline__ AdamCoef adam_coef(float t, float lr, float beta1, float beta2, float weight_decay) {
  return AdamCoef{lr / adam_bias_correction(beta1, t), rsqrtf(adam_bias_correction(beta2, t)), 1.f - lr * weight_decay};
}
// g is the already scaled gradient
__device__ __forceinline__ void adam_update(float& p, float& m, float& v, float g, float beta1, float beta2, float eps,
                                            const AdamCoef& c) {
  const float mi = beta1 * m + (1.f - beta1) * g;
  const float vi = beta2 * v + (1.f - beta2) * g * g;
  m = mi;
  v = vi;
  p = p * c.decay - c.step_size * mi / (sqrtf(vi) * c.inv_sqrt_bc2 + eps);
}

}  // namespace b200rnn
