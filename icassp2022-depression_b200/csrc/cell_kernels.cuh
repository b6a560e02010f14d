// cell_kernels.cuh — host-side launch interface of the one-step GRUCell / LSTMCell kernels (cell.cu).
#pragma once
#include "common.cuh"

namespace b200rnn {

// h' (and c') = cell(x W_ih^T + b_ih, h W_hh^T + b_hh) for B rows, one launch.
struct CellFwdParams {
  int mode, B, I, H;
  int tf32;                 // single-pass TF32 contraction (B200RNN_FLAG_TF32), else 3xTF32
  const float* x;           // [B, I], row b at x + b * x_ld (any alignment)
  long long x_ld;
  const float* h;           // [B, H] at h + b * h_ld, or NULL (zeros)
  long long h_ld;
  const float* c;           // LSTM: [B, H] at c + b * c_ld, or NULL (zeros)
  long long c_ld;
  const float* w_ih;        // [G*H, I] contiguous
  const float* w_hh;        // [G*H, H] contiguous
  const float* b_ih;        // [G*H] or NULL (bias=False; NULL together with b_hh)
  const float* b_hh;
  float* h_out;             // [B, H] contiguous
  float* c_out;             // LSTM: [B, H] contiguous
  float* gates;             // NULL, or [B, G*H]: the activated gates (GRU r, z, n; LSTM i, f, g, o)
  float* extra;             // with gates: [B, H], GRU W_hn h + b_hn, LSTM c'
};
int launch_cell_fwd(const CellFwdParams& p, cudaStream_t stream);

// The elementwise cell backward: gate gradients for the x-part and the h-part, the direct state-gradient terms and the
// per-slice bias partial sums launch_bias_reduce reads.
struct CellBwdParams {
  int mode, B, H;
  const float* gates;       // saved by the forward, [B, G*H]
  const float* extra;       // [B, H]
  const float* h;           // GRU: h of the forward ([B, H] at h + b * h_ld), or NULL (zeros)
  long long h_ld;
  const float* c;           // LSTM: c of the forward, or NULL (zeros)
  long long c_ld;
  const float* dh_out;      // [B, H] contiguous gradient w.r.t. h', or NULL (zeros)
  const float* dc_out;      // LSTM: [B, H] gradient w.r.t. c', or NULL (zeros)
  float* dg_x;              // out [B, G*H]: gradient w.r.t. the x-projection (and, LSTM, the h-projection)
  float* dg_h;              // GRU out [B, G*H]: gradient w.r.t. the h-projection (the n block is dg_x's times r)
  float* direct;            // out, or NULL: GRU z * dh' [B, H]; LSTM dc = f * (dc' + ...) [B, H], the final dc
  float* part;              // out [cell_bwd_slices(B)][(G+1)*H]: column sums of dg_x, GRU tail: of dg_h's n block
};
int cell_bwd_slices(int B);
int launch_cell_bwd(const CellBwdParams& p, cudaStream_t stream);

}  // namespace b200rnn
