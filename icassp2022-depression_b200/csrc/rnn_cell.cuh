// rnn_cell.cuh — the gate math of one GRU / LSTM / Elman step, shared by the persistent recurrence kernels (rnn_rec.cu,
// rnn_anyh.cu) and the one-step cell kernels (cell.cu), so that a cell and a sequence step apply the same
// non-linearities in the same order. Gate order as in torch/nn/modules/rnn.py: GRU r, z, n; LSTM i, f, g, o.
#pragma once
#include "common.cuh"

namespace b200rnn {

// The GRU cell, forward: gi = x-projection with b_ih (and, for r and z, b_hh) folded in, pre = W_hh h, bhn = b_hn,
// h = h_{t-1}. Returns the activated gates, hn = (W_hn h)_j + b_hn and the new state.
struct GruStep {
  float r, z, n, hn, h;
};

__device__ __forceinline__ GruStep gru_cell_fwd(const float (&gi)[3], const float (&pre)[3], float bhn, float h) {
  GruStep s;
  s.r = sigmoid_f(gi[0] + pre[0]);
  s.z = sigmoid_f(gi[1] + pre[1]);
  s.hn = pre[2] + bhn;
  s.n = tanh_f(gi[2] + s.r * s.hn);
  s.h = s.n + s.z * (h - s.n);
  return s;
}

// The GRU cell, backward: from the saved gates sv = (r, z, n), hn, h_{t-1} and the gradient dh of h_t, the gate
// gradients dg of the x-projection and dhn = dn * r, the n-block gradient of the h-projection (W_hn h + b_hn; the r and z
// blocks equal dg's); returns the direct term z * dh of the gradient w.r.t. h_{t-1}
__device__ __forceinline__ float gru_cell_bwd(const float (&sv)[3], float hn, float h_prev, float dh, float (&dg)[3],
                                              float& dhn) {
  const float r = sv[0], z = sv[1], n = sv[2];
  const float dn = dh * (1.f - z) * (1.f - n * n);
  const float dz = dh * (h_prev - n) * z * (1.f - z);
  const float dr = dn * hn * r * (1.f - r);
  dhn = dn * r;
  dg[0] = dr; dg[1] = dz; dg[2] = dn;
  return dh * z;
}

// The LSTM cell, forward: gate pre-activations gi + pre -> activated gates, c_t and o * tanh(c_t)
struct LstmStep {
  float i, f, g, o, c, h;
};

__device__ __forceinline__ LstmStep lstm_cell_fwd(const float (&gi)[4], const float (&pre)[4], float c) {
  LstmStep s;
  s.i = sigmoid_f(gi[0] + pre[0]);
  s.f = sigmoid_f(gi[1] + pre[1]);
  s.g = tanh_f(gi[2] + pre[2]);
  s.o = sigmoid_f(gi[3] + pre[3]);
  s.c = fmaf(s.f, c, s.i * s.g);  // spelled out: which product is fused must not be left to the compiler
  s.h = s.o * tanh_f(s.c);
  return s;
}

// The LSTM cell, backward: from the saved gates sv = (i, f, g, o), c_t, c_{t-1}, the gradient dh of o * tanh(c_t) and
// the carried dc, the gate gradients dg; returns the dc carried to step t - 1
__device__ __forceinline__ float lstm_cell_bwd(const float (&sv)[4], float c_t, float c_prev, float dh, float dc_carry,
                                               float (&dg)[4]) {
  const float ig = sv[0], fg = sv[1], gg = sv[2], og = sv[3];
  const float tc = tanh_f(c_t);
  const float dout = dh * tc * og * (1.f - og);
  const float dc = dc_carry + dh * og * (1.f - tc * tc);
  dg[0] = dc * gg * ig * (1.f - ig);
  dg[1] = dc * c_prev * fg * (1.f - fg);
  dg[2] = dc * ig * (1.f - gg * gg);
  dg[3] = dout;
  return dc * fg;
}

// The Elman cell, forward: gi = x-projection with b_ih + b_hh folded in, pre = W_hh h. Returns h = tanh(gi + pre) (the
// tanh of the GRU n gate) or relu(gi + pre); a NaN pre-activation stays NaN, as torch.relu keeps it
__device__ __forceinline__ float elman_cell_fwd(float gi, float pre, bool relu) {
  const float a = gi + pre;
  return relu ? (a < 0.f ? 0.f : a) : tanh_f(a);
}

// The Elman cell, backward: from the saved output h and its gradient dh, the gradient of the pre-activation (relu:
// torch's threshold_backward on the output, dh where h > 0)
__device__ __forceinline__ float elman_cell_bwd(float h, float dh, bool relu) {
  return relu ? (h > 0.f ? dh : 0.f) : dh * (1.f - h * h);
}

// ---- linearised cells (forward-mode AD): the tangent of a step from the saved activations, sigma' = s (1 - s),
// tanh' = 1 - t^2, relu' = [h > 0]

// The GRU cell: sv = (r, z, n), hn = W_hn h + b_hn, h_prev = h_{t-1}; a[0..1] the r, z pre-activation tangents, a[2] the
// n block's x-side tangent, ahn the tangent of W_hn h + b_hn, hd the tangent of h_{t-1}. Returns the tangent of h_t.
__device__ __forceinline__ float gru_cell_jvp(const float (&sv)[3], float hn, float h_prev, const float (&a)[3], float ahn,
                                              float hd) {
  const float r = sv[0], z = sv[1], n = sv[2];
  const float dr = r * (1.f - r) * a[0];
  const float dz = z * (1.f - z) * a[1];
  const float dn = (1.f - n * n) * (a[2] + dr * hn + r * ahn);
  return (1.f - z) * dn + z * hd + dz * (h_prev - n);
}

// The LSTM cell: sv = (i, f, g, o), c_t, c_prev = c_{t-1}; a the pre-activation tangents, cd the tangent of c_{t-1}.
// Returns the tangent of h_t; cd becomes the tangent of c_t.
__device__ __forceinline__ float lstm_cell_jvp(const float (&sv)[4], float c_t, float c_prev, const float (&a)[4],
                                               float& cd) {
  const float ig = sv[0], fg = sv[1], gg = sv[2], og = sv[3];
  const float di = ig * (1.f - ig) * a[0];
  const float df = fg * (1.f - fg) * a[1];
  const float dg = (1.f - gg * gg) * a[2];
  const float dout = og * (1.f - og) * a[3];
  cd = df * c_prev + fg * cd + di * gg + ig * dg;
  const float tc = tanh_f(c_t);
  return dout * tc + og * (1.f - tc * tc) * cd;
}

// The Elman cell: from the saved output h and the pre-activation tangent a, the tangent of h
__device__ __forceinline__ float elman_cell_jvp(float h, float a, bool relu) {
  return relu ? (h > 0.f ? a : 0.f) : a * (1.f - h * h);
}

}  // namespace b200rnn
