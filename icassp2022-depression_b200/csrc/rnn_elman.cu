// rnn_elman.cu — the Elman recurrence (torch.nn.RNN, nonlinearity 'tanh' or 'relu'), forward and BPTT, at every hidden
// size H % 16 == 0, 16 <= H <= 1024. The cluster design, exchange protocol, weight tiers and launch contract are those
// of the runtime-sized GRU / LSTM kernels (rnn_anyh.cu, anyh_core.cuh) with one gate block (G = 1):
//   * forward step: pre = gi_t + W_hh h_{t-1} (gi holds the x-projection with b_ih + b_hh folded in, api.cu), one
//     fixed-order FFMA chain of length H per (unit, batch slot), h_t = tanh(pre) or relu(pre) (elman_cell_fwd). The
//     activated h_t is saved as the gate block of the reserve; there is no second saved block.
//   * backward step: dpre = dh (1 - h^2) for tanh, dh [h > 0] for relu (elman_cell_bwd, from the saved h_t), then
//     dh_{t-1} = direct + W_hh^T dpre at the start of the next step against the exchanged dpre slices.
// The nonlinearity is a warp-uniform runtime flag (p.mode), so the kernels are templated only on ragged batches (VL)
// and the weight tier (ONCHIP): 4 forward and 4 backward instantiations.
#include "anyh_core.cuh"
#include "rnn_cell.cuh"

namespace b200rnn {

namespace {

// Shared memory: [W_s: n x (H+4), ONCHIP only] [h: 2 x BS x H] [bars: 2 x C] (anyh_smem with G = 1)
template <bool VL, bool ONCHIP>
__global__ void __launch_bounds__(ANYH_MAX_NT, 1) elman_fwd_kernel(const RecFwdParams p, const int nslices) {
  const int H = p.H, B = p.B, LD = H + 4;
  const bool relu = p.mode == B200RNN_RNN_RELU;
  const AnyhSlice s = anyh_slice<VL>(p, nslices);
  const int C = s.C, HS = s.HS, BS = s.BS, NT = s.NT, dir = s.dir, b0 = s.b0, j0 = s.j0, n = s.n, T = s.T;
  const uint32_t rank = s.rank;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* W_s = reinterpret_cast<float*>(smem_raw);  // [n][LD]
  float* h_s = W_s + (ONCHIP ? (size_t)HS * LD : 0);
  uint64_t* bars = reinterpret_cast<uint64_t*>(h_s + (size_t)2 * BS * H);
  const int tid = threadIdx.x;
  const float* w_hh = p.w_hh[dir];

  if (tid == 0) init_bars(bars, C);
  if constexpr (ONCHIP) stage_rows(W_s, w_hh, n, H, NT, [&](int r) { return (size_t)(j0 + r) * H; });
  for (int i = tid; i < BS * H; i += NT) {  // buffer 0: h_0 of the cluster's slots (zeros past the batch / without h_0)
    const int q = i / H, k = i - q * H;
    const int slot = b0 + q;
    float v = 0.f;
    if (p.h_0 && slot < B) v = p.h_0[((size_t)dir * B + (VL ? p.order[slot] : slot)) * H + k];
    h_s[i] = v;
  }
  __syncthreads();
  ptx::cluster_sync_all();  // peers' barriers are initialised before anyone sends

  const int u = s.u, b = s.b, j = j0 + u, slot = b0 + b;
  const bool valid = s.active && slot < B;
  const int row = valid ? (VL ? p.order[slot] : slot) : 0;
  const int len = (VL && valid) ? p.lengths[row] : p.T;
  float* gates = p.gates[dir];
  float h = (p.h_0 && valid) ? p.h_0[((size_t)dir * B + row) * H + j] : 0.f;
  float gi = 0.f;
  auto load_gi = [&](int t) { gi = valid ? gates[((size_t)t * B + row) * H + j] : 0.f; };
  if (T > 0) load_gi(dir ? T - 1 : 0);
  const float* wrow = ONCHIP ? W_s + (size_t)u * LD : w_hh + (size_t)(j0 + u) * H;

  for (int step = 0; step < T; ++step) {
    const int t = dir ? T - 1 - step : step;
    const int cur = step & 1, nxt = cur ^ 1;
    if (step > 0) wait_bars(bars, cur, C, rank, ((step - 1) >> 1) & 1);
    if (tid == 0 && step + 1 < T) arm_bars(bars, nxt, s, H, 1);
    float acc[1] = {0.f};
    dot_rows<1, ONCHIP, false>(wrow, 0, h_s + ((size_t)cur * BS + b) * H, 0, H, acc);
    const float act = elman_cell_fwd(gi, acc[0], relu);
    const bool frozen = VL && t >= len;  // past its length a row keeps its state and emits 0
    const float hnew = frozen ? h : act;
    h = hnew;
    if (valid) {
      if (p.y) p.y[(long long)t * p.y_st + (long long)row * p.y_sb + dir * H + j] = frozen ? 0.f : hnew;
      if (p.training) gates[((size_t)t * B + row) * H + j] = act;  // the activated h_t over the x-projection
    }
    if (step + 1 < T) {
      float* h_nxt = h_s + (size_t)nxt * BS * H;
      if (s.active) h_nxt[(size_t)b * H + j] = hnew;
      __syncthreads();  // the own slice is complete (and every thread is past step - 1's reads of buffer nxt)
      send_slice(h_nxt, H, 1, H, s, &bars[nxt * C + rank]);
      load_gi(dir ? T - 2 - step : step + 1);
    }
  }
  if (valid) {
    p.h_n[((size_t)dir * B + row) * H + j] = h;
    if (VL && p.y)  // the steps [T, p.T) the cluster skipped emit 0, as past any sequence's length
      for (int t = T; t < p.T; ++t) p.y[(long long)t * p.y_st + (long long)row * p.y_sb + dir * H + j] = 0.f;
  }
  ptx::cluster_sync_all();  // nobody exits while a peer could still address its shared memory
}

// Shared memory: [W_s: n x (H+4), ONCHIP only] [d: 2 x BS x H] [red: BS x HS] [bars: 2 x C] (within anyh_smem, G = 1)
// Step s: dh = direct_{s-1} + W_hh^T dpre_{s-1} (the exchange of step s - 1, all H columns), the cell backward, then this
// CTA's dpre to every CTA. Step T only contracts, for dh_0.
template <bool VL, bool ONCHIP>
__global__ void __launch_bounds__(ANYH_MAX_NT, 1) elman_bwd_kernel(const RecBwdParams p, const int nslices) {
  const int H = p.H, B = p.B, LD = H + 4;
  const bool relu = p.mode == B200RNN_RNN_RELU;
  const AnyhSlice s = anyh_slice<VL>(p, nslices);
  const int C = s.C, HS = s.HS, BS = s.BS, NT = s.NT, dir = s.dir, b0 = s.b0, j0 = s.j0, n = s.n, T = s.T;
  const uint32_t rank = s.rank;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* W_s = reinterpret_cast<float*>(smem_raw);  // [n][LD]
  float* d_s = W_s + (ONCHIP ? (size_t)HS * LD : 0);
  float* red = d_s + (size_t)2 * BS * H;
  uint64_t* bars = reinterpret_cast<uint64_t*>(red + (size_t)BS * HS);
  const int tid = threadIdx.x;
  // rows u of this CTA: W_hh[:][j0 + u], contiguous from j0 * H (anyh_prep_kernel with G = 1)
  const float* w_prep = p.w_prep[dir] + (size_t)j0 * H;

  if (tid == 0) init_bars(bars, C);
  if constexpr (ONCHIP) stage_rows(W_s, w_prep, n, H, NT, [&](int r) { return (size_t)r * H; });
  __syncthreads();
  ptx::cluster_sync_all();

  const int u = s.u, b = s.b, j = j0 + u, slot = b0 + b;
  const bool valid = s.active && slot < B;
  const int row = valid ? (VL ? p.order[slot] : slot) : 0;
  const int len = (VL && valid) ? p.lengths[row] : T;
  const float* gates = p.gates[dir];
  float* dgates = p.dgates[dir];
  const float* wrow = ONCHIP ? W_s + (size_t)u * LD : w_prep + (size_t)u * H;

  float dh_carry = 0.f, direct = 0.f, bsum = 0.f;
  if (valid && p.dh_n) dh_carry = p.dh_n[((size_t)dir * B + row) * H + j];
  float hv = 0.f, dyv = 0.f;  // the saved h_t and dy (prefetched)
  auto load_step = [&](int step) {
    const int t = dir ? step : (T - 1 - step);
    hv = gates[((size_t)t * B + row) * H + j];
    dyv = p.dy[(long long)t * p.dy_st + (long long)row * p.dy_sb + dir * H + j];
  };
  if (valid && T > 0) load_step(0);
  const bool want_dh0 = p.dh_0 != nullptr;

  for (int step = 0; step <= T; ++step) {
    if (step > 0) {  // dh of this step from the dpre slices step - 1 sent
      const int cur = step & 1;
      wait_bars(bars, cur, C, rank, ((step - 1) >> 1) & 1);
      float acc[1] = {0.f};
      dot_rows<1, ONCHIP, false>(wrow, 0, d_s + ((size_t)cur * BS + b) * H, 0, H, acc);
      dh_carry = direct + acc[0];
    }
    if (step == T) break;
    const int t = dir ? step : (T - 1 - step);
    const bool last = step == T - 1;
    const bool send = !last || want_dh0;
    const int nxt = (step + 1) & 1;
    if (tid == 0 && send) arm_bars(bars, nxt, s, H, 1);

    const bool frozen = VL && t >= len;  // frozen: the output is the constant 0, dh passes straight through
    const float dh = frozen ? dh_carry : dh_carry + dyv;
    const float dg = frozen ? 0.f : elman_cell_bwd(hv, dh, relu);
    direct = frozen ? dh : 0.f;
    if (valid) {
      bsum += dg;
      dgates[((size_t)t * B + row) * H + j] = dg;
    }
    if (!send) break;
    float* d_nxt = d_s + (size_t)nxt * BS * H;
    if (s.active) d_nxt[(size_t)b * H + j] = valid ? dg : 0.f;
    __syncthreads();  // the own slice is complete (and every thread is past step - 1's reads of buffer nxt)
    send_slice(d_nxt, H, 1, H, s, &bars[nxt * C + rank]);
    if (valid && !last) load_step(step + 1);
  }
  // the gradient w.r.t. the initial state: what the scan carried past its first step (a cluster that ran no step passes
  // dh_n on)
  if (valid) {
    if (want_dh0) p.dh_0[((size_t)dir * B + row) * H + j] = dh_carry;
    if (VL)  // the steps [T, p.T) the cluster skipped: their gate gradients are 0
      for (int t = T; t < p.T; ++t) dgates[((size_t)t * B + row) * H + j] = 0.f;
  }
  // per-slice bias-gradient partials [nslices][H]: the slice's batch slots summed in slot order
  if (s.active) red[(size_t)b * HS + u] = bsum;
  __syncthreads();
  if (s.active && b == 0) {
    float v = 0.f;
    for (int q = 0; q < BS; ++q) v += red[(size_t)q * HS + u];
    p.dbias_part[dir][(size_t)s.slice * H + j] = v;
  }
  ptx::cluster_sync_all();
}

}  // namespace

AnyhKernel<RecFwdParams> elman_kernel(const RecFwdParams&, bool vl, bool onchip) {
  return vl ? (onchip ? elman_fwd_kernel<true, true> : elman_fwd_kernel<true, false>)
            : (onchip ? elman_fwd_kernel<false, true> : elman_fwd_kernel<false, false>);
}
AnyhKernel<RecBwdParams> elman_kernel(const RecBwdParams&, bool vl, bool onchip) {
  return vl ? (onchip ? elman_bwd_kernel<true, true> : elman_bwd_kernel<true, false>)
            : (onchip ? elman_bwd_kernel<false, true> : elman_bwd_kernel<false, false>);
}

}  // namespace b200rnn
