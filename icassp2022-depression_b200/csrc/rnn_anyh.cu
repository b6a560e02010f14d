// rnn_anyh.cu — the GRU / LSTM recurrence, forward and BPTT, at every hidden size H % 16 == 0, 16 <= H <= 1024 that the
// fixed configs of rnn_rec.cu (H = 128, 256) do not cover. H, the cluster width C and the batch rows per cluster BS are
// known only at run time; the kernels are templated on the mode, ragged batches (VL) and where W_hh lives (ONCHIP).
//
// Same launch shape and contract as rec_fwd_kernel / rec_bwd_kernel (rnn_kernels.cuh): grid = D * nslices clusters of C
// CTAs, cluster = one direction of BS batch slots. The H / 8 groups of 8 units are split as evenly as possible over the
// C CTAs (anyh_units): CTA `rank` owns n units from j0, n a multiple of 8 and at most HS = 8 * ceil(H / 8 / C), so every
// multiple of 16 has a shape, and a CTA's slice of a state row is a whole number of 16-byte chunks. One thread per
// (unit u, batch slot b), 8 consecutive units by BS slots per group of 8 * BS threads (the projected kernels'
// proj_thread), NT = HS * BS rounded up to whole warps; threads past the CTA's units are idle.
//   * Weights: ONCHIP, the CTA's G * n rows (forward: W_hh[g*H + j0 + u][:]; backward: W_hh[g*H + :][j0 + u], the
//     w_prep slice of anyh_prep_kernel) are staged once into shared memory, rows padded to H + 4 floats so that the 8
//     units a quarter-warp reads with one 16-byte load sit in different banks. Otherwise (the L2 tier) the same rows are
//     read from global memory every step: weight_hh in place in the forward, w_prep in the backward.
//   * Step: G fixed-order FFMA chains of length H per thread (k ascending), the cell of rnn_cell.cuh, then the CTA's
//     slice of the new state (forward: h_t, BS x n; backward: the recurrent-side gate gradients, BS x G*n) is written
//     into its own buffer with ordinary stores (published by __syncthreads) and sent to the C - 1 peers with st.async,
//     which completes transaction bytes on the destination's mbarrier of that source and buffer. Double buffered:
//     step s contracts against what step s - 1 sent (the ExchangeBars protocol of rnn_rec.cu with LAG = 1).
//   * The waits are bounded: a protocol bug traps (a CUDA error) instead of hanging the GPU.
#include <map>
#include <mutex>
#include <stdlib.h>
#include <tuple>

#include "anyh_core.cuh"
#include "rnn_cell.cuh"

namespace b200rnn {

namespace {

// =================================================================================================
// forward
// =================================================================================================
// Shared memory: [W_s: G*n x (H+4), ONCHIP only] [h: 2 x BS x H] [bars: 2 x C]
template <int MODE, bool VL, bool ONCHIP>
__global__ void __launch_bounds__(ANYH_MAX_NT, 1) anyh_fwd_kernel(const RecFwdParams p, const int nslices) {
  constexpr int G = MODE == B200RNN_GRU ? 3 : 4;
  const int H = p.H, B = p.B, LD = H + 4;
  const AnyhSlice s = anyh_slice<VL>(p, nslices);
  const int C = s.C, HS = s.HS, BS = s.BS, NT = s.NT, dir = s.dir, b0 = s.b0, j0 = s.j0, n = s.n, T = s.T;
  const uint32_t rank = s.rank;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* W_s = reinterpret_cast<float*>(smem_raw);  // [G][n][LD]
  float* h_s = W_s + (ONCHIP ? (size_t)G * HS * LD : 0);
  uint64_t* bars = reinterpret_cast<uint64_t*>(h_s + (size_t)2 * BS * H);
  const int tid = threadIdx.x;
  const float* w_hh = p.w_hh[dir];

  if (tid == 0) init_bars(bars, C);
  if constexpr (ONCHIP)
    stage_rows(W_s, w_hh, G * n, H, NT, [&](int r) { return ((size_t)(r / n) * H + j0 + r % n) * H; });
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
  float c = (MODE == B200RNN_LSTM && p.c_0 && valid) ? p.c_0[((size_t)dir * B + row) * H + j] : 0.f;
  const float bhn = MODE == B200RNN_GRU ? p.b_hh[dir][2 * H + j] : 0.f;
  float gi[G];
  auto load_gi = [&](int t) {
#pragma unroll
    for (int g = 0; g < G; ++g) gi[g] = valid ? gates[((size_t)t * B + row) * (G * H) + g * H + j] : 0.f;
  };
  if (T > 0) load_gi(dir ? T - 1 : 0);
  const float* wrow = ONCHIP ? W_s + (size_t)u * LD : w_hh + (size_t)(j0 + u) * H;
  const size_t wg = ONCHIP ? (size_t)n * LD : (size_t)H * H;

  for (int step = 0; step < T; ++step) {
    const int t = dir ? T - 1 - step : step;
    const int cur = step & 1, nxt = cur ^ 1;
    if (step > 0) wait_bars(bars, cur, C, rank, ((step - 1) >> 1) & 1);
    if (tid == 0 && step + 1 < T) arm_bars(bars, nxt, s, H, 1);
    float acc[G];
#pragma unroll
    for (int g = 0; g < G; ++g) acc[g] = 0.f;
    dot_rows<G, ONCHIP, false>(wrow, wg, h_s + ((size_t)cur * BS + b) * H, 0, H, acc);

    float hnew, sg[G], sx;
    const bool frozen = VL && t >= len;  // past its length a row keeps its state and emits 0
    if constexpr (MODE == B200RNN_GRU) {
      const GruStep st = gru_cell_fwd(gi, acc, bhn, h);
      hnew = frozen ? h : st.h;
      sg[0] = st.r; sg[1] = st.z; sg[2] = st.n; sx = st.hn;
    } else {
      const LstmStep st = lstm_cell_fwd(gi, acc, c);
      hnew = frozen ? h : st.h;
      c = frozen ? c : st.c;
      sg[0] = st.i; sg[1] = st.f; sg[2] = st.g; sg[3] = st.o; sx = c;
    }
    h = hnew;
    if (valid) {
      if (p.y) p.y[(long long)t * p.y_st + (long long)row * p.y_sb + dir * H + j] = frozen ? 0.f : hnew;
      if (p.training) {  // the activated gates over the x-projection, and GRU W_hn h + b_hn / LSTM c_t
        float* gp = gates + ((size_t)t * B + row) * (G * H) + j;
#pragma unroll
        for (int g = 0; g < G; ++g) gp[g * H] = sg[g];
        p.extra[dir][((size_t)t * B + row) * H + j] = sx;
      }
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
    if (MODE == B200RNN_LSTM && p.c_n) p.c_n[((size_t)dir * B + row) * H + j] = c;
    if (VL && p.y)  // the steps [T, p.T) the cluster skipped emit 0, as past any sequence's length
      for (int t = T; t < p.T; ++t) p.y[(long long)t * p.y_st + (long long)row * p.y_sb + dir * H + j] = 0.f;
  }
  ptx::cluster_sync_all();  // nobody exits while a peer could still address its shared memory
}

// =================================================================================================
// backward (BPTT)
// =================================================================================================
// Shared memory: [W_s: G*n x (H+4), ONCHIP only] [d: 2 x BS x G*H] [red: BS x (G+1) x HS] [bars: 2 x C]
// Step s: dh = direct_{s-1} + sum_g W_hh[g-block]^T dgh_{s-1} (the exchange of step s - 1, all G*H columns), the cell
// backward, then this CTA's dgh (GRU: n-block dn * r) to every CTA. Step T only contracts, for dh_0.
template <int MODE, bool VL, bool ONCHIP>
__global__ void __launch_bounds__(ANYH_MAX_NT, 1) anyh_bwd_kernel(const RecBwdParams p, const int nslices) {
  constexpr int G = MODE == B200RNN_GRU ? 3 : 4;
  const int H = p.H, B = p.B, LD = H + 4, GH = G * H;
  const AnyhSlice s = anyh_slice<VL>(p, nslices);
  const int C = s.C, HS = s.HS, BS = s.BS, NT = s.NT, dir = s.dir, b0 = s.b0, j0 = s.j0, n = s.n, T = s.T;
  const uint32_t rank = s.rank;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* W_s = reinterpret_cast<float*>(smem_raw);  // [G][n][LD]
  float* d_s = W_s + (ONCHIP ? (size_t)G * HS * LD : 0);
  float* red = d_s + (size_t)2 * BS * GH;
  uint64_t* bars = reinterpret_cast<uint64_t*>(red + (size_t)BS * (G + 1) * HS);
  const int tid = threadIdx.x;
  // rows (g, u) of this CTA: W_hh[g*H + :][j0 + u], contiguous from G * j0 * H (anyh_prep_kernel)
  const float* w_prep = p.w_prep[dir] + (size_t)G * j0 * H;

  if (tid == 0) init_bars(bars, C);
  if constexpr (ONCHIP) stage_rows(W_s, w_prep, G * n, H, NT, [&](int r) { return (size_t)r * H; });
  __syncthreads();
  ptx::cluster_sync_all();

  const int u = s.u, b = s.b, j = j0 + u, slot = b0 + b;
  const bool valid = s.active && slot < B;
  const int row = valid ? (VL ? p.order[slot] : slot) : 0;
  const int len = (VL && valid) ? p.lengths[row] : T;
  const float* gates = p.gates[dir];
  const float* extra = p.extra[dir];
  float* dgates = p.dgates[dir];
  const float* wrow = ONCHIP ? W_s + (size_t)u * LD : w_prep + (size_t)u * H;
  const size_t wg = ONCHIP ? (size_t)n * LD : (size_t)n * H;

  float dh_carry = 0.f, dc_carry = 0.f, direct = 0.f;
  if (valid) {
    if (p.dh_n) dh_carry = p.dh_n[((size_t)dir * B + row) * H + j];
    if (MODE == B200RNN_LSTM && p.dc_n) dc_carry = p.dc_n[((size_t)dir * B + row) * H + j];
  }
  float bsum[G + 1];
#pragma unroll
  for (int g = 0; g <= G; ++g) bsum[g] = 0.f;
  float sv[G], sx = 0.f, hp = 0.f, dyv = 0.f;  // saved gates, hn / c_t, h_{prev} / c_{prev}, dy (prefetched)
#pragma unroll
  for (int g = 0; g < G; ++g) sv[g] = 0.f;
  const float* s0 = MODE == B200RNN_GRU ? p.h_0 : p.c_0;  // the state before the first step (zeros when NULL)
  auto load_step = [&](int step) {
    const int t = dir ? step : (T - 1 - step);
    const int tp = dir ? t + 1 : t - 1;
    // GRU, VL: the output at tp >= len is the masked 0, not the kept state; the LSTM reads the kept c from `extra`
    const bool has_prev = step < T - 1 && !(MODE == B200RNN_GRU && VL && tp >= len);
#pragma unroll
    for (int g = 0; g < G; ++g) sv[g] = gates[((size_t)t * B + row) * GH + g * H + j];
    sx = extra[((size_t)t * B + row) * H + j];
    dyv = p.dy[(long long)t * p.dy_st + (long long)row * p.dy_sb + dir * H + j];
    if (!has_prev)
      hp = s0 ? s0[((size_t)dir * B + row) * H + j] : 0.f;
    else if (MODE == B200RNN_GRU)
      hp = p.y[(long long)tp * p.y_st + (long long)row * p.y_sb + dir * H + j];
    else
      hp = extra[((size_t)tp * B + row) * H + j];
  };
  if (valid && T > 0) load_step(0);
  const bool want_dh0 = p.dh_0 != nullptr;

  for (int step = 0; step <= T; ++step) {
    if (step > 0) {  // dh of this step from the gate gradients step - 1 sent
      const int cur = step & 1;
      wait_bars(bars, cur, C, rank, ((step - 1) >> 1) & 1);
      float acc[G];
#pragma unroll
      for (int g = 0; g < G; ++g) acc[g] = 0.f;
      dot_rows<G, ONCHIP, true>(wrow, wg, d_s + ((size_t)cur * BS + b) * GH, H, H, acc);
      float sum = acc[0];
#pragma unroll
      for (int g = 1; g < G; ++g) sum += acc[g];
      dh_carry = direct + sum;
    }
    if (step == T) break;
    const int t = dir ? step : (T - 1 - step);
    const bool last = step == T - 1;
    const bool send = !last || want_dh0;
    const int nxt = (step + 1) & 1;
    if (tid == 0 && send) arm_bars(bars, nxt, s, H, G);

    const bool frozen = VL && t >= len;  // the output of a frozen step is the constant 0: its dy reaches nothing
    const float dh = frozen ? dh_carry : dh_carry + dyv;
    float dg[G], dhn = 0.f;
    if constexpr (MODE == B200RNN_GRU) {
      direct = gru_cell_bwd(sv, sx, hp, dh, dg, dhn);
    } else {
      const float dc_next = lstm_cell_bwd(sv, sx, hp, dh, dc_carry, dg);
      direct = 0.f;
      if (!frozen) dc_carry = dc_next;  // frozen: dh and dc pass straight through
    }
    if (frozen) {
#pragma unroll
      for (int g = 0; g < G; ++g) dg[g] = 0.f;
      dhn = 0.f;
      direct = dh;
    }
    if (valid) {
#pragma unroll
      for (int g = 0; g < G; ++g) bsum[g] += dg[g];
      bsum[G] += dhn;
      float* gp = dgates + ((size_t)t * B + row) * GH + j;
#pragma unroll
      for (int g = 0; g < G; ++g) gp[g * H] = dg[g];
      if (MODE == B200RNN_GRU) p.dghn[dir][((size_t)t * B + row) * H + j] = dhn;
    }
    if (!send) break;
    float* d_nxt = d_s + (size_t)nxt * BS * GH;
#pragma unroll
    for (int g = 0; g < G; ++g) {  // the recurrent-side gate gradient (GRU n block: dn * r)
      const float v = (MODE == B200RNN_GRU && g == 2) ? dhn : dg[g];
      if (s.active) d_nxt[(size_t)b * GH + g * H + j] = valid ? v : 0.f;
    }
    __syncthreads();  // the own slice is complete (and every thread is past step - 1's reads of buffer nxt)
    send_slice(d_nxt, GH, G, H, s, &bars[nxt * C + rank]);
    if (valid && !last) load_step(step + 1);
  }
  // gradients w.r.t. the initial state: what the scan carried past its first step (a cluster that ran no step passes
  // dh_n / dc_n on)
  if (valid) {
    if (want_dh0) p.dh_0[((size_t)dir * B + row) * H + j] = dh_carry;
    if (MODE == B200RNN_LSTM && p.dc_0) p.dc_0[((size_t)dir * B + row) * H + j] = dc_carry;
    if (VL)  // the steps [T, p.T) the cluster skipped: their gate gradients are 0
      for (int t = T; t < p.T; ++t) {
        float* gp = dgates + ((size_t)t * B + row) * GH + j;
#pragma unroll
        for (int g = 0; g < G; ++g) gp[g * H] = 0.f;
        if (MODE == B200RNN_GRU) p.dghn[dir][((size_t)t * B + row) * H + j] = 0.f;
      }
  }
  // per-slice bias-gradient partials: the slice's batch slots summed in slot order
  if (s.active) {
#pragma unroll
    for (int g = 0; g <= G; ++g) red[((size_t)b * (G + 1) + g) * HS + u] = bsum[g];
  }
  __syncthreads();
  if (s.active && b == 0) {
    float* out = p.dbias_part[dir] + (size_t)s.slice * (G + 1) * H;
    for (int g = 0; g <= G; ++g) {
      float v = 0.f;
      for (int q = 0; q < BS; ++q) v += red[((size_t)q * (G + 1) + g) * HS + u];
      out[g * H + j] = v;
    }
  }
  ptx::cluster_sync_all();
}

// The backward's W_hh, per CTA of a C-CTA cluster and contiguous: CTA r's block starts at G * j0_r * H and holds
// out[G*j0_r*H + (g*n_r + u)*H + jj] = W_hh[g*H + jj][j0_r + u] (anyh_units). For even slices this is whh_prep_kernel's
// layout; that kernel tiles by 32 and takes H / C units per CTA.
__global__ void anyh_prep_kernel(const float* __restrict__ w_hh, float* __restrict__ out, int G, int H, int C) {
  __shared__ float tile[32][33];
  const int nt = (H + 31) / 32;
  for (int tix = blockIdx.x; tix < G * nt * nt; tix += gridDim.x) {
    const int g = tix / (nt * nt), rem = tix - g * nt * nt;
    const int tj = rem / nt, tk = rem - tj * nt;  // row tile of the gate block, column tile
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
      const int r = tj * 32 + i, k = tk * 32 + threadIdx.x;
      tile[i][threadIdx.x] = (r < H && k < H) ? w_hh[((size_t)g * H + r) * H + k] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
      const int col = tk * 32 + i, jj = tj * 32 + threadIdx.x;
      if (col < H && jj < H) {
        int rk = (col / 8) * C / (H / 8), j0, n;  // the CTA that owns unit col (anyh_units), found from its group
        anyh_units(H, C, rk, j0, n);
        while (col >= j0 + n) anyh_units(H, C, ++rk, j0, n);
        while (col < j0) anyh_units(H, C, --rk, j0, n);
        out[(size_t)G * j0 * H + ((size_t)g * n + col - j0) * H + jj] = tile[threadIdx.x][i];
      }
    }
    __syncthreads();
  }
}

// =================================================================================================
// config choice
// =================================================================================================
size_t anyh_smem(int G, int H, int C, int BS, bool bwd, bool onchip) {
  const size_t HS = (size_t)anyh_max_units(H, C);
  size_t f = onchip ? (size_t)G * HS * (H + 4) : 0;
  f += (size_t)2 * BS * (bwd ? G * H : H);
  if (bwd) f += (size_t)BS * (G + 1) * HS;
  return f * sizeof(float) + (size_t)2 * C * sizeof(uint64_t);
}

// How many clusters of C CTAs of `kernel` (NT threads, smem bytes) can be co-resident, from the driver; cached per
// (kernel, device, shape). 0 when the query fails or the shape cannot run.
int anyh_capacity(const void* kernel, int C, int NT, size_t smem) {
  static std::mutex mu;
  static std::map<std::tuple<const void*, int, int, int, size_t>, int> cache;
  const auto key = std::make_tuple(kernel, current_device(), C, NT, smem);
  std::lock_guard<std::mutex> lk(mu);
  auto it = cache.find(key);
  if (it == cache.end()) {
    int n = 0;
    // every shape of the kernel may take up to the opt-in limit; 16-CTA clusters are non-portable
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_SMEM) == cudaSuccess &&
        cudaFuncSetAttribute(kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) == cudaSuccess) {
      cudaLaunchAttribute attr[1];
      attr[0].id = cudaLaunchAttributeClusterDimension;
      attr[0].val.clusterDim.x = (unsigned)C;
      attr[0].val.clusterDim.y = 1;
      attr[0].val.clusterDim.z = 1;
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = dim3((unsigned)(C * NUM_SMS), 1, 1);
      cfg.blockDim = dim3((unsigned)NT, 1, 1);
      cfg.dynamicSmemBytes = smem;
      cfg.attrs = attr;
      cfg.numAttrs = 1;
      if (cudaOccupancyMaxActiveClusters(&n, kernel, &cfg) != cudaSuccess) n = 0;
    }
    if (n == 0) cudaGetLastError();  // a failed query leaves its error pending: clear that one, not an older one
    it = cache.emplace(key, n).first;
  }
  return it->second;
}

template <int MODE>
AnyhKernel<RecFwdParams> anyh_kernel(const RecFwdParams&, bool vl, bool onchip) {
  return vl ? (onchip ? anyh_fwd_kernel<MODE, true, true> : anyh_fwd_kernel<MODE, true, false>)
            : (onchip ? anyh_fwd_kernel<MODE, false, true> : anyh_fwd_kernel<MODE, false, false>);
}
template <int MODE>
AnyhKernel<RecBwdParams> anyh_kernel(const RecBwdParams&, bool vl, bool onchip) {
  return vl ? (onchip ? anyh_bwd_kernel<MODE, true, true> : anyh_bwd_kernel<MODE, true, false>)
            : (onchip ? anyh_bwd_kernel<MODE, false, true> : anyh_bwd_kernel<MODE, false, false>);
}

// The cluster shape of one launch. Candidates: C in {2, 4, 8, 16} with at least one group of 8 units per CTA
// (anyh_units: every multiple of 16 from 16 to 1024 has one), BS in {2, 4, ..., 64}, NT = HS * BS rounded up to whole
// warps (HS: the widest CTA's units), at most 512 threads. The weights stay on chip when any candidate's
// slice and buffers fit MAX_SMEM; only when none does is the L2 tier taken.
//   * On chip, a step costs each SM its G*H*HS*BS FMAs: the shape with the fewest waves x max(NT, 128) wins (a CTA of up
//     to 4 warps has one warp per scheduler, so a smaller one shortens no step), ties to the fewest CTAs.
//   * In the L2 tier a step costs each CTA its G*HS*H weights streamed from L2, whatever BS (a warp's batch slots share
//     every load): the widest cluster, then the fewest waves, then the fewest batch rows.
// Capacities come from the driver (anyh_capacity), never from the SM count; clusters that do not fit run in waves.
template <typename P>
int plan_anyh(const P& p, bool bwd, ClusterLaunch<P>* L) {
  const int G = gates_of(p.mode), H = p.H;
  const bool vl = p.lengths != nullptr;
  for (int tier = 0; tier < 2; ++tier) {
    const bool onchip = tier == 0;
    const AnyhKernel<P> kernel = p.mode == B200RNN_GRU    ? anyh_kernel<B200RNN_GRU>(p, vl, onchip)
                                 : p.mode == B200RNN_LSTM ? anyh_kernel<B200RNN_LSTM>(p, vl, onchip)
                                                          : elman_kernel(p, vl, onchip);
    bool found = false;
    long long best[3] = {0, 0, 0};
    ClusterLaunch<P> pick{};
    for (int C = 2; C <= 16; C *= 2) {
      if (C > H / 8) continue;
      const int HS = anyh_max_units(H, C);
      for (int BS = 2; BS <= 64; BS *= 2) {
        const int NT = (HS * BS + 31) / 32 * 32;
        if (NT > ANYH_MAX_NT) continue;
        const size_t smem = anyh_smem(G, H, C, BS, bwd, onchip);
        if (smem > (size_t)MAX_SMEM) continue;
        const int nslices = (p.B + BS - 1) / BS, nclusters = nslices * p.D;
        const int capacity = anyh_capacity((const void*)kernel, C, NT, smem);
        if (capacity <= 0) continue;
        const long long waves = (nclusters + capacity - 1) / capacity;
        long long key[3];
        if (onchip) {
          key[0] = waves * (NT > 128 ? NT : 128); key[1] = (long long)nclusters * C; key[2] = 0;
        } else {
          key[0] = -C; key[1] = waves; key[2] = BS;
        }
        if (!found || key[0] < best[0] || (key[0] == best[0] && (key[1] < best[1] ||
                                                                  (key[1] == best[1] && key[2] < best[2])))) {
          found = true;
          best[0] = key[0]; best[1] = key[1]; best[2] = key[2];
          pick = ClusterLaunch<P>{kernel, C, NT, nslices, nclusters, capacity, smem};
          pick.anyh = true;
          pick.BS = BS;
          pick.onchip = onchip;
        }
      }
    }
    if (found) {
      static const bool debug = getenv("B200RNN_DEBUG") != nullptr;
      if (debug)
        fprintf(stderr, "[b200rnn] %s %s cfg %s VL=%d H=%d C=%d BS=%d tier=%s: need %d clusters, capacity %d, smem %zu\n",
                bwd ? "bwd" : "fwd", G == 1 ? "elman" : "anyh", mode_name(p.mode), (int)vl, H, pick.C, pick.BS,
                onchip ? "smem" : "l2", pick.nclusters, pick.capacity, pick.smem);
      *L = pick;
      return B200RNN_OK;
    }
  }
  set_error("recurrence: no cluster shape runs hidden_size %d on this device", H);
  return B200RNN_ERR_UNSUPPORTED;
}

}  // namespace

bool anyh_hidden_size(int H) { return H >= 16 && H <= 1024 && H % 16 == 0; }

int plan_anyh_fwd(const RecFwdParams& p, RecFwdLaunch* L) {
  if (p.y_pool || p.ready || p.shell_nograd || p.P > 0) {
    set_error("recurrence: hidden_size %d runs without the model-shell fusions (y_pool, streamed x-projection, "
              "no-grad fused forward) and without proj_size", p.H);
    return B200RNN_ERR_UNSUPPORTED;
  }
  return plan_anyh(p, false, L);
}

int plan_anyh_bwd(const RecBwdParams& p, RecBwdLaunch* L) {
  if (!p.dy || p.P > 0) {
    set_error("recurrence backward: hidden_size %d takes the full output gradient dy and no proj_size", p.H);
    return B200RNN_ERR_UNSUPPORTED;
  }
  return plan_anyh(p, true, L);
}

int launch_anyh_prep(const float* w_hh, float* w_prep, int G, int H, int C, cudaStream_t s) {
  anyh_prep_kernel<<<NUM_SMS, dim3(32, 8), 0, s>>>(w_hh, w_prep, G, H, C);
  if (cudaGetLastError() != cudaSuccess) {
    set_error("anyh_prep launch failed");
    return B200RNN_ERR_CUDA;
  }
  count_launch();
  return B200RNN_OK;
}

}  // namespace b200rnn
