// rnn_anyh.cu — the runtime-sized recurrence, forward and BPTT, at every hidden size H % 16 == 0, 16 <= H <= 1024: the
// GRU / LSTM at the sizes the fixed configs of rnn_rec.cu (H = 128, 256) do not cover, and the Elman RNN
// (torch.nn.RNN, nonlinearity 'tanh' or 'relu') at all of them. H, the cluster width C and the batch rows per cluster BS
// are known only at run time; the kernels are templated on the mode, ragged batches (VL) and where W_hh lives (ONCHIP).
// The Elman kernels are instantiated once, as B200RNN_RNN_TANH, with one gate block (G = 1); the nonlinearity is the
// warp-uniform runtime flag p.mode.
//
// Same launch shape and contract as rec_fwd_kernel / rec_bwd_kernel (rnn_kernels.cuh): grid = D * nslices clusters of C
// CTAs, cluster = one direction of BS batch slots. The H / 8 groups of 8 units are split as evenly as possible over the
// C CTAs (anyh_units): CTA `rank` owns n units from j0, n a multiple of 8 and at most HS = 8 * ceil(H / 8 / C), so every
// multiple of 16 has a shape, and a CTA's slice of a state row is a whole number of 16-byte chunks. One thread per
// (unit u, batch slot b), 8 consecutive units by BS slots per group of 8 * BS threads (the projected kernels'
// proj_thread), NT = HS * BS rounded up to whole warps; threads past the CTA's units are idle.
//   * Weights: ONCHIP, the CTA's G * n rows (forward: W_hh[g*H + j0 + u][:]; backward: W_hh[g*H + :][j0 + u], the
//     w_prep slice of whh_prep_kernel) are staged once into shared memory, rows padded to H + 4 floats so that the 8
//     units a quarter-warp reads with one 16-byte load sit in different banks. Otherwise (the L2 tier) the same rows are
//     read from global memory every step: weight_hh in place in the forward, w_prep in the backward.
//   * Step: G fixed-order FFMA chains of length H per thread (k ascending), the cell of rnn_cell.cuh, then the CTA's
//     slice of the new state (forward: h_t, BS x n; backward: the recurrent-side gate gradients, BS x G*n) is written
//     into its own buffer with ordinary stores (published by __syncthreads) and sent to the C - 1 peers with st.async,
//     which completes transaction bytes on the destination's mbarrier of that source and buffer. Double buffered:
//     step s contracts against what step s - 1 sent (the ExchangeBars protocol of rnn_rec.cu with LAG = 1).
//   * Elman: the forward saves the activated h_t as its one gate block and nothing in `extra`; the backward takes
//     dpre = dh (1 - h^2) for tanh, dh [h > 0] for relu from that saved h_t (elman_cell_bwd).
//   * The waits are bounded: a protocol bug traps (a CUDA error) instead of hanging the GPU.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdlib.h>

#include "h16.cuh"
#include "ptx.cuh"
#include "rnn_cell.cuh"
#include "rnn_kernels.cuh"

namespace b200rnn {

namespace {

constexpr int ANYH_MAX_NT = 512;  // 128 registers per thread: the step keeps G accumulators and G + 1 float4 loads in flight

__device__ __forceinline__ uint32_t cluster_nctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
  return r;
}

// mbarrier phase wait that gives up after ~2^24 polls (seconds): a lost exchange becomes a trap, not a hang
__device__ __forceinline__ void bounded_wait(uint64_t* bar, uint32_t parity) {
  for (uint32_t n = 0; !ptx::mbar_try_wait(bar, parity); ++n)
    if (n > (1u << 24)) __trap();
}

// What a CTA owns, derived from the launch: C from the cluster, its units from anyh_units, BS = ceil(B / nslices) batch
// slots (at most the BS the host planned with: the shared-memory layout uses this one). Threads whose unit is past the
// CTA's n units (a partial last warp, or a CTA with fewer units than the widest) are idle: they take unit 0's operands,
// meet every barrier, and store nothing.
struct AnyhSlice {
  int C, HS, BS, NT;  // HS: units of the widest CTA (the row count of W_s)
  uint32_t rank;
  int dir, slice, b0, j0, n, T;  // units [j0, j0 + n); T: steps the cluster runs (VL: its longest row's)
  int u, b;                      // this thread's unit (within the slice; 0 when idle) and batch slot
  bool active;
};

template <bool VL, typename Params>
__device__ __forceinline__ AnyhSlice anyh_slice(const Params& p, int nslices) {
  AnyhSlice s;
  s.C = (int)cluster_nctarank();
  s.HS = anyh_max_units(p.H, s.C);
  s.NT = (int)blockDim.x;
  s.BS = (p.B + nslices - 1) / nslices;
  s.rank = ptx::cluster_ctarank();
  const int cid = (blockIdx.x / s.C) % (p.D * nslices);  // clusters: model-major (anyh_model), direction, slice
  s.dir = cid / nslices;
  s.slice = cid - s.dir * nslices;
  s.b0 = s.slice * s.BS;
  anyh_units(p.H, s.C, (int)s.rank, s.j0, s.n);
  s.T = VL ? min(max(p.lengths[p.order[s.b0]], 0), p.T) : p.T;
  const int tid = threadIdx.x;
  s.u = (tid & 7) + 8 * (tid / (8 * s.BS));
  s.b = (tid >> 3) % s.BS;
  s.active = s.u < s.n;
  if (!s.active) s.u = 0;
  return s;
}

// The model of this CTA's cluster when one launch runs several (RecModels): clusters are model-major
template <typename Params>
__device__ __forceinline__ int anyh_model(const Params& p, int nslices) {
  return (int)(blockIdx.x / (cluster_nctarank() * p.D * nslices));
}

// Thread 0: the [2][C] exchange barriers, one arrival (the local arm) per phase
__device__ __forceinline__ void init_bars(uint64_t* bars, int C) {
  for (int i = 0; i < 2 * C; ++i) ptx::mbar_init(&bars[i], 1u);
  ptx::fence_mbar_init();
}

// Thread 0: buffer `buf` expects from every peer its slice: BS rows of NB blocks of its units
__device__ __forceinline__ void arm_bars(uint64_t* bars, int buf, const AnyhSlice& s, int H, int NB) {
  for (int src = 0; src < s.C; ++src) {
    if ((uint32_t)src == s.rank) continue;
    int j0, n;
    anyh_units(H, s.C, src, j0, n);
    ptx::mbar_arrive_expect_tx(&bars[buf * s.C + src], (uint32_t)(s.BS * NB * n * sizeof(float)));
  }
}

// Every thread: the peers' slices of buffer `buf` have landed
__device__ __forceinline__ void wait_bars(uint64_t* bars, int buf, int C, uint32_t rank, uint32_t parity) {
  for (int src = 0; src < C; ++src)
    if ((uint32_t)src != rank) bounded_wait(&bars[buf * C + src], parity);
}

// Send this CTA's slice of buffer `vec` (BS rows of `width` floats, NB blocks of its n units from column j0 + k * H of
// each row) to the same place in every peer, completing the bytes on the peer's barrier `bar` (this CTA's source slot)
__device__ __forceinline__ void send_slice(float* vec, int width, int NB, int H, const AnyhSlice& s, uint64_t* bar) {
  const int per_row = NB * s.n / 4;  // 16-byte chunks of one row
  const int n = s.BS * per_row;
  const uint32_t bar_addr = ptx::smem_u32(bar);
  for (int i = threadIdx.x; i < (s.C - 1) * n; i += s.NT) {
    const int r = i / n, v = i - r * n;
    const int q = v / per_row, c = v - q * per_row;
    const int blk = c / (s.n / 4), e = c - blk * (s.n / 4);
    float* src = vec + (size_t)q * width + s.j0 + blk * H + e * 4;
    const uint32_t peer = (s.rank + 1 + (uint32_t)r) % (uint32_t)s.C;
    ptx::st_async_v4(ptx::mapa(ptx::smem_u32(src), peer), *reinterpret_cast<const float4*>(src),
                     ptx::mapa(bar_addr, peer));
  }
}

// acc[g] += sum_k w[g * wg + k] * v[g * vg + k], k ascending (one FMA chain per gate: deterministic); vg = 0 in the
// forward (one state row), H in the backward (gate block g of the gradient row). w from shared memory or, in the L2
// tier, from global memory (read-only for the whole launch). WT: the storage of w, float or 16-bit (__half /
// __nv_bfloat16, widened exactly in registers: the same chains)
template <typename WT>
__device__ __forceinline__ float4 widen4(uint2 u) {
  if constexpr (__is_same(WT, __nv_bfloat16)) {
    return make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xffff0000u), __uint_as_float(u.y << 16),
                       __uint_as_float(u.y & 0xffff0000u));
  } else {
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
    const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
    return make_float4(a.x, a.y, b.x, b.y);
  }
}
template <int G, bool ONCHIP, bool PER_GATE_V>
__device__ __forceinline__ void dot_rows(const float* __restrict__ w, size_t wg, const float* __restrict__ v, int vg,
                                         int K, float (&acc)[G]) {
  // the backward loads G gradient vectors per k, the L2-tier LSTM forward four global rows: no deeper, or they spill
  constexpr int UNROLL = PER_GATE_V ? 1 : (G == 4 && !ONCHIP) ? 2 : 4;
#pragma unroll UNROLL
  for (int k = 0; k < K; k += 4) {
    float4 x = *reinterpret_cast<const float4*>(v + k);
#pragma unroll
    for (int g = 0; g < G; ++g) {
      if (PER_GATE_V && g > 0) x = *reinterpret_cast<const float4*>(v + g * vg + k);
      const float4 a = ONCHIP ? *reinterpret_cast<const float4*>(w + g * wg + k)
                              : __ldg(reinterpret_cast<const float4*>(w + g * wg + k));
      float r = acc[g];
      r = fmaf(a.x, x.x, r);
      r = fmaf(a.y, x.y, r);
      r = fmaf(a.z, x.z, r);
      r = fmaf(a.w, x.w, r);
      acc[g] = r;
    }
  }
}
// The same chains over 16-bit weights, widened exactly in registers (8-byte loads of 4 weights)
template <int G, bool ONCHIP, bool PER_GATE_V, typename WT>
__device__ __forceinline__ void dot_rows16(const WT* __restrict__ w, size_t wg, const float* __restrict__ v, int vg,
                                           int K, float (&acc)[G]) {
  constexpr int UNROLL = PER_GATE_V ? 1 : (G == 4 && !ONCHIP) ? 2 : 4;
#pragma unroll UNROLL
  for (int k = 0; k < K; k += 4) {
    float4 x = *reinterpret_cast<const float4*>(v + k);
#pragma unroll
    for (int g = 0; g < G; ++g) {
      if (PER_GATE_V && g > 0) x = *reinterpret_cast<const float4*>(v + g * vg + k);
      const float4 a = widen4<WT>(ONCHIP ? *reinterpret_cast<const uint2*>(w + g * wg + k)
                                         : __ldg(reinterpret_cast<const uint2*>(w + g * wg + k)));
      float r = acc[g];
      r = fmaf(a.x, x.x, r);
      r = fmaf(a.y, x.y, r);
      r = fmaf(a.z, x.z, r);
      r = fmaf(a.w, x.w, r);
      acc[g] = r;
    }
  }
}
// Stage rows r = 0 .. rows-1 of length H (row r at src + rowoff(r)) into W_s[r][H + 4]
template <typename RowOff>
__device__ __forceinline__ void stage_rows(float* W_s, const float* __restrict__ src, int rows, int H, int NT,
                                           RowOff rowoff) {
  const int q4 = H / 4, LD = H + 4;
  for (int i = threadIdx.x; i < rows * q4; i += NT) {
    const int r = i / q4, k = (i - r * q4) * 4;
    *reinterpret_cast<float4*>(&W_s[(size_t)r * LD + k]) = __ldg(reinterpret_cast<const float4*>(src + rowoff(r) + k));
  }
}

// The same with 16-bit rows: W_s[r][H + 8], 16-byte chunks of 8 elements (the pad keeps 16 bytes, as above)
template <typename WT, typename RowOff>
__device__ __forceinline__ void stage_rows16(WT* W_s, const WT* __restrict__ src, int rows, int H, int NT, RowOff rowoff) {
  const int q8 = H / 8, LD = H + 8;
  for (int i = threadIdx.x; i < rows * q8; i += NT) {
    const int r = i / q8, k = (i - r * q8) * 8;
    *reinterpret_cast<uint4*>(&W_s[(size_t)r * LD + k]) = __ldg(reinterpret_cast<const uint4*>(src + rowoff(r) + k));
  }
}

// =================================================================================================
// forward
// =================================================================================================
// Shared memory: [W_s: G*n x (H+4), ONCHIP only] [h: 2 x BS x H] [bars: 2 x C]
template <int MODE, bool VL, bool ONCHIP>
__global__ void __launch_bounds__(ANYH_MAX_NT, 1) anyh_fwd_kernel(const RecFwdParams p, const int nslices, const RecModels mdl) {
  constexpr int G = gates_of(MODE);
  const int H = p.H, B = p.B, LD = H + 4;
  const bool relu = p.mode == B200RNN_RNN_RELU;  // Elman
  const AnyhSlice s = anyh_slice<VL>(p, nslices);
  const int C = s.C, HS = s.HS, BS = s.BS, NT = s.NT, dir = s.dir, b0 = s.b0, j0 = s.j0, n = s.n, T = s.T;
  const uint32_t rank = s.rank;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* W_s = reinterpret_cast<float*>(smem_raw);  // [G][n][LD]
  float* h_s = W_s + (ONCHIP ? (size_t)G * HS * LD : 0);
  uint64_t* bars = reinterpret_cast<uint64_t*>(h_s + (size_t)2 * BS * H);
  const int tid = threadIdx.x;
  // this cluster's model: every pointer offset by the model's block (0 for model 0, or for a shared tensor). The GRU's
  // L2 tier, which has no register to spare in its step loop, reads the index again from the launch registers each time
  constexpr bool REMAT = !ONCHIP && MODE == B200RNN_GRU;
  const int m = mdl.M > 1 ? anyh_model(p, nslices) : 0;
  auto moff = [&](long long stride) {
    if constexpr (!REMAT) return (long long)m * stride;
    return mdl.M > 1 ? (long long)anyh_model(p, nslices) * stride : 0ll;
  };
  const float* w_hh = p.w_hh[dir] + m * (dir ? mdl.whh[1] : mdl.whh[0]);
  const float* h_0 = p.h_0 ? p.h_0 + m * mdl.state : nullptr;
  const float* c_0 = p.c_0 ? p.c_0 + m * mdl.state : nullptr;

  if (tid == 0) init_bars(bars, C);
  if constexpr (ONCHIP) {
    if constexpr (G == 1)
      stage_rows(W_s, w_hh, n, H, NT, [&](int r) { return (size_t)(j0 + r) * H; });
    else
      stage_rows(W_s, w_hh, G * n, H, NT, [&](int r) { return ((size_t)(r / n) * H + j0 + r % n) * H; });
  }
  for (int i = tid; i < BS * H; i += NT) {  // buffer 0: h_0 of the cluster's slots (zeros past the batch / without h_0)
    const int q = i / H, k = i - q * H;
    const int slot = b0 + q;
    float v = 0.f;
    if (h_0 && slot < B) v = h_0[((size_t)dir * B + (VL ? p.order[slot] : slot)) * H + k];
    h_s[i] = v;
  }
  __syncthreads();
  ptx::cluster_sync_all();  // peers' barriers are initialised before anyone sends

  const int u = s.u, b = s.b, j = j0 + u, slot = b0 + b;
  const bool valid = s.active && slot < B;
  const int row = valid ? (VL ? p.order[slot] : slot) : 0;
  const int len = (VL && valid) ? p.lengths[row] : p.T;
  float* gates = p.gates[dir];
  float h = (h_0 && valid) ? h_0[((size_t)dir * B + row) * H + j] : 0.f;
  float c = (MODE == B200RNN_LSTM && c_0 && valid) ? c_0[((size_t)dir * B + row) * H + j] : 0.f;
  const float bhn = MODE == B200RNN_GRU ? p.b_hh[dir][m * (dir ? mdl.bhh[1] : mdl.bhh[0]) + 2 * H + j] : 0.f;
  float gi[G];
  // Elman: 0 until the first load, the register allocation its timings (tools/elman_steps_results.json) were taken with
  if constexpr (G == 1) gi[0] = 0.f;
  auto load_gi = [&](int t) {
#pragma unroll
    for (int g = 0; g < G; ++g) gi[g] = valid ? gates[moff(mdl.saved) + ((size_t)t * B + row) * (G * H) + g * H + j] : 0.f;
  };
  if (T > 0) load_gi(dir ? T - 1 : 0);
  const size_t wg = ONCHIP ? (size_t)n * LD : (size_t)H * H;

  for (int step = 0; step < T; ++step) {
    const int t = dir ? T - 1 - step : step;
    const int cur = step & 1, nxt = cur ^ 1;
    if (step > 0) wait_bars(bars, cur, C, rank, ((step - 1) >> 1) & 1);
    if (tid == 0 && step + 1 < T) arm_bars(bars, nxt, s, H, 1);
    float acc[G];
#pragma unroll
    for (int g = 0; g < G; ++g) acc[g] = 0.f;
    // the L2 tier reads this model's weight_hh in place (its address formed per step where REMAT)
    const float* wrow = ONCHIP ? W_s + (size_t)u * LD
                               : p.w_hh[dir] + moff(dir ? mdl.whh[1] : mdl.whh[0]) + (size_t)(j0 + u) * H;
    dot_rows<G, ONCHIP, false>(wrow, wg, h_s + ((size_t)cur * BS + b) * H, 0, H, acc);

    float hnew, sg[G], sx;
    const bool frozen = VL && t >= len;  // past its length a row keeps its state and emits 0
    if constexpr (MODE == B200RNN_GRU) {
      const GruStep st = gru_cell_fwd(gi, acc, bhn, h);
      hnew = frozen ? h : st.h;
      sg[0] = st.r; sg[1] = st.z; sg[2] = st.n; sx = st.hn;
    } else if constexpr (MODE == B200RNN_LSTM) {
      const LstmStep st = lstm_cell_fwd(gi, acc, c);
      hnew = frozen ? h : st.h;
      c = frozen ? c : st.c;
      sg[0] = st.i; sg[1] = st.f; sg[2] = st.g; sg[3] = st.o; sx = c;
    } else {
      sg[0] = elman_cell_fwd(gi[0], acc[0], relu);
      hnew = frozen ? h : sg[0];
    }
    h = hnew;
    if (valid) {
      if (p.y) p.y[moff(mdl.y) + (long long)t * p.y_st + (long long)row * p.y_sb + dir * H + j] = frozen ? 0.f : hnew;
      if (p.training) {  // the activated gates over the x-projection, and GRU W_hn h + b_hn / LSTM c_t (Elman: h_t)
        float* gp = gates + moff(mdl.saved) + ((size_t)t * B + row) * (G * H) + j;
#pragma unroll
        for (int g = 0; g < G; ++g) gp[g * H] = sg[g];
        if constexpr (G > 1) p.extra[dir][moff(mdl.saved) + ((size_t)t * B + row) * H + j] = sx;
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
    p.h_n[moff(mdl.state) + ((size_t)dir * B + row) * H + j] = h;
    if (MODE == B200RNN_LSTM && p.c_n) p.c_n[moff(mdl.state) + ((size_t)dir * B + row) * H + j] = c;
    if (VL && p.y)  // the steps [T, p.T) the cluster skipped emit 0, as past any sequence's length
      for (int t = T; t < p.T; ++t) p.y[moff(mdl.y) + (long long)t * p.y_st + (long long)row * p.y_sb + dir * H + j] = 0.f;
  }
  ptx::cluster_sync_all();  // nobody exits while a peer could still address its shared memory
}

// The forward over a 16-bit weight_hh (WT = __half / __nv_bfloat16), anyh16_fwd_kernel: anyh_fwd_kernel's step with
// rows of H + 8 elements on chip and the weights widened in registers (dot_rows16). anyh_fwd_kernel keeps its own
// text so that the fp32 instantiations compile exactly as before.
// Shared memory: [W_s: G*n x (H+8) WT, ONCHIP only] [h: 2 x BS x H] [bars: 2 x C]
template <int MODE, bool VL, bool ONCHIP, typename WT>
__device__ __forceinline__ void anyh_fwd_body(const RecFwdParams p, const int nslices) {
  constexpr int G = gates_of(MODE);
  const int H = p.H, B = p.B, LD = H + 8;
  const bool relu = p.mode == B200RNN_RNN_RELU;  // Elman
  const AnyhSlice s = anyh_slice<VL>(p, nslices);
  const int C = s.C, HS = s.HS, BS = s.BS, NT = s.NT, dir = s.dir, b0 = s.b0, j0 = s.j0, n = s.n, T = s.T;
  const uint32_t rank = s.rank;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  WT* W_s = reinterpret_cast<WT*>(smem_raw);  // [G][n][LD]
  float* h_s = reinterpret_cast<float*>(W_s + (ONCHIP ? (size_t)G * HS * LD : 0));
  uint64_t* bars = reinterpret_cast<uint64_t*>(h_s + (size_t)2 * BS * H);
  const int tid = threadIdx.x;
  const WT* w_hh = reinterpret_cast<const WT*>(p.w_hh[dir]);

  if (tid == 0) init_bars(bars, C);
  if constexpr (ONCHIP) {
    if constexpr (G == 1)
      stage_rows16(W_s, w_hh, n, H, NT, [&](int r) { return (size_t)(j0 + r) * H; });
    else
      stage_rows16(W_s, w_hh, G * n, H, NT, [&](int r) { return ((size_t)(r / n) * H + j0 + r % n) * H; });
  }
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
  // Elman: 0 until the first load, the register allocation its timings (tools/elman_steps_results.json) were taken with
  if constexpr (G == 1) gi[0] = 0.f;
  auto load_gi = [&](int t) {
#pragma unroll
    for (int g = 0; g < G; ++g) gi[g] = valid ? gates[((size_t)t * B + row) * (G * H) + g * H + j] : 0.f;
  };
  if (T > 0) load_gi(dir ? T - 1 : 0);
  const WT* wrow = ONCHIP ? W_s + (size_t)u * LD : w_hh + (size_t)(j0 + u) * H;
  const size_t wg = ONCHIP ? (size_t)n * LD : (size_t)H * H;

  for (int step = 0; step < T; ++step) {
    const int t = dir ? T - 1 - step : step;
    const int cur = step & 1, nxt = cur ^ 1;
    if (step > 0) wait_bars(bars, cur, C, rank, ((step - 1) >> 1) & 1);
    if (tid == 0 && step + 1 < T) arm_bars(bars, nxt, s, H, 1);
    float acc[G];
#pragma unroll
    for (int g = 0; g < G; ++g) acc[g] = 0.f;
    dot_rows16<G, ONCHIP, false, WT>(wrow, wg, h_s + ((size_t)cur * BS + b) * H, 0, H, acc);

    float hnew, sg[G], sx;
    const bool frozen = VL && t >= len;  // past its length a row keeps its state and emits 0
    if constexpr (MODE == B200RNN_GRU) {
      const GruStep st = gru_cell_fwd(gi, acc, bhn, h);
      hnew = frozen ? h : st.h;
      sg[0] = st.r; sg[1] = st.z; sg[2] = st.n; sx = st.hn;
    } else if constexpr (MODE == B200RNN_LSTM) {
      const LstmStep st = lstm_cell_fwd(gi, acc, c);
      hnew = frozen ? h : st.h;
      c = frozen ? c : st.c;
      sg[0] = st.i; sg[1] = st.f; sg[2] = st.g; sg[3] = st.o; sx = c;
    } else {
      sg[0] = elman_cell_fwd(gi[0], acc[0], relu);
      hnew = frozen ? h : sg[0];
    }
    h = hnew;
    if (valid) {
      if (p.y) p.y[(long long)t * p.y_st + (long long)row * p.y_sb + dir * H + j] = frozen ? 0.f : hnew;
      if (p.training) {  // the activated gates over the x-projection, and GRU W_hn h + b_hn / LSTM c_t (Elman: h_t)
        float* gp = gates + ((size_t)t * B + row) * (G * H) + j;
#pragma unroll
        for (int g = 0; g < G; ++g) gp[g * H] = sg[g];
        if constexpr (G > 1) p.extra[dir][((size_t)t * B + row) * H + j] = sx;
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


// 16-bit weight_hh (__half or __nv_bfloat16): half the shared memory per weight row, so more hidden sizes stay on chip
template <int MODE, bool VL, bool ONCHIP, typename WT>
__global__ void __launch_bounds__(ANYH_MAX_NT, 1) anyh16_fwd_kernel(const RecFwdParams p, const int nslices, const RecModels) {
  anyh_fwd_body<MODE, VL, ONCHIP, WT>(p, nslices);
}

// =================================================================================================
// backward (BPTT)
// =================================================================================================
// Shared memory: [W_s: G*n x (H+4), ONCHIP only] [d: 2 x BS x G*H] [red: BS x NP x HS] [bars: 2 x C]
// Step s: dh = direct_{s-1} + sum_g W_hh[g-block]^T dgh_{s-1} (the exchange of step s - 1, all G*H columns), the cell
// backward, then this CTA's dgh (GRU: n-block dn * r; Elman: dpre) to every CTA. Step T only contracts, for dh_0.
template <int MODE, bool VL, bool ONCHIP>
__global__ void __launch_bounds__(ANYH_MAX_NT, 1) anyh_bwd_kernel(const RecBwdParams p, const int nslices, const RecModels mdl) {
  constexpr int G = gates_of(MODE);
  constexpr int NP = G == 1 ? 1 : G + 1;  // bias-partial blocks per slice: dGi (+ the GRU dghn block, 0 for the LSTM)
  const int H = p.H, B = p.B, LD = H + 4, GH = G * H;
  const bool relu = p.mode == B200RNN_RNN_RELU;  // Elman
  const AnyhSlice s = anyh_slice<VL>(p, nslices);
  const int C = s.C, HS = s.HS, BS = s.BS, NT = s.NT, dir = s.dir, b0 = s.b0, j0 = s.j0, n = s.n, T = s.T;
  const uint32_t rank = s.rank;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* W_s = reinterpret_cast<float*>(smem_raw);  // [G][n][LD]
  float* d_s = W_s + (ONCHIP ? (size_t)G * HS * LD : 0);
  float* red = d_s + (size_t)2 * BS * GH;
  uint64_t* bars = reinterpret_cast<uint64_t*>(red + (size_t)BS * NP * HS);
  const int tid = threadIdx.x;
  // rows (g, u) of this CTA: W_hh[g*H + :][j0 + u], contiguous from G * j0 * H (whh_prep_kernel)
  // this cluster's model: every pointer offset by the model's block (0 for model 0, or for a shared tensor)
  const long long m = mdl.M > 1 ? anyh_model(p, nslices) : 0;
  const float* w_prep = p.w_prep[dir] + m * (dir ? mdl.wprep[1] : mdl.wprep[0]) + (size_t)G * j0 * H;

  if (tid == 0) init_bars(bars, C);
  if constexpr (ONCHIP) stage_rows(W_s, w_prep, G * n, H, NT, [&](int r) { return (size_t)r * H; });
  __syncthreads();
  ptx::cluster_sync_all();

  const int u = s.u, b = s.b, j = j0 + u, slot = b0 + b;
  const bool valid = s.active && slot < B;
  const int row = valid ? (VL ? p.order[slot] : slot) : 0;
  const int len = (VL && valid) ? p.lengths[row] : T;
  const float* gates = p.gates[dir] + m * mdl.saved;
  const float* extra = p.extra[dir] ? p.extra[dir] + m * mdl.saved : nullptr;
  float* dgates = p.dgates[dir] + m * mdl.scr;
  float* dghn = p.dghn[dir] ? p.dghn[dir] + m * mdl.scr : nullptr;
  const float* y = p.y + m * mdl.y;
  const float* dy = p.dy + m * mdl.dy;
  const float* dh_n = p.dh_n ? p.dh_n + m * mdl.state : nullptr;
  const float* dc_n = p.dc_n ? p.dc_n + m * mdl.state : nullptr;
  float* dh_0 = p.dh_0 ? p.dh_0 + m * mdl.state : nullptr;
  float* dc_0 = p.dc_0 ? p.dc_0 + m * mdl.state : nullptr;
  const float* wrow = ONCHIP ? W_s + (size_t)u * LD : w_prep + (size_t)u * H;
  const size_t wg = ONCHIP ? (size_t)n * LD : (size_t)n * H;

  float dh_carry = 0.f, dc_carry = 0.f, direct = 0.f;
  if (valid) {
    if (dh_n) dh_carry = dh_n[((size_t)dir * B + row) * H + j];
    if (MODE == B200RNN_LSTM && dc_n) dc_carry = dc_n[((size_t)dir * B + row) * H + j];
  }
  float bsum[NP] = {};
  // saved gates (Elman: h_t), hn / c_t, h_{prev} / c_{prev}, dy (prefetched)
  float sv[G] = {}, sx = 0.f, hp = 0.f, dyv = 0.f;
  const float* s0 = MODE == B200RNN_GRU ? p.h_0 : p.c_0;  // the state before the first step (zeros when NULL)
  if (s0) s0 += m * mdl.state;
  auto load_step = [&](int step) {
    const int t = dir ? step : (T - 1 - step);
    const int tp = dir ? t + 1 : t - 1;
    // GRU, VL: the output at tp >= len is the masked 0, not the kept state; the LSTM reads the kept c from `extra`
    const bool has_prev = step < T - 1 && !(MODE == B200RNN_GRU && VL && tp >= len);
#pragma unroll
    for (int g = 0; g < G; ++g) sv[g] = gates[((size_t)t * B + row) * GH + g * H + j];
    if constexpr (G > 1) sx = extra[((size_t)t * B + row) * H + j];
    dyv = dy[(long long)t * p.dy_st + (long long)row * p.dy_sb + dir * H + j];
    if constexpr (G > 1) {
      if (!has_prev)
        hp = s0 ? s0[((size_t)dir * B + row) * H + j] : 0.f;
      else if (MODE == B200RNN_GRU)
        hp = y[(long long)tp * p.y_st + (long long)row * p.y_sb + dir * H + j];
      else
        hp = extra[((size_t)tp * B + row) * H + j];
    }
  };
  if (valid && T > 0) load_step(0);
  const bool want_dh0 = dh_0 != nullptr;

  for (int step = 0; step <= T; ++step) {
    if (step > 0) {  // dh of this step from the gate gradients step - 1 sent
      const int cur = step & 1;
      wait_bars(bars, cur, C, rank, ((step - 1) >> 1) & 1);
      float acc[G];
#pragma unroll
      for (int g = 0; g < G; ++g) acc[g] = 0.f;
      dot_rows<G, ONCHIP, (G > 1)>(wrow, wg, d_s + ((size_t)cur * BS + b) * GH, H, H, acc);
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
    } else if constexpr (MODE == B200RNN_LSTM) {
      const float dc_next = lstm_cell_bwd(sv, sx, hp, dh, dc_carry, dg);
      direct = 0.f;
      if (!frozen) dc_carry = dc_next;  // frozen: dh and dc pass straight through
    } else {  // Elman: dpre from the saved h_t; frozen as below
      dg[0] = frozen ? 0.f : elman_cell_bwd(sv[0], dh, relu);
      direct = frozen ? dh : 0.f;
    }
    if (G > 1 && frozen) {
#pragma unroll
      for (int g = 0; g < G; ++g) dg[g] = 0.f;
      dhn = 0.f;
      direct = dh;
    }
    if (valid) {
#pragma unroll
      for (int g = 0; g < G; ++g) bsum[g] += dg[g];
      if constexpr (NP > G) bsum[G] += dhn;
      float* gp = dgates + ((size_t)t * B + row) * GH + j;
#pragma unroll
      for (int g = 0; g < G; ++g) gp[g * H] = dg[g];
      if (MODE == B200RNN_GRU) dghn[((size_t)t * B + row) * H + j] = dhn;
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
    if (want_dh0) dh_0[((size_t)dir * B + row) * H + j] = dh_carry;
    if (MODE == B200RNN_LSTM && dc_0) dc_0[((size_t)dir * B + row) * H + j] = dc_carry;
    if (VL)  // the steps [T, p.T) the cluster skipped: their gate gradients are 0
      for (int t = T; t < p.T; ++t) {
        float* gp = dgates + ((size_t)t * B + row) * GH + j;
#pragma unroll
        for (int g = 0; g < G; ++g) gp[g * H] = 0.f;
        if (MODE == B200RNN_GRU) dghn[((size_t)t * B + row) * H + j] = 0.f;
      }
  }
  // per-slice bias-gradient partials [nslices][NP * H] (api.cu reduces them): the slice's batch slots summed in slot
  // order
  if (s.active) {
#pragma unroll
    for (int g = 0; g < NP; ++g) red[((size_t)b * NP + g) * HS + u] = bsum[g];
  }
  __syncthreads();
  if (s.active && b == 0) {
    for (int g = 0; g < NP; ++g) {
      float v = 0.f;
      for (int q = 0; q < BS; ++q) v += red[((size_t)q * NP + g) * HS + u];
      float* out = p.dbias_part[dir] + m * mdl.scr + (size_t)s.slice * NP * H;
      out[g * H + j] = v;
    }
  }
  ptx::cluster_sync_all();
}

// The BPTT over the 16-bit transposed weight_hh (whh_prep16_kernel's output), anyh16_bwd_kernel: as anyh_bwd_kernel,
// whose text is kept for the fp32 instantiations
template <int MODE, bool VL, bool ONCHIP, typename WT>
__device__ __forceinline__ void anyh_bwd_body(const RecBwdParams& p, const int nslices) {
  constexpr int G = gates_of(MODE);
  constexpr int NP = G == 1 ? 1 : G + 1;  // bias-partial blocks per slice: dGi (+ the GRU dghn block, 0 for the LSTM)
  const int H = p.H, B = p.B, LD = H + 8, GH = G * H;
  const bool relu = p.mode == B200RNN_RNN_RELU;  // Elman
  const AnyhSlice s = anyh_slice<VL>(p, nslices);
  const int C = s.C, HS = s.HS, BS = s.BS, NT = s.NT, dir = s.dir, b0 = s.b0, j0 = s.j0, n = s.n, T = s.T;
  const uint32_t rank = s.rank;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  WT* W_s = reinterpret_cast<WT*>(smem_raw);  // [G][n][LD]
  float* d_s = reinterpret_cast<float*>(W_s + (ONCHIP ? (size_t)G * HS * LD : 0));
  float* red = d_s + (size_t)2 * BS * GH;
  uint64_t* bars = reinterpret_cast<uint64_t*>(red + (size_t)BS * NP * HS);
  const int tid = threadIdx.x;
  // rows (g, u) of this CTA: W_hh[g*H + :][j0 + u], contiguous from G * j0 * H (whh_prep_kernel)
  const WT* w_prep = reinterpret_cast<const WT*>(p.w_prep[dir]) + (size_t)G * j0 * H;

  if (tid == 0) init_bars(bars, C);
  if constexpr (ONCHIP) stage_rows16(W_s, w_prep, G * n, H, NT, [&](int r) { return (size_t)r * H; });
  __syncthreads();
  ptx::cluster_sync_all();

  const int u = s.u, b = s.b, j = j0 + u, slot = b0 + b;
  const bool valid = s.active && slot < B;
  const int row = valid ? (VL ? p.order[slot] : slot) : 0;
  const int len = (VL && valid) ? p.lengths[row] : T;
  const float* gates = p.gates[dir];
  const float* extra = p.extra[dir];
  float* dgates = p.dgates[dir];
  const WT* wrow = ONCHIP ? W_s + (size_t)u * LD : w_prep + (size_t)u * H;
  const size_t wg = ONCHIP ? (size_t)n * LD : (size_t)n * H;

  float dh_carry = 0.f, dc_carry = 0.f, direct = 0.f;
  if (valid) {
    if (p.dh_n) dh_carry = p.dh_n[((size_t)dir * B + row) * H + j];
    if (MODE == B200RNN_LSTM && p.dc_n) dc_carry = p.dc_n[((size_t)dir * B + row) * H + j];
  }
  float bsum[NP] = {};
  // saved gates (Elman: h_t), hn / c_t, h_{prev} / c_{prev}, dy (prefetched)
  float sv[G] = {}, sx = 0.f, hp = 0.f, dyv = 0.f;
  const float* s0 = MODE == B200RNN_GRU ? p.h_0 : p.c_0;  // the state before the first step (zeros when NULL)
  auto load_step = [&](int step) {
    const int t = dir ? step : (T - 1 - step);
    const int tp = dir ? t + 1 : t - 1;
    // GRU, VL: the output at tp >= len is the masked 0, not the kept state; the LSTM reads the kept c from `extra`
    const bool has_prev = step < T - 1 && !(MODE == B200RNN_GRU && VL && tp >= len);
#pragma unroll
    for (int g = 0; g < G; ++g) sv[g] = gates[((size_t)t * B + row) * GH + g * H + j];
    if constexpr (G > 1) sx = extra[((size_t)t * B + row) * H + j];
    dyv = p.dy[(long long)t * p.dy_st + (long long)row * p.dy_sb + dir * H + j];
    if constexpr (G > 1) {
      if (!has_prev)
        hp = s0 ? s0[((size_t)dir * B + row) * H + j] : 0.f;
      else if (MODE == B200RNN_GRU)
        hp = p.y[(long long)tp * p.y_st + (long long)row * p.y_sb + dir * H + j];
      else
        hp = extra[((size_t)tp * B + row) * H + j];
    }
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
      dot_rows16<G, ONCHIP, (G > 1), WT>(wrow, wg, d_s + ((size_t)cur * BS + b) * GH, H, H, acc);
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
    } else if constexpr (MODE == B200RNN_LSTM) {
      const float dc_next = lstm_cell_bwd(sv, sx, hp, dh, dc_carry, dg);
      direct = 0.f;
      if (!frozen) dc_carry = dc_next;  // frozen: dh and dc pass straight through
    } else {  // Elman: dpre from the saved h_t; frozen as below
      dg[0] = frozen ? 0.f : elman_cell_bwd(sv[0], dh, relu);
      direct = frozen ? dh : 0.f;
    }
    if (G > 1 && frozen) {
#pragma unroll
      for (int g = 0; g < G; ++g) dg[g] = 0.f;
      dhn = 0.f;
      direct = dh;
    }
    if (valid) {
#pragma unroll
      for (int g = 0; g < G; ++g) bsum[g] += dg[g];
      if constexpr (NP > G) bsum[G] += dhn;
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
  // per-slice bias-gradient partials [nslices][NP * H] (api.cu reduces them): the slice's batch slots summed in slot
  // order
  if (s.active) {
#pragma unroll
    for (int g = 0; g < NP; ++g) red[((size_t)b * NP + g) * HS + u] = bsum[g];
  }
  __syncthreads();
  if (s.active && b == 0) {
    for (int g = 0; g < NP; ++g) {
      float v = 0.f;
      for (int q = 0; q < BS; ++q) v += red[((size_t)q * NP + g) * HS + u];
      float* out = p.dbias_part[dir] + (size_t)s.slice * NP * H;
      out[g * H + j] = v;
    }
  }
  ptx::cluster_sync_all();
}


// 16-bit transposed weight_hh: half the shared memory per weight row, as in the forward
template <int MODE, bool VL, bool ONCHIP, typename WT>
__global__ void __launch_bounds__(ANYH_MAX_NT, 1) anyh16_bwd_kernel(const RecBwdParams p, const int nslices, const RecModels) {
  anyh_bwd_body<MODE, VL, ONCHIP, WT>(p, nslices);
}

// =================================================================================================
// tangent (forward-mode AD)
// =================================================================================================
// The linearised forward: the same slice, staged W_hh rows, contraction and exchange as anyh_fwd_kernel, applied to the
// tangent state h'_{t-1}; the cell is the linearised cell of rnn_cell.cuh at the primal's saved activations. Step t:
// a = pre_t + b' + W_hh h'_{t-1} (GRU n block: pre_t is the x side, preh_t + b_hn' + W_hn h'_{t-1} the h side).
// Cluster m / (D * nslices) is tangent direction m (mdl.M of them); the primal tensors are shared by all.
// Shared memory: [W_s: G*n x (H+4), ONCHIP only] [h': 2 x BS x H] [bars: 2 x C]
template <int MODE, bool ONCHIP>
__global__ void __launch_bounds__(ANYH_MAX_NT, 1) anyh_tangent_kernel(const RecTanParams p, const int nslices, const RecModels mdl) {
  constexpr int G = gates_of(MODE);
  const int H = p.H, B = p.B, LD = H + 4, GH = G * H;
  const bool relu = p.mode == B200RNN_RNN_RELU;  // Elman
  const AnyhSlice s = anyh_slice<false>(p, nslices);
  const int C = s.C, HS = s.HS, BS = s.BS, NT = s.NT, dir = s.dir, b0 = s.b0, j0 = s.j0, n = s.n, T = s.T;
  const uint32_t rank = s.rank;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* W_s = reinterpret_cast<float*>(smem_raw);  // [G][n][LD]
  float* h_s = W_s + (ONCHIP ? (size_t)G * HS * LD : 0);
  uint64_t* bars = reinterpret_cast<uint64_t*>(h_s + (size_t)2 * BS * H);
  const int tid = threadIdx.x;
  // the tangent direction of this cluster, and the offset of its block of a tangent tensor. The L2 tier, which has no
  // register to spare in its step loop, forms the pointers from the launch registers at each use
  const long long m = mdl.M > 1 ? anyh_model(p, nslices) : 0;
  auto tan_ptr = [&](const float* base, long long stride) -> const float* {
    if (!base) return nullptr;
    if constexpr (ONCHIP) return base + m * stride;
    return base + (mdl.M > 1 ? (long long)anyh_model(p, nslices) : 0ll) * stride;
  };
  const float* w_hh = p.w_hh[dir];
  const float* h0_dot = p.h0_dot ? p.h0_dot + m * p.m_state : nullptr;
  const float* c0_dot = p.c0_dot ? p.c0_dot + m * p.m_state : nullptr;

  if (tid == 0) init_bars(bars, C);
  if constexpr (ONCHIP) {
    if constexpr (G == 1)
      stage_rows(W_s, w_hh, n, H, NT, [&](int r) { return (size_t)(j0 + r) * H; });
    else
      stage_rows(W_s, w_hh, G * n, H, NT, [&](int r) { return ((size_t)(r / n) * H + j0 + r % n) * H; });
  }
  for (int i = tid; i < BS * H; i += NT) {  // buffer 0: h'_0 of the cluster's slots (zeros past the batch / without it)
    const int q = i / H, k = i - q * H;
    const int slot = b0 + q;
    h_s[i] = (h0_dot && slot < B) ? h0_dot[((size_t)dir * B + slot) * H + k] : 0.f;
  }
  __syncthreads();
  ptx::cluster_sync_all();  // peers' barriers are initialised before anyone sends

  const int u = s.u, b = s.b, j = j0 + u, row = b0 + b;
  const bool valid = s.active && row < B;
  const size_t st0 = ((size_t)dir * B + row) * H + j;  // this thread's element of a [D,B,H] state
  float hd = (h0_dot && valid) ? h0_dot[st0] : 0.f;
  float cd = (MODE == B200RNN_LSTM && c0_dot && valid) ? c0_dot[st0] : 0.f;
  // the primal state before the step: GRU h_{t-1}, LSTM c_{t-1}
  const float* s0 = MODE == B200RNN_GRU ? p.h_0 : p.c_0;
  float sp = (G > 1 && s0 && valid) ? s0[st0] : 0.f;
  const size_t wg = ONCHIP ? (size_t)n * LD : (size_t)H * H;
  const float* wrow = ONCHIP ? W_s + (size_t)u * LD : w_hh + (size_t)(j0 + u) * H;

  for (int step = 0; step < T; ++step) {
    const int t = dir ? T - 1 - step : step;
    const int cur = step & 1, nxt = cur ^ 1;
    // this step's saved activations and tangent pre-activations: loaded before the exchange wait, but in the
    // L2 tier, which has no register to keep them through the contraction
    float sv[G], sx = 0.f, a[G], ah = 0.f;
    auto load_step = [&]() {
      const size_t tb = (size_t)t * B + row;
      const float* gates = p.gates[dir];
      const float* pre = tan_ptr(p.pre[dir], p.m_pre);
      const float* bih = tan_ptr(p.bih_dot[dir], p.m_bdot);
      const float* bhh = tan_ptr(p.bhh_dot[dir], p.m_bdot);
#pragma unroll
      for (int g = 0; g < G; ++g) {
        sv[g] = valid ? gates[tb * GH + g * H + j] : 0.f;
        a[g] = (valid && pre) ? pre[tb * GH + g * H + j] : 0.f;
        // the bias tangents, folded as the forward folds the biases (GRU: b_hn' on the h side); re-read every step
        // from L1 rather than held in registers through the contraction
        if (bih) a[g] += bih[g * H + j];
        if (bhh && !(MODE == B200RNN_GRU && g == 2)) a[g] += bhh[g * H + j];
      }
      if constexpr (G > 1) sx = valid ? p.extra[dir][tb * H + j] : 0.f;
      const float* preh = MODE == B200RNN_GRU ? tan_ptr(p.preh[dir], p.m_preh) : nullptr;
      if (valid && preh) ah = preh[tb * H + j];
      if (MODE == B200RNN_GRU && bhh) ah += bhh[2 * H + j];
    };
    constexpr bool LATE = !ONCHIP;
    if constexpr (!LATE) load_step();
    if (step > 0) wait_bars(bars, cur, C, rank, ((step - 1) >> 1) & 1);
    if (tid == 0 && step + 1 < T) arm_bars(bars, nxt, s, H, 1);
    float acc[G];
#pragma unroll
    for (int g = 0; g < G; ++g) acc[g] = 0.f;
    dot_rows<G, ONCHIP, false>(wrow, wg, h_s + ((size_t)cur * BS + b) * H, 0, H, acc);
    if constexpr (LATE) load_step();

    float hdn;
    if constexpr (MODE == B200RNN_GRU) {
      const float ar[3] = {a[0] + acc[0], a[1] + acc[1], a[2]};
      hdn = gru_cell_jvp(sv, sx, sp, ar, ah + acc[2], hd);
      sp = valid ? p.y[(long long)t * p.y_st + (long long)row * p.y_sb + dir * H + j] : 0.f;  // h_t
    } else if constexpr (MODE == B200RNN_LSTM) {
      const float ar[4] = {a[0] + acc[0], a[1] + acc[1], a[2] + acc[2], a[3] + acc[3]};
      hdn = lstm_cell_jvp(sv, sx, sp, ar, cd);
      sp = sx;  // c_t
    } else {
      hdn = elman_cell_jvp(sv[0], a[0] + acc[0], relu);
    }
    hd = hdn;
    if (valid) const_cast<float*>(tan_ptr(p.ydot, p.m_ydot))[(long long)t * p.yd_st + (long long)row * p.yd_sb + dir * H + j] = hdn;
    if (step + 1 < T) {
      float* h_nxt = h_s + (size_t)nxt * BS * H;
      if (s.active) h_nxt[(size_t)b * H + j] = valid ? hdn : 0.f;
      __syncthreads();  // the own slice is complete (and every thread is past step - 1's reads of buffer nxt)
      send_slice(h_nxt, H, 1, H, s, &bars[nxt * C + rank]);
    }
  }
  if (valid) {
    p.hn_dot[m * p.m_state + st0] = hd;
    if (MODE == B200RNN_LSTM && p.cn_dot) p.cn_dot[m * p.m_state + st0] = cd;
  }
  ptx::cluster_sync_all();  // nobody exits while a peer could still address its shared memory
}

// =================================================================================================
// config choice
// =================================================================================================
}  // namespace

// the Elman backward uses BS x HS floats fewer than this; each staged weight row is padded by 16 bytes
size_t anyh_smem(int G, int H, int C, int BS, bool bwd, bool onchip, int wbytes) {
  const size_t HS = (size_t)anyh_max_units(H, C);
  const size_t w = onchip ? (size_t)G * HS * (H + 16 / wbytes) * wbytes : 0;
  size_t f = (size_t)2 * BS * (bwd ? G * H : H);
  if (bwd) f += (size_t)BS * (G + 1) * HS;
  return w + f * sizeof(float) + (size_t)2 * C * sizeof(uint64_t);
}

namespace {

template <typename P>
using AnyhKernel = void (*)(P, int, RecModels);

template <int MODE, typename WT>
AnyhKernel<RecFwdParams> anyh16_kernel(const RecFwdParams&, bool vl, bool onchip) {
  return vl ? (onchip ? anyh16_fwd_kernel<MODE, true, true, WT> : anyh16_fwd_kernel<MODE, true, false, WT>)
            : (onchip ? anyh16_fwd_kernel<MODE, false, true, WT> : anyh16_fwd_kernel<MODE, false, false, WT>);
}
template <int MODE, typename WT>
AnyhKernel<RecBwdParams> anyh16_kernel(const RecBwdParams&, bool vl, bool onchip) {
  return vl ? (onchip ? anyh16_bwd_kernel<MODE, true, true, WT> : anyh16_bwd_kernel<MODE, true, false, WT>)
            : (onchip ? anyh16_bwd_kernel<MODE, false, true, WT> : anyh16_bwd_kernel<MODE, false, false, WT>);
}
template <int MODE>
AnyhKernel<RecBwdParams> anyh_kernel(const RecBwdParams&, bool vl, bool onchip) {
  return vl ? (onchip ? anyh_bwd_kernel<MODE, true, true> : anyh_bwd_kernel<MODE, true, false>)
            : (onchip ? anyh_bwd_kernel<MODE, false, true> : anyh_bwd_kernel<MODE, false, false>);
}
template <int MODE>
AnyhKernel<RecFwdParams> anyh_kernel(const RecFwdParams&, bool vl, bool onchip) {
  return vl ? (onchip ? anyh_fwd_kernel<MODE, true, true> : anyh_fwd_kernel<MODE, true, false>)
            : (onchip ? anyh_fwd_kernel<MODE, false, true> : anyh_fwd_kernel<MODE, false, false>);
}
// the tangent recurrence: fp32 weight_hh and full-length rows only
template <int MODE, typename WT>
AnyhKernel<RecTanParams> anyh16_kernel(const RecTanParams&, bool, bool) {
  return nullptr;
}
template <int MODE>
AnyhKernel<RecTanParams> anyh_kernel(const RecTanParams&, bool, bool onchip) {
  return onchip ? anyh_tangent_kernel<MODE, true> : anyh_tangent_kernel<MODE, false>;
}
// w16: the storage of weight_hh, DT_F32 or DT_F16 / DT_BF16 (h16.cuh)
template <int MODE, typename P>
AnyhKernel<P> anyh_kernel_w(const P& p, bool vl, bool onchip, int w16) {
  if (w16 == DT_F16) return anyh16_kernel<MODE, __half>(p, vl, onchip);
  if (w16 == DT_BF16) return anyh16_kernel<MODE, __nv_bfloat16>(p, vl, onchip);
  return anyh_kernel<MODE>(p, vl, onchip);
}

// The cluster shape of one launch. Candidates: C in {2, 4, 8, 16} with at least one group of 8 units per CTA
// (anyh_units: every multiple of 16 from 16 to 1024 has one), BS in {2, 4, ..., 64}, NT = HS * BS rounded up to whole
// warps (HS: the widest CTA's units), at most 512 threads. The weights stay on chip when any candidate's
// slice and buffers fit MAX_SMEM; only when none does is the L2 tier taken.
//   * On chip, a step costs each SM its G*H*HS*BS FMAs: the shape with the fewest waves x max(NT, 128) wins (a CTA of up
//     to 4 warps has one warp per scheduler, so a smaller one shortens no step), ties to the fewest CTAs.
//   * In the L2 tier a step costs each CTA its G*HS*H weights streamed from L2, whatever BS (a warp's batch slots share
//     every load): the widest cluster, then the fewest waves, then the fewest batch rows.
// Capacities come from the driver (cluster_capacity), never from the SM count; clusters that do not fit run in waves.
template <typename P>
int plan_anyh(const P& p, bool bwd, ClusterLaunch<P>* L, int w16, int models) {
  const int wbytes = w16 ? 2 : 4;
  const int G = gates_of(p.mode), H = p.H;
  const bool vl = p.lengths != nullptr;
  for (int tier = 0; tier < 2; ++tier) {
    const bool onchip = tier == 0;
    // one Elman instantiation for both nonlinearities
    const AnyhKernel<P> kernel = p.mode == B200RNN_GRU    ? anyh_kernel_w<B200RNN_GRU>(p, vl, onchip, w16)
                                 : p.mode == B200RNN_LSTM ? anyh_kernel_w<B200RNN_LSTM>(p, vl, onchip, w16)
                                                          : anyh_kernel_w<B200RNN_RNN_TANH>(p, vl, onchip, w16);
    bool found = false;
    long long best[3] = {0, 0, 0};
    ClusterLaunch<P> pick{};
    for (int C = 2; C <= 16; C *= 2) {
      if (C > H / 8) continue;
      const int HS = anyh_max_units(H, C);
      for (int BS = 2; BS <= 64; BS *= 2) {
        const int NT = (HS * BS + 31) / 32 * 32;
        if (NT > ANYH_MAX_NT) continue;
        const size_t smem = anyh_smem(G, H, C, BS, bwd, onchip, wbytes);
        if (smem > (size_t)MAX_SMEM) continue;
        // the shape is chosen as for one model, so that each model computes what it computes alone (the bias
        // gradient's slice sums included); several models add clusters, in waves when they do not all fit
        const int nslices = (p.B + BS - 1) / BS, nclusters = nslices * p.D;
        int capacity = 0;
        const int rc = cluster_capacity((const void*)kernel, C, NT, smem, &capacity);
        if (rc != B200RNN_OK) return rc;
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
          pick = ClusterLaunch<P>{(const void*)kernel, C, NT, nslices, nclusters * models, capacity, smem};
          pick.anyh = true;
          pick.BS = BS;
          pick.onchip = onchip;
          pick.models.M = models;
        }
      }
    }
    if (found) {
      static const bool debug = getenv("B200RNN_DEBUG") != nullptr;
      if (debug)
        fprintf(stderr, "[b200rnn] %s %s cfg %s VL=%d H=%d C=%d BS=%d tier=%s%s: need %d clusters, capacity %d, smem %zu\n",
                __is_same(P, RecTanParams) ? "tan" : bwd ? "bwd" : "fwd", G == 1 ? "elman" : "anyh", mode_name(p.mode), (int)vl, H, pick.C, pick.BS,
                onchip ? "smem" : "l2", wbytes == 2 ? " w_hh=16bit" : "", pick.nclusters, pick.capacity,
                pick.smem);
      *L = pick;
      return B200RNN_OK;
    }
  }
  set_error("recurrence: no cluster shape runs hidden_size %d on this device", H);
  return B200RNN_ERR_UNSUPPORTED;
}

}  // namespace

bool anyh_hidden_size(int H) { return H >= 16 && H <= 1024 && H % 16 == 0; }

int plan_anyh_fwd(const RecFwdParams& p, RecFwdLaunch* L, int w16, int models) {
  if (p.y_pool || p.ready || p.shell_nograd || p.P > 0) {
    set_error("recurrence: hidden_size %d runs without the model-shell fusions (y_pool, streamed x-projection, "
              "no-grad fused forward) and without proj_size", p.H);
    return B200RNN_ERR_UNSUPPORTED;
  }
  return plan_anyh(p, false, L, w16, models);
}

int plan_anyh_tangent(const RecTanParams& p, RecTanLaunch* L, int directions) {
  if (p.lengths) {
    set_error("tangent recurrence: ragged batches (lengths) are not supported");
    return B200RNN_ERR_UNSUPPORTED;
  }
  return plan_anyh(p, false, L, 0, directions);
}

int plan_anyh_bwd(const RecBwdParams& p, RecBwdLaunch* L, int w16, int models) {
  if (!p.dy || p.P > 0) {
    set_error("recurrence backward: hidden_size %d takes the full output gradient dy and no proj_size", p.H);
    return B200RNN_ERR_UNSUPPORTED;
  }
  return plan_anyh(p, true, L, w16, models);
}

}  // namespace b200rnn
