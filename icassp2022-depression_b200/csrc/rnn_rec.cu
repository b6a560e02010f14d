// rnn_rec.cu — persistent recurrence kernels for sm_90a (K2/K3 forward, K4/K5 backward).
//
// Replaces the T-serial inner loop the reference reaches through torch.nn.GRU / torch.nn.LSTM
// (GRU cell equations torch/nn/modules/rnn.py:1221-1224, LSTM cell :842-847; call sites
// audio_gru_whole.py:105, text_bilstm_whole.py:105, fuse_net_whole.py:347,361).
//
// Design (one launch = every time step of every direction of one layer):
//   * grid = D * nslices thread-block clusters of C CTAs. A cluster owns BS batch rows; CTA `rank` of the
//     cluster owns HS = H/C hidden units and keeps the matching rows of W_hh (forward) or columns of W_hh
//     (backward) on chip for the whole sequence: G-RG gate blocks in shared memory, staged once with TMA bulk
//     copies (cp.async.bulk ... mbarrier::complete_tx), and RG gate blocks in registers.
//   * per step every warp contracts its rows against the BS state vectors (rnn_core.cuh: K across lanes,
//     transposing shuffle butterfly); the lane that ends up owning (unit, batch) applies the gate
//     non-linearities and the state update in registers.
//   * the new state slice is all-gathered into the C peer CTAs with st.async (16-byte DSMEM stores that complete
//     transaction bytes on an mbarrier in the destination CTA): data and "ready" signal travel together, the
//     consumer waits on a local mbarrier, double buffered. No cluster barrier, fence or L1 flush in the loop.
//   * batch slices are independent clusters: no grid-wide synchronisation anywhere.
//   * ragged batches (the VL instantiations): the batch slots hold the rows sorted by descending length
//     (RecFwdParams::order), and a cluster runs only the steps of its longest sequence; the skipped steps' outputs and
//     gate gradients are written as zeros after the loop.
//
// fp32 FFMA for most configs: the per-step contraction is [BS x H] x [H x G*HS] with BS = 2..8 rows per CTA — far too
// skinny for wgmma tiles, and parity is judged at 1e-5 against an fp32 reference. The GRU H=256 8-row config runs it
// on the tensor cores with warp-level mma.sync (N = 8) in 3xTF32 instead (rec_fwd_tc_kernel), or on fp16 pairs split
// once per launch in the no-grad forward of b200rnn_forward_fused (rec_fwd_h16_kernel); in that forward the LSTM H=128
// layers take the same body on 2-CTA clusters of 8 rows (lstm_fwd_h16_kernel).
#include <map>
#include <mutex>
#include <set>
#include <stdlib.h>
#include <tuple>
#include <type_traits>
#include <utility>

#include <cuda_fp16.h>

#include "profile.cuh"
#include "ptx.cuh"
#include "rec_h16_layout.cuh"
#include "rnn_cell.cuh"
#include "rnn_core.cuh"
#include "rnn_kernels.cuh"

namespace b200rnn {

namespace {

// The CTA's own state slice is delivered locally (st.shared + mbarrier.arrive per warp). -DB200RNN_SELF_VIA_CLUSTER
// builds the round-1 behaviour (own slice through st.async like the peers') for the FFMA kernels rec_fwd_kernel and
// rec_bwd_kernel only: compute-sanitizer's racecheck does not model the ordering that inline-PTX mbarrier.arrive /
// try_wait give to ordinary shared-memory stores and flags every local store / LDS pair of the default build, so the
// race-free evidence of the REST of those kernels is taken on that build; the ordering argument for the local path is in
// allgather_units' comment. The tc8 kernels always deliver the own slice locally (sending it through the cluster would
// need a staging buffer), and the projected kernels never send to or wait on their own slot.
#ifdef B200RNN_SELF_VIA_CLUSTER
constexpr bool kLocalSelf = false;
#else
constexpr bool kLocalSelf = true;
#endif
constexpr unsigned FULLMASK = 0xffffffffu;

template <int MODE, int H, int C, int BS, int KL, int UPL, int RG>
struct RecCfg {
  static constexpr int G = gates_of(MODE);
  static constexpr int GH = G * H;
  static constexpr int HS = H / C;
  static constexpr int UPW = (32 / KL) * UPL;  // units per warp
  static constexpr int NW = HS / UPW;
  static constexpr int NT = NW * 32;
  static constexpr int NSM = G - RG;  // gate blocks held in shared memory
  static constexpr int CW = 4 * KL;   // floats of the contraction dimension per chunk
  static constexpr int NCH = H / CW;  // chunks per state vector (per gate block in the backward)
  static constexpr bool ROT = (CW <= HS);           // chunk order rotates so the CTA's own slice comes first
  static constexpr int CPS = ROT ? HS / CW : 1;     // chunks per source slice (ROT)
  static constexpr int SPC = ROT ? 1 : CW / HS;     // source slices per chunk (!ROT)
  static constexpr int NBAR = 1 + 2 * C;            // [0] weights, [1 + buf*C + src] state slices
  static constexpr size_t BAR_BYTES = 256;
  static constexpr size_t W_BYTES = (size_t)NSM * HS * H * sizeof(float);
  static constexpr size_t FWD_SMEM = W_BYTES + (size_t)2 * BS * H * sizeof(float) + BAR_BYTES;
  static constexpr size_t BWD_SMEM = W_BYTES + (size_t)2 * BS * GH * sizeof(float) + BAR_BYTES;
  static_assert(NBAR * 8 <= (int)BAR_BYTES, "barrier block too small");
  static_assert(ROT ? (HS % CW == 0) : (CW % HS == 0), "chunks must tile the per-CTA slices");
  static_assert(RG >= 0 && RG <= 2, "at most two register-resident gate blocks");
  static_assert(HS * C == H && NW * UPW == HS && NW >= 1, "bad split");
  static_assert(UPW % 4 == 0, "the exchange packs 4 units per 16-byte store");
  static_assert(NT <= 1024, "too many threads");
};

// VL: the steps a cluster runs, the length of its first batch slot (the longest: order sorts by descending length)
__device__ __forceinline__ int slice_steps(const int* lengths, const int* order, int b0, int T) {
  return min(max(lengths[order[b0]], 0), T);
}

// What a CTA owns: cluster blockIdx.x / C runs direction `dir` of batch slice `slice` (slots b0 .. b0 + BS - 1), and
// CTA `rank` of it the HS units from j0. T is the number of steps the cluster runs: p.T, or under VL its longest row's.
struct ClusterSlice {
  uint32_t rank;
  int dir, slice, b0, j0, T;
};

template <int C, int BS, int HS, bool VL, typename Params>
__device__ __forceinline__ ClusterSlice cluster_slice(const Params& p, int nslices) {
  ClusterSlice s;
  s.rank = ptx::cluster_ctarank();
  const int cid = blockIdx.x / C;
  s.dir = cid / nslices;
  s.slice = cid - s.dir * nslices;
  s.b0 = s.slice * BS;
  s.j0 = (int)s.rank * HS;
  s.T = VL ? slice_steps(p.lengths, p.order, s.b0, p.T) : p.T;
  return s;
}

// The [2][C] mbarriers of a double-buffered exchange between the C CTAs of a cluster: bar(buf, src) completes when the
// slice of source CTA `src` has landed in buffer `buf`. Remote sources complete transaction bytes, one expect_tx per
// exchange re-armed by thread 0 (arm). LOCAL_SELF: the own slice is delivered locally, with ordinary stores published by
// plain arrives (the own barrier's arrival count, init), and is never armed.
// Step s contracts against buffer s & 1, which holds what step s - LAG sent (LAG = 1: the forward kernels and the
// projected BPTT; LAG = 0: rec_bwd_kernel, which contracts in the step that sends). Each buffer carries every other
// exchange, so the wait of step s is for phase ((s - LAG) >> 1) & 1. Thread 0 arms a buffer for the next exchange only
// after its own waits on that buffer's previous phase have passed.
// The barriers are bars[FIRST + buf * C + src]: FIRST = 1 where bars[0] is the weight barrier of the FFMA kernels.
template <int C, int LAG, bool LOCAL_SELF, int FIRST = 0>
struct ExchangeBars {
  uint64_t* bars;
  uint32_t rank;

  static __device__ __forceinline__ int buf(int s) { return s & 1; }
  static __device__ __forceinline__ uint32_t parity(int s) { return ((s - LAG) >> 1) & 1; }
  __device__ __forceinline__ uint64_t* bar(int b, int src) const { return &bars[FIRST + b * C + src]; }

  // thread 0, before fence_mbar_init
  __device__ __forceinline__ void init(uint32_t self_arrivals) const {
    for (int i = 0; i < 2 * C; ++i)
      ptx::mbar_init(&bars[FIRST + i], (LOCAL_SELF && (uint32_t)(i % C) == rank) ? self_arrivals : 1u);
  }
  // thread 0: buffer b expects `bytes` from every source that sends through the cluster
  __device__ __forceinline__ void arm(int b, uint32_t bytes) const {
#pragma unroll
    for (int src = 0; src < C; ++src)
      if (!LOCAL_SELF || (uint32_t)src != rank) ptx::mbar_arrive_expect_tx(bar(b, src), bytes);
  }
  // the slice of source `src` has landed in buffer b = buf(s), phase par = parity(s) (computed once per step)
  __device__ __forceinline__ void wait(int b, int src, uint32_t par) const { ptx::mbar_wait(bar(b, src), par); }
};

// All-gather `val` (owned by lane (unit, batch) of every warp) into vec[b][col0 + unit] of all C CTAs:
// 4 shuffles gather 4 consecutive units, one 16-byte store per (destination, chunk).
// Remote destinations get st.async (data + complete_tx on the destination's per-source mbarrier). With LOCAL_SELF the
// CTA's own copy does not take the trip through the cluster network (measured: >= 600 cycles from the store to the
// barrier flip even for the own CTA, tools/trace_rec.py): it is written with ordinary st.shared and published with one
// mbarrier.arrive per warp on the own-source barrier (initialised with the warp count instead of a byte count).
// Ordering of the local path: RAW - readers pass mbarrier.try_wait (acquire) on that barrier, which completes only
// after every warp's arrive (release) that follows its st.shared + __syncwarp. WAR - a warp writes buffer b at the end
// of step s; the last readers of b ran in step s-1's contraction, and no warp can leave chunk 0 of step s before all
// NW warps have arrived for step s-1, i.e. finished that contraction.
// PAIRED: the destination uses the batch-paired layout of rnn_core.cuh (paired_index): one 16-byte store carries units
// j and j+4 for the two batch rows of a pair (j % 8 < 4; both land in adjacent k-lanes of the same chunk row).
template <int C, int KL, int UPL, int BS, bool LOCAL_SELF = false, bool PAIRED = false>
__device__ __forceinline__ void allgather_units(float val, float* vec_local, int vstride, int col0,
                                                uint64_t* bar_local, int lane, uint32_t rank = 0) {
  using LM = LaneMap<KL, UPL, BS>;
  constexpr int UPW = LM::UPW;
  constexpr int NCH = UPW * BS / 4;  // 16-byte chunks per destination
  constexpr int NST = C * NCH;
  static_assert(!PAIRED || (UPW % 8 == 0 && BS % 2 == 0), "paired layout: 8 units per store group, even batch slice");
  const uint32_t bar_addr = ptx::smem_u32(bar_local);
#pragma unroll
  for (int it = 0; it < (NST + 31) / 32; ++it) {
    const int idx = it * 32 + lane;
    const bool act = idx < NST;
    const int id2 = act ? idx : 0;
    const int r = id2 / NCH, ch = id2 % NCH;
    float4 v;
    float* dst_ptr;
    if constexpr (PAIRED) {
      const int pr = ch % (BS / 2), ue = ch / (BS / 2);   // batch pair, unit slot (group of 8 units, e = unit % 4)
      const int u = (ue / 4) * 8 + (ue % 4);
      v.x = __shfl_sync(FULLMASK, val, LM::lane_of(u, 2 * pr));
      v.y = __shfl_sync(FULLMASK, val, LM::lane_of(u, 2 * pr + 1));
      v.z = __shfl_sync(FULLMASK, val, LM::lane_of(u + 4, 2 * pr));
      v.w = __shfl_sync(FULLMASK, val, LM::lane_of(u + 4, 2 * pr + 1));
      dst_ptr = &vec_local[paired_index<KL, BS>(col0 + u, 2 * pr)];
    } else {
      const int b = ch / (UPW / 4), quad = ch % (UPW / 4);
      v.x = __shfl_sync(FULLMASK, val, LM::lane_of(quad * 4 + 0, b));
      v.y = __shfl_sync(FULLMASK, val, LM::lane_of(quad * 4 + 1, b));
      v.z = __shfl_sync(FULLMASK, val, LM::lane_of(quad * 4 + 2, b));
      v.w = __shfl_sync(FULLMASK, val, LM::lane_of(quad * 4 + 3, b));
      dst_ptr = &vec_local[b * vstride + col0 + quad * 4];
    }
    if (act) {
      if (LOCAL_SELF && (uint32_t)r == rank) {
        *reinterpret_cast<float4*>(dst_ptr) = v;
      } else {
        const uint32_t dst = ptx::smem_u32(dst_ptr);
        ptx::st_async_v4(ptx::mapa(dst, (uint32_t)r), v, ptx::mapa(bar_addr, (uint32_t)r));
      }
    }
  }
  if (LOCAL_SELF) {
    __syncwarp();
    if (lane == 0) ptx::mbar_arrive(bar_local);
  }
}

// =================================================================================================
// forward
// =================================================================================================
// One (unit j, batch row b) output of a forward lane, everything it does outside the contraction: the x-projection
// prefetched one step ahead, the gate math and state update, the step's global stores, and the final h_n / c_n / y_pool
// stores. VL: past its length a sequence keeps its state and emits 0 (PackedSequence semantics), and batch slot `slot`
// holds row order[slot]. A slot past the batch (!valid) computes on zeros and stores nothing.
// The stores of a step are held in registers until flush(), which the kernels call behind the next step's first chunk:
// between the exchange and the next contraction they sat on the serial path of every step (225 cycles).
// Saved for the backward, in the format rec_bwd_kernel's load_step reads: gates[t][b][g*H + j] (the x-projection on
// entry) is overwritten with the activated gate g (GRU r, z, n; LSTM i, f, g, o), and extra[t][b][j] holds
// hn = (W_hn h_{t-1})_j + b_hn (GRU) or c_t (LSTM).
template <int MODE, int H, bool VL>
struct FwdCell {
  static constexpr int G = gates_of(MODE);
  float* gates;
  float* extra;
  int j, b, len;
  bool valid;
  float bhn, h = 0.f, c = 0.f, h_sum = 0.f;
  float gi[G];                       // x-projection of the step update() computes next
  float pend_y, pend_s[G], pend_sx;  // stores of the last step update() computed

  __device__ __forceinline__ FwdCell(const RecFwdParams& p, int dir, int j_, int slot)
      : gates(p.gates[dir]), extra(p.extra[dir]), j(j_), b(slot), len(p.T), valid(slot < p.B) {
    bhn = (MODE == B200RNN_GRU) ? p.b_hh[dir][2 * H + j] : 0.f;
    if constexpr (VL) {
      if (valid) {
        b = p.order[slot];
        len = p.lengths[b];
      }
    }
#pragma unroll
    for (int g = 0; g < G; ++g) gi[g] = 0.f;
  }

  // The state starts at h_0 / c_0 (zeros when NULL); a ragged row keeps it until its first real step. Called right
  // before the step loop: a state loaded earlier stays live through the prologue and changes how ptxas schedules the
  // loop. Only the uniform pointer test branches (a per-lane branch costs the loop its warp-uniform barrier waits): a
  // slot past the batch loads the last row and discards it.
  __device__ __forceinline__ void start(const RecFwdParams& p, int dir) {
    const size_t s0 = ((size_t)dir * p.B + min(b, p.B - 1)) * H + j;
    if (p.h_0) h = valid ? p.h_0[s0] : 0.f;
    if (MODE == B200RNN_LSTM && p.c_0) c = valid ? p.c_0[s0] : 0.f;
  }

  __device__ __forceinline__ void load_gi(const RecFwdParams& p, int t) {
    if (valid) {
      const float* gp = gates + ((size_t)t * p.B + b) * (G * H) + j;
#pragma unroll
      for (int g = 0; g < G; ++g) gi[g] = gp[g * H];
    }
  }

  // step at time t from the recurrent pre-activations pre[g] = (W_hh h_{t-1})[g*H + j]; returns the new state
  __device__ __forceinline__ float update(int t, const float (&pre)[G]) {
    float hnew, s[G], sx;
    if constexpr (MODE == B200RNN_GRU) {
      const GruStep st = gru_cell_fwd(gi, pre, bhn, h);
      hnew = st.h;
      if constexpr (VL) {
        if (t >= len) hnew = h;
      }
      s[0] = st.r; s[1] = st.z; s[2] = st.n; sx = st.hn;
    } else {
      const LstmStep st = lstm_cell_fwd(gi, pre, c);
      float cnew = st.c;
      hnew = st.h;
      if constexpr (VL) {
        if (t >= len) {
          cnew = c;
          hnew = h;
        }
      }
      c = cnew;
      s[0] = st.i; s[1] = st.f; s[2] = st.g; s[3] = st.o; sx = cnew;
    }
    h = hnew;
    float yv = hnew;  // what the caller sees at this step
    if constexpr (VL) {
      if (t >= len) yv = 0.f;
    }
    h_sum += yv;
    pend_y = yv;
#pragma unroll
    for (int g = 0; g < G; ++g) pend_s[g] = s[g];
    pend_sx = sx;
    return hnew;
  }

  // the stores of the last update(), which computed time t
  __device__ __forceinline__ void flush(const RecFwdParams& p, int dir, int t) {
    if (valid) {
      if (p.y) p.y[(long long)t * p.y_st + (long long)b * p.y_sb + dir * H + j] = pend_y;
      if (p.training) {
        float* gp = gates + ((size_t)t * p.B + b) * (G * H) + j;
#pragma unroll
        for (int g = 0; g < G; ++g) gp[g * H] = pend_s[g];
        extra[((size_t)t * p.B + b) * H + j] = pend_sx;
      }
    }
  }

  // after the last step: the final state and the sum over time of the output
  __device__ __forceinline__ void finish(const RecFwdParams& p, int dir) {
    if (valid) {
      p.h_n[((size_t)dir * p.B + b) * H + j] = h;
      if (p.y_pool) p.y_pool[(size_t)b * p.D * H + dir * H + j] = h_sum;
      if (MODE == B200RNN_LSTM && p.c_n) p.c_n[((size_t)dir * p.B + b) * H + j] = c;
    }
  }

  // VL, after the cluster's Ts steps: the outputs of the steps [Ts, T) it skipped are 0, as past any sequence's length
  // (the caller and the W_hh gradient GEMM read them). A cluster of empty sequences never reached finish().
  __device__ __forceinline__ void skip_tail(const RecFwdParams& p, int dir, int Ts) {
    if (Ts == 0) finish(p, dir);
    if (valid && p.y)
      for (int t = Ts; t < p.T; ++t) p.y[(long long)t * p.y_st + (long long)b * p.y_sb + dir * H + j] = 0.f;
  }
};

// Initial value of element (unit k, batch slot q) of the shared state buffer the first step contracts against: h_0 of
// the row in slot b0 + q (zero past the batch). Every CTA fills its whole buffer from global memory, so step 0 needs no
// exchange; the caller tests p.h_0 (uniform) and zero-fills without it. Branch-free per lane, like FwdCell's load.
// This runs in the prologue, which with the streamed x-projection (RecFwdParams::ready) may overlap the GEMM before the
// kernel: h_0 is an input of the call, which that GEMM never writes, so reading it that early is safe.
template <bool VL>
__device__ __forceinline__ float initial_state(const RecFwdParams& p, int dir, int b0, int q, int k) {
  const int slot = min(b0 + q, p.B - 1);
  const int row = VL ? p.order[slot] : slot;
  const float v = p.h_0[((size_t)dir * p.B + row) * p.H + k];
  return b0 + q < p.B ? v : 0.f;
}

// Streamed x-projection (RecFwdParams::ready, api.cu): before a warp reads the x-projection of step t, it waits until
// the GEMM has published every row tile that holds rows [t*B, (t+1)*B). The whole warp polls the counter with acquire
// semantics (one broadcast load; a poll loop run by one lane alone made ptxas spill the FFMA configs' registers), and
// the loads of `gates` that follow stay ordinary loads. `upto`, the last row tile this warp has seen complete, makes a
// step whose tiles are already known complete cost one compare. Steps are visited in increasing t: only
// unidirectional layers are streamed. In the tensor-core kernels the producer lane alone polls (rec_fwd_tc_body).
// The wait always ends: the GEMM never waits on anything, and the programmatic launch starts this kernel only after
// every GEMM CTA has started. It is bounded all the same (trap after 4M polls, seconds, like the peer exchange in
// fuse_head.cu), so that a protocol bug is a CUDA error, not a hung GPU.
struct GiReady {
  int upto = -1;
  __device__ __forceinline__ void wait(const RecFwdParams& p, int t) {
    if (p.ready == nullptr) return;
    const int last = ((t + 1) * p.B - 1) / TC_TILE_M;
    if (last <= upto) return;
    for (int m = max(upto + 1, t * p.B / TC_TILE_M); m <= last; ++m)
      for (int n = 0; ptx::ld_acquire_gpu(p.ready + m) < p.tiles_n; ++n)
        if (n > (1 << 22)) __trap();
    upto = last;
  }
};

// PB = true: batch-paired contraction and state layout (rnn_core.cuh, dots_chunk2b), see plan_rec_fwd
template <int MODE, int H, int C, int BS, int KL, int UPL, int RG, bool VL = false, bool PB = false>
__global__ void __launch_bounds__(RecCfg<MODE, H, C, BS, KL, UPL, RG>::NT, 1)
    rec_fwd_kernel(const RecFwdParams p, const int nslices) {
  using Cfg = RecCfg<MODE, H, C, BS, KL, UPL, RG>;
  using LM = LaneMap<KL, UPL, BS>;
  constexpr int G = Cfg::G, HS = Cfg::HS, NT = Cfg::NT, UPW = Cfg::UPW, NSM = Cfg::NSM;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* W_s = reinterpret_cast<float*>(smem_raw);                 // [NSM*HS][H]
  float* h_s = W_s + (size_t)NSM * HS * H;                         // [2][BS][H]
  uint64_t* bars = reinterpret_cast<uint64_t*>(h_s + 2 * BS * H);  // [0] weights, [1 + buf*C + src] state slices
  constexpr int NCH = Cfg::NCH, CPS = Cfg::CPS;

  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const ClusterSlice cs = cluster_slice<C, BS, HS, VL>(p, nslices);
  const uint32_t rank = cs.rank;
  const int dir = cs.dir, b0 = cs.b0, j0 = cs.j0, T = cs.T;
  const float* w_hh = p.w_hh[dir];
  // step s contracts against the state step s - 1 sent; step 0 against the initial state in buffer 0
  const ExchangeBars<C, 1, kLocalSelf, 1> xb{bars, rank};

  if (tid == 0) {
    ptx::mbar_init(&bars[0], 1u);  // weights (tx bytes)
    xb.init((uint32_t)Cfg::NW);    // the own slice: one arrive per warp
    ptx::fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    // this CTA's rows of the first NSM gate blocks of W_hh: NSM contiguous [HS,H] blocks, one TMA bulk copy each
    ptx::mbar_arrive_expect_tx(&bars[0], (uint32_t)Cfg::W_BYTES);
#pragma unroll
    for (int g = 0; g < NSM; ++g)
      ptx::tma_bulk_g2s(W_s + (size_t)g * HS * H, w_hh + ((size_t)g * H + j0) * H,
                        (uint32_t)(HS * H * sizeof(float)), &bars[0]);
  }
  if (p.h_0) {  // buffer 0: the initial state of the cluster's batch slots, in the layout the all-gather writes
    for (int i = tid; i < BS * H; i += NT) {
      const int q = i / H, k = i - q * H;
      h_s[PB ? paired_index<KL, BS>(k, q) : i] = initial_state<VL>(p, dir, b0, q, k);
      h_s[BS * H + i] = 0.f;
    }
  } else {
    for (int i = tid; i < 2 * BS * H; i += NT) h_s[i] = 0.f;  // h_0 = 0 (rnn.py:1432-1440)
  }
  const int rot = Cfg::ROT ? (int)rank * CPS : 0;
  float wreg[RG > 0 ? RG : 1][UPL][H / KL];
  load_resident<RG, KL, UPL, BS, H>(w_hh, H, (long long)NSM * H + j0 + w * UPW, rot, lane, wreg);
  ptx::mbar_wait(&bars[0], 0);
  __syncthreads();
  ptx::cluster_sync_all();  // peers' barriers and state buffers are initialised before anyone writes into them

  // ---- lane identity: after the butterfly this lane owns (unit, batch) ------------------------------
  FwdCell<MODE, H, VL> cell(p, dir, j0 + w * UPW + LM::unit(lane), b0 + LM::q(lane));
  GiReady gi_ready;
  if (T > 0) {
    gi_ready.wait(p, dir ? T - 1 : 0);
    cell.load_gi(p, dir ? T - 1 : 0);
  }
  cell.start(p, dir);

  for (int step = 0; step < T; ++step) {
    const int t = dir ? (T - 1 - step) : step;
    const int cur = xb.buf(step), nxt = cur ^ 1;
    const float* h_cur = h_s + cur * BS * H;
    float* h_nxt = h_s + nxt * BS * H;
    const uint32_t par = xb.parity(step);
#ifdef B200RNN_TRACE
    const bool tr = p.trace != nullptr && blockIdx.x == 0 && lane == 0;  // one row of 8 stamps per (step, warp)
#else
    constexpr bool tr = false;  // build with -DB200RNN_TRACE for the per-phase clock64 timeline (tools/trace_rec.py)
#endif
    long long* trow = p.trace + ((size_t)step * 8 + (w & 7)) * 8;
    if (tr) trow[0] = clock64();

    // float2 accumulators for the GRU only: k-paired (PACK2: float2 = even-k / odd-k partial sums of one output,
    // folded before the butterfly) or batch-paired (PACKB: float2 = two batch rows of one unit, one weight for both,
    // state kept in the paired shared-memory layout); the LSTM keeps scalar accumulators
    constexpr bool PACKB = PB;
    constexpr bool PACK2 = !PACKB && (MODE == B200RNN_GRU) && RG < 2;
    float2 acc2[PACK2 ? G : 1][UPL][BS];
    float2 acc2b[PACKB ? G : 1][UPL][BS / 2];
    float acc[G][UPL][BS];
#pragma unroll
    for (int g = 0; g < G; ++g)
#pragma unroll
      for (int au = 0; au < UPL; ++au)
#pragma unroll
        for (int ab = 0; ab < BS; ++ab) {
          acc[g][au][ab] = 0.f;
          if (PACK2) acc2[g][au][ab] = make_float2(0.f, 0.f);
          if (PACKB && ab < BS / 2) acc2b[g][au][ab] = make_float2(0.f, 0.f);
        }
    // contraction over h, one chunk at a time, starting with the slice this CTA produced itself; a chunk is
    // touched only after the slice(s) it belongs to have arrived (per-source mbarriers)
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const int ca = (c + rot) % NCH;
      if (step > 0) {
        if (Cfg::ROT) {
          if (c % CPS == 0) xb.wait(cur, ca / CPS, par);
        } else {
#pragma unroll
          for (int s2 = 0; s2 < Cfg::SPC; ++s2) xb.wait(cur, ca * Cfg::SPC + s2, par);
        }
      }
      if (tr && c < 4) trow[1 + c] = clock64();     // slice of chunk c has arrived (this warp passed its wait)
      if constexpr (PACKB)
        dots_chunk2b<G, RG, KL, UPL, BS, H>(W_s, HS, w * UPW, wreg, h_cur, c, ca, lane, acc2b);
      else if constexpr (PACK2)
        dots_chunk2<G, RG, KL, UPL, BS, H, H>(W_s, HS, w * UPW, wreg, h_cur, c, ca, lane, acc2);
      else
        dots_chunk<G, RG, KL, UPL, BS, H, H>(W_s, HS, w * UPW, wreg, h_cur, c, ca, lane, acc);
      if (c == 0 && step > 0) cell.flush(p, dir, dir ? (T - step) : (step - 1));  // the previous step's stores
    }
    // every slice of h_step has been consumed by this thread => the barriers of the other buffer are re-armed
    if (tid == 0 && step + 1 < T) xb.arm(nxt, (uint32_t)(BS * HS * sizeof(float)));
    if constexpr (PACKB) {
      float red[G];
      warp_transpose_reduce2b<G, KL, UPL, BS>(acc2b, red, lane);
#pragma unroll
      for (int g = 0; g < G; ++g) acc[g][0][0] = red[g];
    } else {
      if constexpr (PACK2) fold_pairs<G, UPL, BS>(acc2, acc);
      warp_transpose_reduce<G, KL, UPL, BS>(acc);
    }
    if (tr) trow[5] = clock64() + (long long)(acc[0][0][0] == 12345.678f);  // butterfly done (value dependence pins it)

    float pre[G];
#pragma unroll
    for (int g = 0; g < G; ++g) pre[g] = acc[g][0][0];
    const float hnew = cell.update(t, pre);
    if (tr) trow[6] = clock64() + (long long)(hnew == 12345.678f);          // gate math done

    if (step + 1 < T)
      allgather_units<C, KL, UPL, BS, kLocalSelf, PACKB>(hnew, h_nxt, H, j0 + w * UPW, xb.bar(nxt, rank), lane, rank);
    if (tr) trow[7] = clock64();                                            // exchange issued

    if (step == T - 1) {
      cell.flush(p, dir, t);
      cell.finish(p, dir);
    }
    if (step + 1 < T) {  // long latency, consumed at the next gate math
      gi_ready.wait(p, dir ? (T - 2 - step) : (step + 1));
      cell.load_gi(p, dir ? (T - 2 - step) : (step + 1));
    }
  }
  if constexpr (VL) cell.skip_tail(p, dir, T);
  ptx::cluster_sync_all();  // nobody exits while a peer could still address its shared memory
}

// =================================================================================================
// forward, GRU H = 256 on the tensor cores (config tc8)
// =================================================================================================
// The cluster design of rec_fwd_kernel at C = 4, BS = 8 (weights staged once, per-source mbarriers, double-buffered
// state, st.async all-gather with the own slice delivered locally, own slice first, deferred global stores), but the
// x-projection arrives through a shared-memory ring that a producer warp fills with bulk copies (it alone polls the
// streamed GEMM's counters, off the compute warps' serial path), and the per-step contraction
// [192 gate rows of the CTA] x [K = 256] x [8 batch rows] runs
// on the tensor cores as mma.sync m16n8k8 in 3xTF32 (ptx.cuh split_tf32), at fp32-level error:
//   * unit group ug (16 units of the CTA's slice) has three gate tiles (r, z, n): three M = 16 tiles of W_hh rows,
//     N = the 8 batch rows, K in 32 k-steps of 8. Two warps share a unit group and split K: warp (ug, kh) takes k-steps
//     kh*4 .. kh*4+3 of every source slice, so each scheduler runs two warps and hides the other's MMA and shared-memory
//     latency (one warp per group was measured slower).
//   * the accumulator fragment leaves lane (g, t) = (lane / 4, lane % 4) units g, g+8 of the group for batch rows 2t,
//     2t+1 of all three gates. Warp kh finishes units g + 8*kh: it swaps the other half's partial sums with its partner
//     through shared memory, and the gate math stays in the lane (2 outputs each), with no butterfly.
//   * weights in A-fragment order: a lane's four values of one (tile, k-step) are one conflict-free LDS.128.
//   * state in B-fragment order (tc_state_index): a lane's two values of one k-step are one conflict-free LDS.64, and
//     the 8 units a warp finishes are one whole k-step, i.e. 64 contiguous floats: the all-gather is one float4 per lane
//     of the first half-warp.
//   * per tile, hi*hi and the two cross terms (lo*hi + hi*lo) have their own accumulators, restarted for each source
//     slice (at most 8 MMAs) and added round-to-nearest into the fp32 sum: six independent MMA chains per warp, and the
//     truncating tensor-core accumulation never runs longer than in gemm_tc.cu (12 MMAs).
// Single-pass TF32 (TF32 = true, B200RNN_FLAG_TF32; rec_fwd_tf32_kernel): W_hh is rounded to TF32 (cvt.rna) once as it
// is staged, and the lane that produces h_t rounds the copy it hands to the contraction (its own buffer and the
// st.async to the peers) while its FwdCell keeps the fp32 h for the update. The step loop then converts nothing and
// runs one mma.sync per (gate tile, k-step): 384 per CTA and step instead of 1,152, one accumulator per tile and source
// slice (4 MMAs). Round-to-nearest, not the truncation of split_tf32: without a lo term a truncated operand would bias
// every product the same way.
// The geometry is a parameter (TcCfg<MODE, L, RT, TAIL_SLOTS, SCALE_ROWS>, L = h16::Geom): the GRU-256 config TcFwdCfg
// runs all three contractions, the LSTM-128 one TcLstmCfg (2-CTA clusters of 8 batch rows, 64 units x 4 gates per CTA)
// only the fp16-pair one. RT gate tiles (the last ones) stay in registers in the fp16-pair kernels; SCALE_ROWS rows'
// loads are in flight at once in the row-scale pass of the prologue.
template <int MODE_, typename L_, int RT_, int TAIL_SLOTS, int SCALE_ROWS_>
struct TcCfg {
  using L = L_;
  static constexpr int MODE = MODE_, RT = RT_, SCALE_ROWS = SCALE_ROWS_;
  static constexpr int H = L::H, C = L::C, BS = L::BS, G = L::G, GH = G * H;
  static constexpr int HS = H / C;        // units per CTA
  static constexpr int NUG = HS / 16;     // unit groups
  static constexpr int NW = 2 * NUG;      // compute warps: (k half, unit group)
  static constexpr int NTC = NW * 32;     // compute threads
  static constexpr int NT = NTC + 128;    // and the producer warpgroup
  static constexpr int KS = H / 8;        // k-steps of the contraction
  static constexpr int KSC = HS / 8;      // k-steps per source slice
  static constexpr size_t W_BYTES = (size_t)G * HS * H * sizeof(float);
  static constexpr size_t RED_BYTES = (size_t)NW * 2 * G * 32 * sizeof(float);  // partial sums swapped between halves
  // x-projection ring behind the swap buffer: the 3xTF32 and TF32 kernels' and the LSTM-128 fp16-pair kernel's (the
  // GRU-256 fp16-pair kernel keeps its ring in dead weight space, rec_h16_layout.cuh)
  static constexpr int RING_SLOTS = TAIL_SLOTS;
  static constexpr size_t RING_BYTES = (size_t)RING_SLOTS * L::RING_SLOT_BYTES;
  static constexpr int NBAR = 2 * C + 2 * h16::RING_SLOTS;  // state [buf][src], ring full[slot], ring empty[slot]
  static constexpr size_t SMEM = W_BYTES + (size_t)2 * BS * H * sizeof(float) + RED_BYTES + RING_BYTES +
                                 NBAR * sizeof(uint64_t);
  // setmaxnreg: the producer warpgroup gives its registers to the two compute warpgroups
  static constexpr int PRODUCER_REGS = 24, COMPUTE_REGS = 240;
  static_assert(PRODUCER_REGS * 128 + COMPUTE_REGS * NTC <= 65536, "register file");
  static_assert(RING_SLOTS <= h16::RING_SLOTS, "ring barriers");
  static_assert(L::RING_IN_TILE || (h16::RING_SLOTS == RING_SLOTS && (size_t)L::ring_byte(0) == W_BYTES +
                                    (size_t)2 * BS * H * sizeof(float) + RED_BYTES), "the ring region of the layout");
  static_assert(L::NW == NW && L::RED_BYTES == (int)RED_BYTES, "h16 layout geometry");
};
using TcFwdCfg = TcCfg<B200RNN_GRU, h16::Gru256, 1, 2, 1>;
// two gate tiles in registers (64 per lane, as the GRU's one tile of four slices) compile with no spill
using TcLstmCfg = TcCfg<B200RNN_LSTM, h16::Lstm128, 2, 4, 8>;

// position of state element (k, batch row b) in the B-fragment-ordered buffer: lane (g, t) of k-step ks reads
// {h[g][ks*8 + t], h[g][ks*8 + t + 4]} as the float2 at ks*64 + lane*2
__device__ __forceinline__ int tc_state_index(int k, int b) {
  return ((k >> 3) * 8 + b) * 8 + (k & 3) * 2 + ((k >> 2) & 1);
}

__device__ __forceinline__ float round_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

// fp16 pairs (rec_fwd_h16_kernel, the no-grad forward of b200rnn_forward_fused; RecFwdParams::shell_nograd): the same
// cluster, warps, exchange and cell, with every operand an fp16 (hi, lo) pair that fills the 4 bytes of its fp32 value
// (rec_h16_layout.cuh). An fp16 significand has TF32's 11 bits, so the pair is as precise as the 3xTF32 split, but it is
// made once: W_hh as it is staged, each row scaled by 2^e_r (h16::scale_exp) so that hi is normal, and h_t by the lane
// that produces it, scaled by 2^14. The step loop splits and converts nothing: per warp and k-block of 16 it loads the
// state pair (one LDS.128) and the hi and lo A fragments of two gate tiles (four LDS.128; the third tile, n, stays in
// registers for the whole launch) and runs nine mma.sync m16n8k16 (hi*hi, lo*hi, hi*lo per tile), with the same chains
// and restarts as 3xTF32. The pre-activations are unscaled by the exact 2^-(e_r + 14) before the gate math. No initial
// state: |h_t| <= 1 is what makes the fixed state scale safe.
enum class TcOp { X3, TF32, F16 };

template <typename Cfg, bool VL, TcOp OP>
__device__ __forceinline__ void rec_fwd_tc_body(const RecFwdParams& p, const int nslices) {
  using L = typename Cfg::L;
  constexpr int H = Cfg::H, C = Cfg::C, BS = Cfg::BS, G = Cfg::G, HS = Cfg::HS, NUG = Cfg::NUG, NW = Cfg::NW,
                NT = Cfg::NT, KS = Cfg::KS, KSC = Cfg::KSC, RT = Cfg::RT;
  constexpr bool TF32 = OP == TcOp::TF32, F16 = OP == TcOp::F16;
  constexpr int KBC = L::KBC;
  static_assert(F16 || Cfg::MODE == B200RNN_GRU, "the 3xTF32 and TF32 contractions are built for the GRU");
  static_assert(RT >= 1 && RT < G, "register tiles");
  static_assert(L::H == H && L::C == C && L::BS == BS && L::G == G && L::NW == NW, "h16 layout geometry");
  static_assert(L::W_HALVES * 2 == (int)Cfg::W_BYTES && L::S_HALVES * 2 == BS * H * 4, "h16 regions");
  static_assert(G * HS <= NW * 2 * G * 32, "the row scales fit the swap buffer");
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float4* W_f = reinterpret_cast<float4*>(smem_raw);                  // [NUG][G][KS][32 lanes] A fragments
  float* h_s = reinterpret_cast<float*>(smem_raw + Cfg::W_BYTES);     // [2][BS * H] B-fragment order
  float* red = h_s + 2 * BS * H;                                       // [NW][2 * G][32 lanes]
  float* ring_tail = red + NW * 2 * G * 32;                             // X3 / TF32: [RING_SLOTS] x-projection slots
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + Cfg::SMEM - Cfg::NBAR * sizeof(uint64_t));
  uint64_t* full = bars + 2 * C;                                        // [slot] x-projection of the step has landed
  uint64_t* empty = full + h16::RING_SLOTS;                             // [slot] every compute warp has read it
  // F16: W_f holds [NUG][G][KB][hi, lo][32 lanes] A fragments and h_s [2][KB][32 slots] state pairs (rec_h16_layout.cuh);
  // red holds the row scales 2^e_r [G][HS] until the step loop first writes it
  __half* W_h = reinterpret_cast<__half*>(smem_raw);
  float* scl = red;
  constexpr int NSLOT = F16 ? h16::RING_SLOTS : Cfg::RING_SLOTS;
  auto ring_slot = [&](int s) {
    return F16 ? reinterpret_cast<float*>(smem_raw + L::ring_byte(s)) : ring_tail + s * (L::RING_SLOT_BYTES / 4);
  };

  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int ug = w % NUG, kh = w / NUG;
  const ClusterSlice cs = cluster_slice<C, BS, HS, VL>(p, nslices);
  const uint32_t rank = cs.rank;
  const int dir = cs.dir, b0 = cs.b0, j0 = cs.j0, T = cs.T;
  const float* w_hh = p.w_hh[dir];
  // as in rec_fwd_kernel, but the own slice is always delivered locally
  const ExchangeBars<C, 1, true> xb{bars, rank};

  if (tid == 0) {
    xb.init((uint32_t)NW);  // the own slice: one arrive per compute warp
    for (int s = 0; s < NSLOT; ++s) {
      ptx::mbar_init(&full[s], 1u);           // the producer's expect_tx, then the copies' bytes
      ptx::mbar_init(&empty[s], (uint32_t)NW);  // one arrive per compute warp
    }
    ptx::fence_mbar_init();
  }
  // the prologue is shared by all NT threads, the producer warpgroup included
  // GRU-256 fp16 pairs from the weight cache (RecFwdParams::whh16, frozen weights): the pairs and row scales the two
  // passes below would make, copied as they lie
  bool staged = false;
  if constexpr (F16 && Cfg::MODE == B200RNN_GRU) {
    if (p.whh16[dir]) {
      const uint4* img = reinterpret_cast<const uint4*>(static_cast<const unsigned char*>(p.whh16[dir]) +
                                                        L::cache_rank_byte((int)rank));
      uint4* dst = reinterpret_cast<uint4*>(smem_raw);
#pragma unroll 8
      for (int i = tid; i < L::W_HALVES * 2 / 16; i += NT) dst[i] = __ldg(img + i);
      for (int i = tid; i < G * HS / 4; i += NT)
        reinterpret_cast<uint4*>(scl)[i] = __ldg(img + L::W_HALVES * 2 / 16 + i);
      staged = true;
    }
  }
  if (!staged) {
  if constexpr (F16) {  // the row scales: each warp reduces SR rows at a time, their loads all in flight
    constexpr int SR = Cfg::SCALE_ROWS, NR = G * HS;
    for (int r0 = w * SR; r0 < NR; r0 += SR * (NT / 32)) {
      float m[SR];
#pragma unroll
      for (int i = 0; i < SR; ++i) {
        const int rr = SR == 1 ? r0 : min(r0 + i, NR - 1);  // past the last row: a repeat, never stored
        const float4* row = reinterpret_cast<const float4*>(w_hh + ((size_t)(rr / HS) * H + j0 + rr % HS) * H);
        m[i] = 0.f;
#pragma unroll
        for (int k = lane; k < H / 4; k += 32) {
          const float4 v = __ldg(row + k);
          m[i] = fmaxf(m[i], fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1)
#pragma unroll
        for (int i = 0; i < SR; ++i) m[i] = fmaxf(m[i], __shfl_xor_sync(FULLMASK, m[i], o));
      if (lane == 0)
#pragma unroll
        for (int i = 0; i < SR; ++i)
          if (SR == 1 || r0 + i < NR) scl[r0 + i] = ldexpf(1.f, h16::scale_exp(m[i]));
    }
    __syncthreads();
  }
  // this CTA's rows of the three gate blocks, read as coalesced float4 and scattered into A-fragment order: row u of
  // gate block g goes to unit group u / 16, tile g, fragment row u % 16; k0..k0+3 are the lanes t = 0..3 of one k-step
  // half
#pragma unroll 8
  for (int i = tid; i < G * HS * H / 4; i += NT) {
    const int rr = i / (H / 4), k0 = (i % (H / 4)) * 4;
    const int g = rr / HS, u = rr % HS;
    const float4 v = __ldg(reinterpret_cast<const float4*>(w_hh + ((size_t)g * H + j0 + u) * H + k0));
    if constexpr (F16) {  // k0, k0 + 1 and k0 + 2, k0 + 3 are the two halves of one f16x2 register each
      const float s = scl[rr];
      const float x[4] = {v.x * s, v.y * s, v.z * s, v.w * s};
#pragma unroll
      for (int e = 0; e < 4; e += 2) {
        const __half2 hi = __floats2half2_rn(x[e], x[e + 1]);
        const __half2 lo = __floats2half2_rn(x[e] - __low2float(hi), x[e + 1] - __high2float(hi));
        *reinterpret_cast<__half2*>(W_h + L::w_index(g, u, k0 + e, 0)) = hi;
        *reinterpret_cast<__half2*>(W_h + L::w_index(g, u, k0 + e, 1)) = lo;
      }
    } else {
      float* dst = reinterpret_cast<float*>(W_f + (((u / 16) * G + g) * KS + k0 / 8) * 32 + (u % 8) * 4) +
                   (u % 16) / 8 + 2 * ((k0 / 4) & 1);
      dst[0] = TF32 ? round_tf32(v.x) : v.x;
      dst[4] = TF32 ? round_tf32(v.y) : v.y;
      dst[8] = TF32 ? round_tf32(v.z) : v.z;
      dst[12] = TF32 ? round_tf32(v.w) : v.w;
    }
  }
  }
  if (!F16 && p.h_0) {  // buffer 0: the initial state in B-fragment order, rounded like the copies the lanes producing h_t hand over
    for (int i = tid; i < BS * H; i += NT) {
      const int q = i / H, k = i - q * H;
      const float v = initial_state<VL>(p, dir, b0, q, k);
      h_s[tc_state_index(k, q)] = TF32 ? round_tf32(v) : v;
      h_s[BS * H + i] = 0.f;
    }
  } else {
    for (int i = tid; i < 2 * BS * H; i += NT) h_s[i] = 0.f;  // h_0 = 0 (rnn.py:1432-1440)
  }
  __syncthreads();

  if (w >= NW) {  // the producer warpgroup: one lane fills the x-projection ring, the rest only meets the cluster barriers
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(Cfg::PRODUCER_REGS));
    ptx::cluster_sync_all();  // F16: the compute warps have read the n tile (the ring's space) into registers
    if (w == NW && lane == 0) {
      const float* gates = p.gates[dir];
      const int nvalid = min(BS, p.B - b0);  // slots past the batch are never read (FwdCell::valid)
      GiReady gi_ready;
      for (int step = 0; step < T; ++step) {
        const int s = step % NSLOT, t = dir ? (T - 1 - step) : step;
        if (step >= NSLOT) ptx::mbar_wait(&empty[s], (step / NSLOT - 1) & 1);
        if (p.ready) {
          gi_ready.wait(p, t);
          ptx::fence_proxy_async_global();  // the GEMM's stores, acquired above, are read by the bulk copies below
        }
        float* slot = ring_slot(s);
        ptx::mbar_arrive_expect_tx(&full[s], (uint32_t)(nvalid * G * HS * sizeof(float)));
        for (int q = 0; q < nvalid; ++q) {
          const int row = VL ? p.order[b0 + q] : b0 + q;
          const float* src = gates + ((size_t)t * p.B + row) * (G * H) + j0;
#pragma unroll
          for (int g = 0; g < G; ++g)
            ptx::tma_bulk_g2s(slot + L::ring_index(g, q, 0), src + g * H, (uint32_t)(HS * sizeof(float)), &full[s]);
        }
      }
    }
    __syncwarp();
    ptx::cluster_sync_all();  // the compute warps' final one
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(Cfg::COMPUTE_REGS));

  // ---- lane identity: output jb is unit ju, batch row b0 + 2 * ft + jb (accumulator fragment elements 2*kh + jb) ---
  const int fg = lane >> 2, ft = lane & 3;
  const int u0 = ug * 16 + kh * 8;  // first unit (within the CTA's slice) this warp finishes
  // F16: the last RT tiles' A fragments of this warp's k-blocks in registers (GRU: the n tile; LSTM: g and o),
  // [tile][slice in visiting order][k-block][hi, lo], and the unscale 2^-(e_r + 14) of the lane's G rows (read before
  // anyone writes `red` in the step loop)
  uint32_t wreg[F16 ? RT : 1][F16 ? C : 1][KBC / 2][2][4];
  float unscale[G];
  if constexpr (F16) {
#pragma unroll
    for (int rt = 0; rt < RT; ++rt)
#pragma unroll
      for (int c = 0; c < C; ++c)
#pragma unroll
        for (int kk = 0; kk < KBC / 2; ++kk)
#pragma unroll
          for (int hl = 0; hl < 2; ++hl) {
            const int kb = ((c + (int)rank) % C) * KBC + kh * (KBC / 2) + kk;
            const uint4 v = *reinterpret_cast<const uint4*>(W_h + L::w_half(ug, G - RT + rt, kb, hl, lane, 0, 0));
            uint32_t* wr = wreg[rt][c][kk][hl];
            wr[0] = v.x; wr[1] = v.y; wr[2] = v.z; wr[3] = v.w;
          }
#pragma unroll
    for (int g = 0; g < G; ++g) unscale[g] = __frcp_rn(scl[g * HS + u0 + fg]) * (1.f / h16::STATE_SCALE);
  }
  ptx::cluster_sync_all();  // peers' barriers and state buffers are initialised before anyone writes into them
  const int ju = j0 + u0 + fg;
  FwdCell<Cfg::MODE, H, VL> cell[2] = {{p, dir, ju, b0 + 2 * ft}, {p, dir, ju, b0 + 2 * ft + 1}};

  const float4* W_w = W_f + (size_t)ug * G * KS * 32 + lane;
  float* red_mine = red + w * 2 * G * 32 + lane;                         // written by this warp
  const float* red_partner = red + (w ^ NUG) * 2 * G * 32 + lane;        // written by the other k half
#pragma unroll
  for (int jb = 0; jb < 2; ++jb) cell[jb].start(p, dir);
  for (int step = 0; step < T; ++step) {
    const int t = dir ? (T - 1 - step) : step;
    const int cur = xb.buf(step), nxt = cur ^ 1;
    const float2* h_cur = reinterpret_cast<const float2*>(h_s + cur * BS * H) + lane;
    const uint32_t par = xb.parity(step);
#ifdef B200RNN_TRACE
    const bool tr = p.trace != nullptr && blockIdx.x == 0 && lane == 0;  // one row of 16 stamps per (step, warp)
#else
    constexpr bool tr = false;  // build with -DB200RNN_TRACE for the per-phase clock64 timeline (tools/trace_rec.py tc)
#endif
    long long* trow = p.trace + ((size_t)step * NW + w) * 16;
    if (tr) trow[0] = clock64();

    float acc[G][4];
#pragma unroll
    for (int g = 0; g < G; ++g)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[g][i] = 0.f;
    // one source slice at a time, starting with the slice this CTA produced itself
#pragma unroll
    for (int c = 0; c < C; ++c) {
      const int src = (c + (int)rank) % C;
      if (step > 0) xb.wait(cur, src, par);
      if (tr) trow[1 + c] = clock64();  // slice c (own first) has arrived
      float d[G][2][4];  // [gate tile][lo*hi + hi*lo, hi*hi]; TF32: [gate tile][-, the single product]
#pragma unroll
      for (int g = 0; g < G; ++g)
#pragma unroll
        for (int m = 0; m < 2; ++m)
#pragma unroll
          for (int i = 0; i < 4; ++i) d[g][m][i] = 0.f;
      if constexpr (F16) {  // k-blocks of 16: this warp takes k-blocks kh*2, kh*2 + 1 of every source slice
        const uint4* h_q = reinterpret_cast<const uint4*>(h_s + cur * BS * H) + h16::state_slot(lane);
#pragma unroll
        for (int kk = 0; kk < KBC / 2; ++kk) {
          const int kb = src * KBC + kh * (KBC / 2) + kk;
          const uint4 hv = h_q[kb * 32];  // {hi b0, hi b1, lo b0, lo b1}
          const uint32_t bh[2] = {hv.x, hv.y}, bl[2] = {hv.z, hv.w};
#pragma unroll
          for (int g = 0; g < G; ++g) {
            uint32_t ah[4], al[4];
            if (g < G - RT) {
              const uint4* wp = reinterpret_cast<const uint4*>(W_h + L::w_half(ug, g, kb, 0, lane, 0, 0));
              const uint4 vh = wp[0], vl = wp[32];  // hi, then lo: 32 lanes x 16 bytes further
              ah[0] = vh.x; ah[1] = vh.y; ah[2] = vh.z; ah[3] = vh.w;
              al[0] = vl.x; al[1] = vl.y; al[2] = vl.z; al[3] = vl.w;
            } else {
#pragma unroll
              for (int r = 0; r < 4; ++r) {
                ah[r] = wreg[g - (G - RT)][c][kk][0][r];
                al[r] = wreg[g - (G - RT)][c][kk][1][r];
              }
            }
            ptx::mma_f16_m16n8k16(d[g][0], al, bh);
            ptx::mma_f16_m16n8k16(d[g][0], ah, bl);
            ptx::mma_f16_m16n8k16(d[g][1], ah, bh);
          }
        }
      } else {
#pragma unroll
      for (int kk = 0; kk < KSC / 2; ++kk) {
        const int ks = src * KSC + kh * (KSC / 2) + kk;
        const float2 hv = h_cur[ks * 32];
        if constexpr (TF32) {  // both operands are TF32 already
          const uint32_t b[2] = {__float_as_uint(hv.x), __float_as_uint(hv.y)};
#pragma unroll
          for (int g = 0; g < G; ++g) {
            const float4 wv = W_w[(g * KS + ks) * 32];
            const uint32_t a[4] = {__float_as_uint(wv.x), __float_as_uint(wv.y), __float_as_uint(wv.z),
                                   __float_as_uint(wv.w)};
            ptx::mma_tf32_m16n8k8(d[g][1], a, b);
          }
        } else {
          uint32_t bh[2], bl[2];
          ptx::split_tf32(hv.x, bh[0], bl[0]);
          ptx::split_tf32(hv.y, bh[1], bl[1]);
#pragma unroll
          for (int g = 0; g < G; ++g) {
            const float4 wv = W_w[(g * KS + ks) * 32];
            uint32_t ah[4], al[4];
            ptx::split_tf32(wv.x, ah[0], al[0]);
            ptx::split_tf32(wv.y, ah[1], al[1]);
            ptx::split_tf32(wv.z, ah[2], al[2]);
            ptx::split_tf32(wv.w, ah[3], al[3]);
            ptx::mma_tf32_m16n8k8(d[g][0], al, bh);
            ptx::mma_tf32_m16n8k8(d[g][0], ah, bl);
            ptx::mma_tf32_m16n8k8(d[g][1], ah, bh);
          }
        }
      }
      }
#pragma unroll
      for (int g = 0; g < G; ++g)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[g][i] += TF32 ? d[g][1][i] : d[g][0][i] + d[g][1][i];
      if (c == 0) {
        if (step > 0) {  // the previous step's stores
#pragma unroll
          for (int jb = 0; jb < 2; ++jb) cell[jb].flush(p, dir, dir ? (T - step) : (step - 1));
        }
        // this step's x-projection from its ring slot (already complete in the steady state); the slot is released
        // to the producer once the whole warp has read it
        const int s = step % NSLOT;
        ptx::mbar_wait(&full[s], (step / NSLOT) & 1);
        const float* slot = ring_slot(s);
#pragma unroll
        for (int jb = 0; jb < 2; ++jb)
          if (cell[jb].valid) {
#pragma unroll
            for (int g = 0; g < G; ++g) cell[jb].gi[g] = slot[L::ring_index(g, 2 * ft + jb, u0 + fg)];
          }
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(&empty[s]);
      }
    }
    // every slice of h_step has been consumed by this thread => the barriers of the other buffer are re-armed
    if (tid == 0 && step + 1 < T) xb.arm(nxt, (uint32_t)(BS * HS * sizeof(float)));
    if (tr) trow[5] = clock64() + (long long)(acc[0][0] + acc[1][0] + acc[2][0] == 12345.678f);  // contraction done
    // swap halves with the partner warp: it finishes the other 8 units. WAR on `red`: the partner overwrites it only
    // after its next step's own-slice wait, which needs this warp's arrive below (after the read).
#pragma unroll
    for (int g = 0; g < G; ++g)
#pragma unroll
      for (int jb = 0; jb < 2; ++jb) red_mine[(g * 2 + jb) * 32] = kh ? acc[g][jb] : acc[g][2 + jb];
    ptx::named_barrier_sync(1 + ug, 64);
    float pre[2][G];  // recurrent pre-activations of this lane's two outputs
#pragma unroll
    for (int g = 0; g < G; ++g)
#pragma unroll
      for (int jb = 0; jb < 2; ++jb) {
        pre[jb][g] = (kh ? acc[g][2 + jb] : acc[g][jb]) + red_partner[(g * 2 + jb) * 32];
        if constexpr (F16) pre[jb][g] *= unscale[g];
      }
    if (tr) trow[6] = clock64() + (long long)(pre[0][0] == 12345.678f);  // k-half swap done
    float hnew[2];
#pragma unroll
    for (int jb = 0; jb < 2; ++jb) hnew[jb] = cell[jb].update(t, pre[jb]);
    if (tr) trow[7] = clock64() + (long long)(hnew[0] + hnew[1] == 12345.678f);  // update done

    if (step + 1 < T) {
      // own copy with ordinary stores; after __syncwarp the warp's k-step is 16 contiguous float4 that go to the peers
      // with st.async (ordering of the local path: allgather_units)
      float* h_nxt = h_s + nxt * BS * H;
      if constexpr (F16) {  // the pair of the scaled state; the cell keeps the fp32 h (h16::exchange_chunk is the
                            // 16-byte chunk index lane * 4 floats below points at)
        __half* h_h = reinterpret_cast<__half*>(h_nxt);
#pragma unroll
        for (int jb = 0; jb < 2; ++jb) {
          const float v = hnew[jb] * h16::STATE_SCALE;
          const __half hi = __float2half_rn(v);
          h_h[L::state_index(ju, 2 * ft + jb, 0)] = hi;
          h_h[L::state_index(ju, 2 * ft + jb, 1)] = __float2half_rn(v - __half2float(hi));
        }
      } else {
#pragma unroll
        for (int jb = 0; jb < 2; ++jb) h_nxt[tc_state_index(ju, 2 * ft + jb)] = TF32 ? round_tf32(hnew[jb]) : hnew[jb];
      }
      __syncwarp();
      if (lane < 16) {
        float* mine = h_nxt + (j0 + u0) / 8 * 64 + lane * 4;
        const float4 v = *reinterpret_cast<const float4*>(mine);
        const uint32_t dst = ptx::smem_u32(mine), bar = ptx::smem_u32(xb.bar(nxt, rank));
#pragma unroll
        for (int r = 1; r < C; ++r) {
          const uint32_t peer = (rank + r) % C;
          ptx::st_async_v4(ptx::mapa(dst, peer), v, ptx::mapa(bar, peer));
        }
      }
      if (lane == 0) ptx::mbar_arrive(xb.bar(nxt, rank));
    }
    if (tr) trow[8] = clock64();  // slice sent

    if (step == T - 1) {
#pragma unroll
      for (int jb = 0; jb < 2; ++jb) cell[jb].flush(p, dir, t);
#pragma unroll
      for (int jb = 0; jb < 2; ++jb) cell[jb].finish(p, dir);
    }
  }
  if constexpr (VL) {
#pragma unroll
    for (int jb = 0; jb < 2; ++jb) cell[jb].skip_tail(p, dir, T);
  }
  ptx::cluster_sync_all();  // nobody exits while a peer could still address its shared memory
}

// GRU-256: 3xTF32 (the default), single-pass TF32 and fp16-pair instantiations, fixed-length and ragged
template <bool VL>
__global__ void __launch_bounds__(TcFwdCfg::NT, 1) rec_fwd_tc_kernel(const RecFwdParams p, const int nslices) {
  rec_fwd_tc_body<TcFwdCfg, VL, TcOp::X3>(p, nslices);
}
template <bool VL>
__global__ void __launch_bounds__(TcFwdCfg::NT, 1) rec_fwd_tf32_kernel(const RecFwdParams p, const int nslices) {
  rec_fwd_tc_body<TcFwdCfg, VL, TcOp::TF32>(p, nslices);
}
template <bool VL>
__global__ void __launch_bounds__(TcFwdCfg::NT, 1) rec_fwd_h16_kernel(const RecFwdParams p, const int nslices) {
  rec_fwd_tc_body<TcFwdCfg, VL, TcOp::F16>(p, nslices);
}
// LSTM-128: fp16 pairs only (the no-grad forward of b200rnn_forward_fused), fixed-length and ragged
template <bool VL>
__global__ void __launch_bounds__(TcLstmCfg::NT, 1) lstm_fwd_h16_kernel(const RecFwdParams p, const int nslices) {
  rec_fwd_tc_body<TcLstmCfg, VL, TcOp::F16>(p, nslices);
}

// W_hh [G*H][H] of a GRU-256 layer -> its weight cache image (h16::Gru256, prep_whh_h16), one warp per row: the row
// scale and split of rec_fwd_tc_body's F16 prologue (the same max, scale and roundings, so the staged pairs are
// bit-identical), written in each rank's A-fragment order
__global__ void __launch_bounds__(256) whh_h16_prep_kernel(const float* __restrict__ w_hh, unsigned char* __restrict__ img) {
  using L = h16::Gru256;
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= L::G * L::H) return;
  const int g = row / L::H, rank = row % L::H / L::HS, u = row % L::HS;
  const float4* src = reinterpret_cast<const float4*>(w_hh + (size_t)row * L::H);
  float4 v[L::H / 128];
  float m = 0.f;
#pragma unroll
  for (int i = 0; i < L::H / 128; ++i) {
    v[i] = __ldg(src + lane + 32 * i);
    m = fmaxf(m, fmaxf(fmaxf(fabsf(v[i].x), fabsf(v[i].y)), fmaxf(fabsf(v[i].z), fabsf(v[i].w))));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(FULLMASK, m, o));
  const float s = ldexpf(1.f, h16::scale_exp(m));
  unsigned char* base = img + L::cache_rank_byte(rank);
  __half* W = reinterpret_cast<__half*>(base);
#pragma unroll
  for (int i = 0; i < L::H / 128; ++i) {
    const int k0 = (lane + 32 * i) * 4;
    const float x[4] = {v[i].x * s, v[i].y * s, v[i].z * s, v[i].w * s};
#pragma unroll
    for (int e = 0; e < 4; e += 2) {
      const __half2 hi = __floats2half2_rn(x[e], x[e + 1]);
      const __half2 lo = __floats2half2_rn(x[e] - __low2float(hi), x[e + 1] - __high2float(hi));
      *reinterpret_cast<__half2*>(W + L::w_index(g, u, k0 + e, 0)) = hi;
      *reinterpret_cast<__half2*>(W + L::w_index(g, u, k0 + e, 1)) = lo;
    }
  }
  if (lane == 0) reinterpret_cast<float*>(base + L::W_HALVES * 2)[g * L::HS + u] = s;
}

// =================================================================================================
// backward (BPTT)
// =================================================================================================
// w_prep layout (written by whh_prep_kernel): [C ranks][G][HS][H],
//   w_prep[rank][g][u][jj] = W_hh[g*H + jj][rank*HS + u]
// i.e. for every gate block the transposed slice a CTA needs, contiguous per CTA (TMA bulk copyable).
template <int MODE, int H, int C, int BS, int KL, int UPL, int RG, bool VL = false>
__global__ void __launch_bounds__(RecCfg<MODE, H, C, BS, KL, UPL, RG>::NT, 1)
    rec_bwd_kernel(const RecBwdParams p, const int nslices) {
  using Cfg = RecCfg<MODE, H, C, BS, KL, UPL, RG>;
  using LM = LaneMap<KL, UPL, BS>;
  static_assert(RG <= 1, "the backward kernel keeps at most one gate block in registers");
  constexpr int G = Cfg::G, GH = Cfg::GH, HS = Cfg::HS, NT = Cfg::NT, UPW = Cfg::UPW, NSM = Cfg::NSM;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* W_s = reinterpret_cast<float*>(smem_raw);   // [NSM][HS][H] transposed gate blocks
  float* d_s = W_s + (size_t)NSM * HS * H;           // [2][BS][G*H] gate gradients of the whole cluster
  uint64_t* bars = reinterpret_cast<uint64_t*>(d_s + 2 * BS * GH);  // [0] weights, [1 + buf*C + src]
  constexpr int NCH = Cfg::NCH, CPS = Cfg::CPS, SPC = Cfg::SPC;

  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const ClusterSlice cs = cluster_slice<C, BS, HS, VL>(p, nslices);
  const uint32_t rank = cs.rank;
  const int dir = cs.dir, slice = cs.slice, b0 = cs.b0, j0 = cs.j0, T = cs.T;
  const int B = p.B;
  const float* w_prep = p.w_prep[dir] + (size_t)rank * G * HS * H;
  // step s contracts against the gate gradients it sent itself
  const ExchangeBars<C, 0, kLocalSelf, 1> xb{bars, rank};

  if (tid == 0) {
    ptx::mbar_init(&bars[0], 1u);          // weights (tx bytes)
    xb.init((uint32_t)(Cfg::NW * G));      // the own slice: G gate-gradient slices x NW warps arrive per exchange
    ptx::fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    ptx::mbar_arrive_expect_tx(&bars[0], (uint32_t)Cfg::W_BYTES);
#pragma unroll
    for (int g = 0; g < NSM; ++g)
      ptx::tma_bulk_g2s(W_s + (size_t)g * HS * H, w_prep + (size_t)g * HS * H, (uint32_t)(HS * H * sizeof(float)),
                        &bars[0]);
  }
  for (int i = tid; i < 2 * BS * GH; i += NT) d_s[i] = 0.f;
  const int rot = Cfg::ROT ? (int)rank * CPS : 0;
  float wreg[1][UPL][H / KL];
  load_resident<RG, KL, UPL, BS, H>(w_prep + (size_t)NSM * HS * H, HS, (long long)w * UPW, rot, lane, wreg);
  ptx::mbar_wait(&bars[0], 0);
  __syncthreads();
  ptx::cluster_sync_all();

  const int uw = LM::unit(lane), qb = LM::q(lane);
  const int j = j0 + w * UPW + uw;
  const bool valid = b0 + qb < B;
  const int b = (VL && valid) ? p.order[b0 + qb] : b0 + qb;  // VL: batch slot b0 + qb holds row order[b0 + qb]
  const float* gates = p.gates[dir];
  const float* extra = p.extra[dir];
  float* dgates = p.dgates[dir];

  int len_b = T;
  if constexpr (VL) {
    if (valid) len_b = p.lengths[b];
  }
  float dh_carry = 0.f, dc_carry = 0.f;
  if (valid) {
    if (p.dh_n) dh_carry = p.dh_n[((size_t)dir * B + b) * H + j];
    if (MODE == B200RNN_LSTM && p.dc_n) dc_carry = p.dc_n[((size_t)dir * B + b) * H + j];
  }
  float bsum[G + 1];
#pragma unroll
  for (int g = 0; g <= G; ++g) bsum[g] = 0.f;

  // pooled output (mean / sum over time fused into the caller's graph): every step receives the same gradient row
  const float dy_pooled = (!p.dy && p.dy_pool && valid) ? p.dy_pool[(size_t)b * p.D * H + dir * H + j] * p.dy_scale : 0.f;
  // operands of the current step (prefetched one step ahead)
  float sv[G], sx = 0.f, hp = 0.f, dyv = 0.f;  // saved gates, hn / c_t, h_{prev} / c_{prev}, dy
#pragma unroll
  for (int g = 0; g < G; ++g) sv[g] = 0.f;
  // the state before the first step: h_0 (GRU, feeds dz) or c_0 (LSTM, feeds df), zeros when NULL
  const float* s0 = (MODE == B200RNN_GRU) ? p.h_0 : p.c_0;
  auto load_step = [&](int step) {
    const int t = dir ? step : (T - 1 - step);
    bool has_prev = step < T - 1;
    const int tp = dir ? t + 1 : t - 1;
    // GRU, VL: the forward output at tp >= len_b is the masked 0, not the state the row kept (h_0: the reverse
    // direction's first real step t = len_b - 1 reads it). The LSTM reads c from `extra`, where frozen steps saved the
    // kept state.
    if (MODE == B200RNN_GRU && VL && tp >= len_b) has_prev = false;
    const float* gp = gates + ((size_t)t * B + b) * GH + j;
#pragma unroll
    for (int g = 0; g < G; ++g) sv[g] = gp[g * H];
    sx = extra[((size_t)t * B + b) * H + j];
    dyv = p.dy ? p.dy[(long long)t * p.dy_st + (long long)b * p.dy_sb + dir * H + j] : dy_pooled;
    if (!has_prev)
      hp = s0 ? s0[((size_t)dir * B + b) * H + j] : 0.f;
    else if (MODE == B200RNN_GRU)
      hp = p.y[(long long)tp * p.y_st + (long long)b * p.y_sb + dir * H + j];
    else
      hp = extra[((size_t)tp * B + b) * H + j];
  };
  if (valid && T > 0) load_step(0);

  // dh_0 requested: the last step also runs the exchange and the contraction, whose result is dh_0 (the same phase
  // bookkeeping as any other step); else it ends after its stores
  const bool want_dh0 = p.dh_0 != nullptr;
  for (int step = 0; step < T; ++step) {
    const int t = dir ? step : (T - 1 - step);
    const int buf = xb.buf(step);
    float* d_buf = d_s + buf * BS * GH;
    const bool last = (step == T - 1);
    const bool contract = !last || want_dh0;
    if (tid == 0 && contract) xb.arm(buf, (uint32_t)(BS * G * HS * sizeof(float)));

    // ---- cell backward for (unit j, batch b) ----------------------------------------------------
    float dh = dh_carry + dyv;
    if constexpr (VL) {
      if (t >= len_b) dh = dh_carry;  // the output of a frozen step is the constant 0: its dy reaches nothing
    }
    float dg[G], direct, dhn = 0.f;
    if constexpr (MODE == B200RNN_GRU) {
      direct = gru_cell_bwd(sv, sx, hp, dh, dg, dhn);
    } else {
      const float dc_next = lstm_cell_bwd(sv, sx, hp, dh, dc_carry, dg);
      direct = 0.f;
      if constexpr (VL) {
        if (t >= len_b) direct = dh;  // frozen step: dh and dc pass straight through
        else dc_carry = dc_next;
      } else {
        dc_carry = dc_next;
      }
    }
    if constexpr (VL) {
      if (t >= len_b) {
#pragma unroll
        for (int g = 0; g < G; ++g) dg[g] = 0.f;
        dhn = 0.f;
        if (MODE == B200RNN_GRU) direct = dh;
      }
    }
    if (valid) {
#pragma unroll
      for (int g = 0; g < G; ++g) bsum[g] += dg[g];
      bsum[G] += dhn;
    }

    if (contract) {
      // all-gather the recurrent-side gate gradient (GRU: n-gate part is dn*r) into every peer CTA
#pragma unroll
      for (int g = 0; g < G; ++g) {
        float v = dg[g];
        if (MODE == B200RNN_GRU && g == 2) v = dhn;
        if (!valid) v = 0.f;
        allgather_units<C, KL, UPL, BS, kLocalSelf>(v, d_buf, GH, g * H + j0 + w * UPW, xb.bar(buf, rank), lane, rank);
      }
    }

    if (valid) {
      float* gp = dgates + ((size_t)t * B + b) * GH + j;
#pragma unroll
      for (int g = 0; g < G; ++g) gp[g * H] = dg[g];
      if (MODE == B200RNN_GRU) p.dghn[dir][((size_t)t * B + b) * H + j] = dhn;
    }
    if (!contract) break;
    if (valid && !last) load_step(step + 1);
    const uint32_t par = xb.parity(step);

    // ---- dh_{prev}[b][j] = direct + sum_col dgh[b][col] * W_hh[col][j], one gate block of columns at a time ----
    // even-k / odd-k partial sums in one float2 accumulator (two independent FMA chains), folded before the butterfly
    float2 acc2[1][UPL][BS];
    float acc[1][UPL][BS];
#pragma unroll
    for (int au = 0; au < UPL; ++au)
#pragma unroll
      for (int ab = 0; ab < BS; ++ab) acc2[0][au][ab] = make_float2(0.f, 0.f);
    // chunk by chunk over the source CTAs (own slice first); a source's G gate-gradient slices share one barrier
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const int ca = (c + rot) % NCH;
      if (Cfg::ROT) {
        if (c % CPS == 0) xb.wait(buf, ca / CPS, par);
      } else {
#pragma unroll
        for (int s2 = 0; s2 < SPC; ++s2) xb.wait(buf, ca * SPC + s2, par);
      }
#pragma unroll
      for (int g = 0; g < G; ++g) {
        if (g < NSM)
          dots_chunk2<1, 0, KL, UPL, BS, H, GH>(W_s + (size_t)g * HS * H, 0, w * UPW, wreg, d_buf + g * H, c, ca,
                                                lane, acc2);
        else
          dots_chunk2<1, 1, KL, UPL, BS, H, GH>(W_s, 0, 0, wreg, d_buf + g * H, c, ca, lane, acc2);
      }
    }
    fold_pairs<1, UPL, BS>(acc2, acc);
    warp_transpose_reduce<1, KL, UPL, BS>(acc);
    dh_carry = direct + acc[0][0][0];
  }
  // gradients w.r.t. the initial state: what the scan carried past its first step (frozen steps pass dh / dc through,
  // and a cluster that ran no step passes dh_n / dc_n on)
  if (valid) {
    if (want_dh0) p.dh_0[((size_t)dir * B + b) * H + j] = dh_carry;
    if (MODE == B200RNN_LSTM && p.dc_0) p.dc_0[((size_t)dir * B + b) * H + j] = dc_carry;
  }
  if constexpr (VL) {
    // the steps [T, p.T) the cluster skipped: their gate gradients are 0, as past any sequence's length (the wgrad and
    // dgrad GEMMs sum over every step)
    if (valid)
      for (int t = T; t < p.T; ++t) {
        float* gp = dgates + ((size_t)t * B + b) * GH + j;
#pragma unroll
        for (int g = 0; g < G; ++g) gp[g * H] = 0.f;
        if (MODE == B200RNN_GRU) p.dghn[dir][((size_t)t * B + b) * H + j] = 0.f;
      }
  }

  // ---- per-slice bias-gradient partials: sum over this slice's batch rows (the low lane bits) -------------
#pragma unroll
  for (int g = 0; g <= G; ++g) {
    float v = bsum[g];
#pragma unroll
    for (int off = 1; off < BS; off <<= 1) v += __shfl_xor_sync(FULLMASK, v, off);
    bsum[g] = v;
  }
  if (qb == 0) {
    float* out = p.dbias_part[dir] + (size_t)slice * (G + 1) * H;
#pragma unroll
    for (int g = 0; g < G; ++g) out[g * H + j] = bsum[g];
    out[G * H + j] = bsum[G];
  }
  ptx::cluster_sync_all();
}

// =================================================================================================
// LSTM with a projection (proj_size P > 0): forward and BPTT
// =================================================================================================
// h_t = W_hr (o_t * tanh c_t), h_t of width P < H. A cluster of C CTAs owns BS batch rows, CTA `rank` owns HS = H/C cell
// units and keeps on chip, for the whole sequence:
//   W_s [G*HS][P]: the W_hh rows of its units (row g*HS + u = W_hh[g*H + j0 + u][:]), K = P;
//   R_s [HS][P]:   the W_hr columns of its units, transposed (R_s[u][p] = W_hr[p][j0 + u]).
// Rows are padded to P + 4 floats, so that the 8 units a quarter-warp reads with one 16-byte load sit in different banks.
// One thread per (unit u, batch slot b): NT = HS * BS. Forward step:
//   1. gate pre-activations W_s h_{t-1} for its 4 rows, cell update, m = o * tanh(c) into m_s[b][u];
//   2. the CTA's partial projection h^(r)[b][:] = R_s^T m_s[b] (all P outputs from its HS units);
//   3. the partial goes to every peer's slot [rank] (st.async, one mbarrier per source and buffer, double buffered);
//   4. next step, every CTA adds the C partials in rank order 0..C-1: all CTAs hold the same bits of h_t, which is the
//      next contraction's operand; CTA r writes its P/C columns of y and h_n.
// One exchange per step, as in the unprojected kernels, with P-wide partials instead of HS-wide state slices. BPTT
// mirrors it: dh_t = dy_t + (the C partials of W_hh^T dgates, in rank order), dm = W_hr[:, units]^T dh_t, the LSTM cell
// backward from dm, and the CTA's partial W_hh[units]^T dgates goes to the peers. dh_t is written to `dhp` for the
// dW_hr GEMM. Ragged batches (VL) as in the other kernels: a frozen step keeps (h, c) and emits 0; in BPTT its dh passes
// through (rank 0 carries it in its partial, the others add zeros, so the sum is exact).
template <int H, int P, int C, int BS>
struct ProjCfg {
  static constexpr int G = 4, HS = H / C, NT = HS * BS;
  static constexpr int LD = P + 4;  // padded row of W_s / R_s
  static constexpr int NG = (NT / P < BS) ? NT / P : BS;  // batch groups of the P-wide partial contraction
  static constexpr int RB = BS / NG;                     // batch rows per thread in it
  static constexpr size_t W_FLOATS = (size_t)G * HS * LD, R_FLOATS = (size_t)HS * LD;
  static constexpr size_t V_FLOATS = (size_t)BS * P, SLOT_FLOATS = (size_t)2 * C * BS * P;
  static constexpr size_t SMEM_F = (W_FLOATS + R_FLOATS + V_FLOATS + SLOT_FLOATS + (size_t)BS * HS) * sizeof(float) +
                                   2 * C * sizeof(uint64_t) + 2 * BS * sizeof(int);
  static constexpr size_t SMEM_B = (W_FLOATS + R_FLOATS + V_FLOATS + SLOT_FLOATS + (size_t)BS * G * HS) * sizeof(float) +
                                   2 * C * sizeof(uint64_t) + 2 * BS * sizeof(int);
  static_assert(HS * C == H && HS % 8 == 0 && P % (4 * C) == 0 && P % 4 == 0, "bad split");
  static_assert(NT % 32 == 0 && NT <= 1024 && NG >= 1 && NG * RB == BS && NT >= P, "bad thread count");
};

// Thread (unit, batch slot) of the projected kernels: 8 consecutive units by 4 batch slots per warp
template <int BS>
__device__ __forceinline__ void proj_thread(int tid, int& u, int& b) {
  u = (tid & 7) + 8 * (tid / (8 * BS));
  b = (tid >> 3) % BS;
}

// Stage this CTA's W_hh rows and W_hr columns (once per launch), the row / length of every batch slot
template <int H, int P, int C, int BS, bool VL>
__device__ __forceinline__ void proj_prologue(const float* __restrict__ w_hh, const float* __restrict__ w_hr, int j0,
                                              int b0, int B, int T, const int* lengths, const int* order, float* W_s,
                                              float* R_s, int* row_s, int* len_s, int tid) {
  using Cfg = ProjCfg<H, P, C, BS>;
  constexpr int G = Cfg::G, HS = Cfg::HS, NT = Cfg::NT, LD = Cfg::LD;
  for (int i = tid; i < G * HS * P / 4; i += NT) {
    const int r = i / (P / 4), k = (i % (P / 4)) * 4;
    const int g = r / HS, u = r - g * HS;
    *reinterpret_cast<float4*>(&W_s[r * LD + k]) =
        __ldg(reinterpret_cast<const float4*>(w_hh + ((size_t)g * H + j0 + u) * P + k));
  }
  for (int i = tid; i < P * HS; i += NT) {
    const int pp = i / HS, u = i - pp * HS;
    R_s[u * LD + pp] = __ldg(w_hr + (size_t)pp * H + j0 + u);
  }
  if (tid < BS) {
    const int slot = b0 + tid;
    const bool valid = slot < B;
    const int row = (VL && valid) ? order[slot] : slot;
    row_s[tid] = valid ? row : -1;
    len_s[tid] = (VL && valid) ? min(max(lengths[row], 0), T) : T;
  }
}

// Send this CTA's partial (own slot, written and published by __syncthreads) to the C-1 peers' slot [rank]
template <int P, int C, int BS, int NT>
__device__ __forceinline__ void proj_send(float* own, uint64_t* bar, uint32_t rank, int tid) {
  constexpr int NV = BS * P / 4;
  const uint32_t bar_addr = ptx::smem_u32(bar);
  for (int i = tid; i < (C - 1) * NV; i += NT) {
    const int r = i / NV, v = i - r * NV;
    const uint32_t peer = (rank + 1 + r) % C;
    float* src = own + v * 4;
    ptx::st_async_v4(ptx::mapa(ptx::smem_u32(src), peer), *reinterpret_cast<const float4*>(src),
                     ptx::mapa(bar_addr, peer));
  }
}

// Partial P-wide contraction of the CTA's K values per batch row: out[b][pp] = sum_k A[k * LD + pp] * v[b][k], k in
// increasing order (one FMA chain per output: deterministic). Threads (pp, batch group) of NG groups of RB rows.
template <int P, int BS, int NG, int RB, int K>
__device__ __forceinline__ void proj_partial(const float* __restrict__ A, int ld, const float* __restrict__ v,
                                             float* __restrict__ out, int tid) {
  if (tid >= P * NG) return;
  const int pp = tid % P, bg = tid / P;
  float acc[RB];
#pragma unroll
  for (int r = 0; r < RB; ++r) acc[r] = 0.f;
#pragma unroll 4
  for (int k = 0; k < K; k += 4) {
    const float a0 = A[(k + 0) * ld + pp], a1 = A[(k + 1) * ld + pp], a2 = A[(k + 2) * ld + pp],
                a3 = A[(k + 3) * ld + pp];
#pragma unroll
    for (int r = 0; r < RB; ++r) {
      const float4 x = *reinterpret_cast<const float4*>(&v[(bg * RB + r) * K + k]);
      float a = acc[r];
      a = fmaf(a0, x.x, a);
      a = fmaf(a1, x.y, a);
      a = fmaf(a2, x.z, a);
      a = fmaf(a3, x.w, a);
      acc[r] = a;
    }
  }
#pragma unroll
  for (int r = 0; r < RB; ++r) out[(bg * RB + r) * P + pp] = acc[r];
}

template <int H, int P, int C, int BS, bool VL>
__global__ void __launch_bounds__(ProjCfg<H, P, C, BS>::NT, 1)
    rec_fwd_proj_kernel(const RecFwdParams p, const int nslices) {
  using Cfg = ProjCfg<H, P, C, BS>;
  constexpr int G = Cfg::G, HS = Cfg::HS, NT = Cfg::NT, LD = Cfg::LD, PC = P / C;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* W_s = reinterpret_cast<float*>(smem_raw);  // [G*HS][LD]
  float* R_s = W_s + Cfg::W_FLOATS;                 // [HS][LD]
  float* h_s = R_s + Cfg::R_FLOATS;                 // [BS][P] h_{t-1}
  float* slot = h_s + Cfg::V_FLOATS;                // [2][C][BS][P] partial projections
  float* m_s = slot + Cfg::SLOT_FLOATS;             // [BS][HS]
  uint64_t* bars = reinterpret_cast<uint64_t*>(m_s + BS * HS);  // [buf * C + src]
  int* row_s = reinterpret_cast<int*>(bars + 2 * C);            // [BS] batch row of each slot (-1: past the batch)
  int* len_s = row_s + BS;                                      // [BS] steps of each slot

  const int tid = threadIdx.x;
  const ClusterSlice cs = cluster_slice<C, BS, HS, VL>(p, nslices);
  const uint32_t rank = cs.rank;
  const int dir = cs.dir, b0 = cs.b0, j0 = cs.j0, T = cs.T;
  const int B = p.B;
  // step s sums the partials step s - 1 sent; the own slot is never awaited
  const ExchangeBars<C, 1, true> xb{bars, rank};

  if (tid == 0) {
    xb.init(1u);
    ptx::fence_mbar_init();
  }
  proj_prologue<H, P, C, BS, VL>(p.w_hh[dir], p.w_hr[dir], j0, b0, B, p.T, p.lengths, p.order, W_s, R_s, row_s, len_s,
                                 tid);
  __syncthreads();
  for (int i = tid; i < BS * P; i += NT) {  // h_0 of the cluster's batch slots (zeros past the batch or without h_0)
    const int q = i / P, k = i - q * P;
    h_s[i] = (p.h_0 && row_s[q] >= 0) ? p.h_0[((size_t)dir * B + row_s[q]) * P + k] : 0.f;
  }
  __syncthreads();
  ptx::cluster_sync_all();  // peers' barriers are initialised before anyone sends

  int u, b;
  proj_thread<BS>(tid, u, b);
  const int j = j0 + u;
  const int row = row_s[b];
  const bool valid = row >= 0;
  const int len = len_s[b];
  float* gates = p.gates[dir];
  float c = (p.c_0 && valid) ? p.c_0[((size_t)dir * B + row) * H + j] : 0.f;
  float gi[G];
  auto load_gi = [&](int t) {
#pragma unroll
    for (int g = 0; g < G; ++g) gi[g] = valid ? gates[((size_t)t * B + row) * (G * H) + g * H + j] : 0.f;
  };
  if (T > 0) load_gi(dir ? T - 1 : 0);

  for (int step = 0; step <= T; ++step) {
    // ---- h of the previous step: the C partials in rank order; this CTA's columns of y --------------------------
    if (step > 0) {
      const int cur = xb.buf(step);
      const int tp = dir ? T - step : step - 1;
      const uint32_t par = xb.parity(step);
#pragma unroll
      for (int src = 0; src < C; ++src)
        if ((uint32_t)src != rank) xb.wait(cur, src, par);
      const float* sl = slot + (size_t)cur * C * BS * P;
      for (int i = tid; i < BS * P; i += NT) {
        const int q = i / P, k = i - q * P;
        float v = sl[i];
#pragma unroll
        for (int src = 1; src < C; ++src) v += sl[src * BS * P + i];
        const bool frozen = VL && tp >= len_s[q];
        if (!frozen) h_s[i] = v;
        if (k / PC == (int)rank && row_s[q] >= 0 && p.y)
          p.y[(long long)tp * p.y_st + (long long)row_s[q] * p.y_sb + dir * P + k] = frozen ? 0.f : v;
      }
      __syncthreads();
    }
    if (step == T) break;
    const int t = dir ? T - 1 - step : step;
    const int nb = xb.buf(step) ^ 1;
    // this step's partials land in buffer nb; its previous phase was consumed at step - 1
    if (tid == 0) xb.arm(nb, (uint32_t)(BS * P * sizeof(float)));
    // ---- gates, cell, m = o * tanh(c) ----------------------------------------------------------------------------
    float acc[G];
#pragma unroll
    for (int g = 0; g < G; ++g) acc[g] = 0.f;
#pragma unroll 4
    for (int k = 0; k < P; k += 4) {
      const float4 hv = *reinterpret_cast<const float4*>(&h_s[b * P + k]);
#pragma unroll
      for (int g = 0; g < G; ++g) {
        const float4 wv = *reinterpret_cast<const float4*>(&W_s[(g * HS + u) * LD + k]);
        float a = acc[g];
        a = fmaf(wv.x, hv.x, a);
        a = fmaf(wv.y, hv.y, a);
        a = fmaf(wv.z, hv.z, a);
        a = fmaf(wv.w, hv.w, a);
        acc[g] = a;
      }
    }
    const LstmStep st = lstm_cell_fwd(gi, acc, c);
    float cnew = st.c;
    float m = st.h;
    if (VL && t >= len) {
      cnew = c;
      m = 0.f;
    }
    c = cnew;
    m_s[b * HS + u] = valid ? m : 0.f;
    if (valid && p.training) {
      float* gp = gates + ((size_t)t * B + row) * (G * H) + j;
      gp[0] = st.i; gp[H] = st.f; gp[2 * H] = st.g; gp[3 * H] = st.o;
      p.extra[dir][((size_t)t * B + row) * H + j] = cnew;
      p.m[dir][((size_t)t * B + row) * H + j] = m;
    }
    if (step + 1 < T) load_gi(dir ? T - 2 - step : step + 1);
    __syncthreads();
    // ---- this CTA's partial projection into its own slot, then to the peers --------------------------------------
    float* own = slot + ((size_t)nb * C + rank) * BS * P;
    proj_partial<P, BS, Cfg::NG, Cfg::RB, HS>(R_s, LD, m_s, own, tid);
    __syncthreads();
    proj_send<P, C, BS, NT>(own, xb.bar(nb, rank), rank, tid);
  }
  // ---- final state: h_n (this CTA's columns of h_s) and c_n; VL: the steps [T, p.T) the cluster skipped ----------
  for (int i = tid; i < BS * P; i += NT) {
    const int q = i / P, k = i - q * P;
    if (k / PC == (int)rank && row_s[q] >= 0) {
      p.h_n[((size_t)dir * B + row_s[q]) * P + k] = h_s[i];
      if (VL && p.y)
        for (int t = T; t < p.T; ++t) p.y[(long long)t * p.y_st + (long long)row_s[q] * p.y_sb + dir * P + k] = 0.f;
    }
  }
  if (valid) {
    if (p.c_n) p.c_n[((size_t)dir * B + row) * H + j] = c;
    if (VL && p.training)  // the dW_hr GEMM reads m of every step
      for (int t = T; t < p.T; ++t) p.m[dir][((size_t)t * B + row) * H + j] = 0.f;
  }
  ptx::cluster_sync_all();  // nobody exits while a peer could still address its shared memory
}

template <int H, int P, int C, int BS, bool VL>
__global__ void __launch_bounds__(ProjCfg<H, P, C, BS>::NT, 1)
    rec_bwd_proj_kernel(const RecBwdParams p, const int nslices) {
  using Cfg = ProjCfg<H, P, C, BS>;
  constexpr int G = Cfg::G, HS = Cfg::HS, NT = Cfg::NT, LD = Cfg::LD, PC = P / C;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* W_s = reinterpret_cast<float*>(smem_raw);  // [G*HS][LD]
  float* R_s = W_s + Cfg::W_FLOATS;                 // [HS][LD]
  float* dh_s = R_s + Cfg::R_FLOATS;                // [BS][P] dh_t
  float* slot = dh_s + Cfg::V_FLOATS;               // [2][C][BS][P] partials of W_hh^T dgates
  float* dg_s = slot + Cfg::SLOT_FLOATS;            // [BS][G*HS] this CTA's gate gradients
  uint64_t* bars = reinterpret_cast<uint64_t*>(dg_s + BS * G * HS);
  int* row_s = reinterpret_cast<int*>(bars + 2 * C);
  int* len_s = row_s + BS;

  const int tid = threadIdx.x;
  const ClusterSlice cs = cluster_slice<C, BS, HS, VL>(p, nslices);
  const uint32_t rank = cs.rank;
  const int dir = cs.dir, slice = cs.slice, b0 = cs.b0, j0 = cs.j0, T = cs.T;
  const int B = p.B;
  // as in the forward: step s sums the partials step s - 1 sent
  const ExchangeBars<C, 1, true> xb{bars, rank};

  if (tid == 0) {
    xb.init(1u);
    ptx::fence_mbar_init();
  }
  proj_prologue<H, P, C, BS, VL>(p.w_hh[dir], p.w_hr[dir], j0, b0, B, p.T, p.lengths, p.order, W_s, R_s, row_s, len_s,
                                 tid);
  __syncthreads();
  ptx::cluster_sync_all();

  int u, b;
  proj_thread<BS>(tid, u, b);
  const int j = j0 + u;
  const int row = row_s[b];
  const bool valid = row >= 0;
  const int len = len_s[b];
  const float* gates = p.gates[dir];
  const float* extra = p.extra[dir];
  float* dgates = p.dgates[dir];
  float* dhp = p.dhp[dir];
  float dc_carry = (valid && p.dc_n) ? p.dc_n[((size_t)dir * B + row) * H + j] : 0.f;
  float bsum[G];
#pragma unroll
  for (int g = 0; g < G; ++g) bsum[g] = 0.f;
  float sv[G] = {0.f, 0.f, 0.f, 0.f}, sx = 0.f, cp = 0.f;  // saved gates, c_t, c_{t-1} of the current step (prefetched)
  auto load_step = [&](int step) {
    const int t = dir ? step : (T - 1 - step);
    const int tp = dir ? t + 1 : t - 1;
    const size_t o = ((size_t)t * B + row) * H + j;
#pragma unroll
    for (int g = 0; g < G; ++g) sv[g] = gates[((size_t)t * B + row) * (G * H) + g * H + j];
    sx = extra[o];
    if (step < T - 1)
      cp = extra[((size_t)tp * B + row) * H + j];
    else
      cp = p.c_0 ? p.c_0[((size_t)dir * B + row) * H + j] : 0.f;
  };
  if (valid && T > 0) load_step(0);

  for (int step = 0; step <= T; ++step) {
    // ---- dh_t = dy_t + the C partials (rank order); dh_n enters at the first step, dh_0 leaves after the last ----
    const int cur = xb.buf(step);
    if (step > 0) {
      const uint32_t par = xb.parity(step);
#pragma unroll
      for (int src = 0; src < C; ++src)
        if ((uint32_t)src != rank) xb.wait(cur, src, par);
    }
    const int t = dir ? step : (T - 1 - step);
    const float* sl = slot + (size_t)cur * C * BS * P;
    for (int i = tid; i < BS * P; i += NT) {
      const int q = i / P, k = i - q * P;
      const int r = row_s[q];
      float rec;
      if (step == 0) {
        rec = (p.dh_n && r >= 0) ? p.dh_n[((size_t)dir * B + r) * P + k] : 0.f;
      } else {
        rec = sl[i];
#pragma unroll
        for (int src = 1; src < C; ++src) rec += sl[src * BS * P + i];
      }
      const bool mine = k / PC == (int)rank && r >= 0;
      if (step < T) {
        const bool frozen = VL && t >= len_s[q];
        float v = rec;
        if (!frozen && r >= 0 && p.dy) v = p.dy[(long long)t * p.dy_st + (long long)r * p.dy_sb + dir * P + k] + rec;
        dh_s[i] = v;
        if (mine) dhp[((size_t)t * B + r) * P + k] = frozen ? 0.f : v;
      } else if (mine && p.dh_0) {
        p.dh_0[((size_t)dir * B + r) * P + k] = rec;
      }
    }
    __syncthreads();
    if (step == T) break;
    const int nb = xb.buf(step) ^ 1;
    if (tid == 0) xb.arm(nb, (uint32_t)(BS * P * sizeof(float)));
    // ---- dm = W_hr[:, j]^T dh_t, then the LSTM cell backward from dm ---------------------------------------------
    float dm = 0.f;
#pragma unroll 4
    for (int k = 0; k < P; k += 4) {
      const float4 wv = *reinterpret_cast<const float4*>(&R_s[u * LD + k]);
      const float4 dv = *reinterpret_cast<const float4*>(&dh_s[b * P + k]);
      dm = fmaf(wv.x, dv.x, dm);
      dm = fmaf(wv.y, dv.y, dm);
      dm = fmaf(wv.z, dv.z, dm);
      dm = fmaf(wv.w, dv.w, dm);
    }
    const bool frozen = VL && t >= len;
    float dg[G];
    const float dc_next = lstm_cell_bwd(sv, sx, cp, dm, dc_carry, dg);
    if (!frozen) dc_carry = dc_next;  // frozen step: dc passes through
    if (frozen || !valid) {
#pragma unroll
      for (int g = 0; g < G; ++g) dg[g] = 0.f;
    }
#pragma unroll
    for (int g = 0; g < G; ++g) {
      dg_s[b * G * HS + g * HS + u] = dg[g];
      bsum[g] += dg[g];
    }
    if (valid) {
      float* gp = dgates + ((size_t)t * B + row) * (G * H) + j;
#pragma unroll
      for (int g = 0; g < G; ++g) gp[g * H] = dg[g];
    }
    if (valid && step + 1 < T) load_step(step + 1);
    __syncthreads();
    // ---- partial W_hh[units]^T dgates into the own slot (frozen rows: rank 0 carries dh_t), then to the peers ------
    float* own = slot + ((size_t)nb * C + rank) * BS * P;
    proj_partial<P, BS, Cfg::NG, Cfg::RB, G * HS>(W_s, LD, dg_s, own, tid);
    if constexpr (VL) {
      __syncthreads();
      for (int i = tid; i < BS * P; i += NT) {
        const int q = i / P;
        if (t >= len_s[q]) own[i] = rank == 0 ? dh_s[i] : 0.f;
      }
    }
    __syncthreads();
    proj_send<P, C, BS, NT>(own, xb.bar(nb, rank), rank, tid);
  }
  if (valid && p.dc_0) p.dc_0[((size_t)dir * B + row) * H + j] = dc_carry;
  if constexpr (VL) {  // the steps [T, p.T) the cluster skipped: no gate gradient, no dh
    if (valid)
      for (int t = T; t < p.T; ++t) {
        float* gp = dgates + ((size_t)t * B + row) * (G * H) + j;
#pragma unroll
        for (int g = 0; g < G; ++g) gp[g * H] = 0.f;
      }
    for (int i = tid; i < BS * P; i += NT) {
      const int q = i / P, k = i - q * P;
      if (k / PC == (int)rank && row_s[q] >= 0)
        for (int t = T; t < p.T; ++t) dhp[((size_t)t * B + row_s[q]) * P + k] = 0.f;
    }
  }
  // ---- per-slice bias-gradient partials: sum over the slice's batch slots in slot order -------------------------
  __syncthreads();
#pragma unroll
  for (int g = 0; g < G; ++g) dg_s[b * G * HS + g * HS + u] = bsum[g];
  __syncthreads();
  if (b == 0) {
    float* out = p.dbias_part[dir] + (size_t)slice * (G + 1) * H;
#pragma unroll
    for (int g = 0; g < G; ++g) {
      float v = 0.f;
      for (int q = 0; q < BS; ++q) v += dg_s[q * G * HS + g * HS + u];
      out[g * H + j] = v;
    }
    out[G * H + j] = 0.f;
  }
  ptx::cluster_sync_all();
}

// =================================================================================================
// launchers
// =================================================================================================
// Launch config of `nclusters` clusters of C CTAs; `attr` is the storage of the attributes it points to: the cluster
// dimension and, when `programmatic`, programmatic stream serialization (the launch may start while the kernel before
// it in the stream still runs, once every CTA of that kernel has executed griddepcontrol.launch_dependents).
cudaLaunchConfig_t cluster_config(int nclusters, int C, int NT, size_t smem, cudaStream_t s,
                                  cudaLaunchAttribute (&attr)[2], bool programmatic = false) {
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = (unsigned)C;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(nclusters * C), 1, 1);
  cfg.blockDim = dim3((unsigned)NT, 1, 1);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cfg.attrs = attr;
  cfg.numAttrs = programmatic ? 2 : 1;
  return cfg;
}

// Chooses `kernel` as D * ceil(B / BS) clusters of C CTAs if the driver reports them all co-resident, or regardless
// when `force` (then in several waves if they do not fit). Returns false when the config is not taken; true when it is
// (*L describes it, nothing is enqueued yet) or when the capacity query failed (*rc). B200RNN_DEBUG prints one line per
// config considered: "[b200rnn] <desc>: need N clusters, capacity M, smem S".
template <typename P, typename... Args>
bool pick_clustered(void (*kernel)(P, int), const P& p, int C, int BS, int NT, size_t smem, bool force,
                    ClusterLaunch<P>* L, int* rc, const char* desc, Args... desc_args) {
  const int nslices = (p.B + BS - 1) / BS;
  const int nclusters = nslices * p.D;
  int capacity = 0;
  *rc = cluster_capacity((const void*)kernel, C, NT, smem, &capacity);
  if (*rc != B200RNN_OK) return true;
  static const bool debug = getenv("B200RNN_DEBUG") != nullptr;
  if (debug) {
    char what[96];
    snprintf(what, sizeof(what), desc, desc_args...);
    fprintf(stderr, "[b200rnn] %s: need %d clusters, capacity %d, smem %zu\n", what, nclusters, capacity, smem);
  }
  if (!force && nclusters > capacity) return false;
  *L = ClusterLaunch<P>{(const void*)kernel, C, NT, nslices, nclusters, capacity, smem};
  return true;
}

template <typename P>
int launch_clustered(const ClusterLaunch<P>& L, const P& p, int prof_kind, bool programmatic, cudaStream_t s) {
  ProfScope prof(prof_kind, s);
  cudaLaunchAttribute attr[2];
  const cudaLaunchConfig_t cfg = cluster_config(L.nclusters, L.C, L.NT, L.smem, s, attr, programmatic);
  // (P, int) kernels read the first two arguments, the runtime-sized ones all three
  int nslices = L.nslices;
  RecModels models = L.models;
  void* args[3] = {const_cast<P*>(&p), &nslices, &models};
  const cudaError_t e = cudaLaunchKernelExC(&cfg, L.kernel, args);
  if (e != cudaSuccess) {
    set_error("cudaLaunchKernelEx of a recurrence kernel failed: %s", cudaGetErrorString(e));
    return B200RNN_ERR_CUDA;
  }
  count_launch();
  return B200RNN_OK;
}

template <int MODE, int H, int C, int BS, int KL, int UPL, int RG, bool PB = false>
bool pick_fwd(const RecFwdParams& p, bool force, RecFwdLaunch* L, int* rc) {
  using Cfg = RecCfg<MODE, H, C, BS, KL, UPL, RG>;
  static_assert(Cfg::FWD_SMEM <= MAX_SMEM, "forward config does not fit an SM");
  auto k = p.lengths ? rec_fwd_kernel<MODE, H, C, BS, KL, UPL, RG, true, PB>
                     : rec_fwd_kernel<MODE, H, C, BS, KL, UPL, RG, false, PB>;
  return pick_clustered(k, p, C, BS, Cfg::NT, Cfg::FWD_SMEM, force, L, rc,
                        "fwd cfg C=%d BS=%d KL=%d UPL=%d RG=%d PB=%d", C, BS, KL, UPL, RG, (int)PB);
}

// the tensor-core config is the widest-cluster one: it is always taken (several waves when its clusters do not all fit).
// Its contraction: single-pass TF32 in TF32 mode, else fp16 pairs for the no-grad forward of b200rnn_forward_fused
// (no initial state there, see rec_fwd_h16_kernel), else 3xTF32
int pick_fwd_tc(const RecFwdParams& p, RecFwdLaunch* L) {
  using Cfg = TcFwdCfg;
  static_assert(Cfg::SMEM <= MAX_SMEM, "forward config does not fit an SM");
  const bool h16 = !p.tf32 && p.shell_nograd;
  auto k = p.tf32 ? (p.lengths ? rec_fwd_tf32_kernel<true> : rec_fwd_tf32_kernel<false>)
           : h16  ? (p.lengths ? rec_fwd_h16_kernel<true> : rec_fwd_h16_kernel<false>)
                  : (p.lengths ? rec_fwd_tc_kernel<true> : rec_fwd_tc_kernel<false>);
  int rc = B200RNN_OK;
  pick_clustered(k, p, Cfg::C, Cfg::BS, Cfg::NT, Cfg::SMEM, true, L, &rc, "fwd cfg tc8 C=%d BS=%d mma.sync %s",
                 Cfg::C, Cfg::BS, p.tf32 ? "TF32" : h16 ? "f16x3" : "3xTF32");
  return rc;
}

// LSTM-128 on fp16 pairs (lstm_fwd_h16_kernel), the no-grad forward of b200rnn_forward_fused only: 2-CTA clusters of 8
// batch rows, always taken (several waves when its clusters do not all fit)
int pick_fwd_tcl(const RecFwdParams& p, RecFwdLaunch* L) {
  using Cfg = TcLstmCfg;
  static_assert(Cfg::SMEM <= MAX_SMEM, "forward config does not fit an SM");
  int rc = B200RNN_OK;
  pick_clustered(p.lengths ? lstm_fwd_h16_kernel<true> : lstm_fwd_h16_kernel<false>, p, Cfg::C, Cfg::BS, Cfg::NT,
                 Cfg::SMEM, true, L, &rc, "fwd cfg tcl8 C=%d BS=%d mma.sync f16x3", Cfg::C, Cfg::BS);
  return rc;
}

template <int MODE, int H, int C, int BS, int KL, int UPL, int RG>
bool pick_bwd(const RecBwdParams& p, bool force, RecBwdLaunch* L, int* rc) {
  using Cfg = RecCfg<MODE, H, C, BS, KL, UPL, RG>;
  static_assert(Cfg::BWD_SMEM <= MAX_SMEM, "backward config does not fit an SM");
  auto k = p.lengths ? rec_bwd_kernel<MODE, H, C, BS, KL, UPL, RG, true> : rec_bwd_kernel<MODE, H, C, BS, KL, UPL, RG, false>;
  return pick_clustered(k, p, C, BS, Cfg::NT, Cfg::BWD_SMEM, force, L, rc, "bwd cfg C=%d BS=%d KL=%d UPL=%d RG=%d", C,
                        BS, KL, UPL, RG);
}

// LSTM with a projection, forward or backward: one config per (H, P), several waves when its clusters do not all fit
template <int H, int P, int C, int BS, typename Params>
int pick_proj(const Params& p, ClusterLaunch<Params>* L) {
  using Cfg = ProjCfg<H, P, C, BS>;
  static_assert(Cfg::SMEM_F <= MAX_SMEM && Cfg::SMEM_B <= MAX_SMEM, "projected config does not fit an SM");
  int rc = B200RNN_OK;
  if constexpr (std::is_same<Params, RecFwdParams>::value)
    pick_clustered(p.lengths ? rec_fwd_proj_kernel<H, P, C, BS, true> : rec_fwd_proj_kernel<H, P, C, BS, false>, p, C,
                   BS, Cfg::NT, Cfg::SMEM_F, true, L, &rc, "fwd proj cfg C=%d BS=%d P=%d", C, BS, P);
  else
    pick_clustered(p.lengths ? rec_bwd_proj_kernel<H, P, C, BS, true> : rec_bwd_proj_kernel<H, P, C, BS, false>, p, C,
                   BS, Cfg::NT, Cfg::SMEM_B, true, L, &rc, "bwd proj cfg C=%d BS=%d P=%d", C, BS, P);
  return rc;
}

}  // namespace

// smallest BS any backward config uses is 2
int rec_bwd_max_slices(int B) { return (B + 1) / 2; }

int cluster_capacity(const void* kernel, int C, int NT, size_t smem, int* capacity) {
  static std::mutex mu;  // forward and autograd-backward threads both launch
  static std::set<std::pair<const void*, int>> opted_in;
  static std::map<std::tuple<const void*, int, int, int, size_t>, int> cache;
  const int dev = current_device();
  const auto key = std::make_tuple(kernel, dev, C, NT, smem);
  std::lock_guard<std::mutex> lk(mu);
  auto it = cache.find(key);
  if (it == cache.end()) {
    if (!opted_in.count({kernel, dev})) {  // every shape of the kernel may take up to the opt-in limit
      B200_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_SMEM));
      B200_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
      opted_in.insert({kernel, dev});
    }
    cudaLaunchAttribute attr[2];
    const cudaLaunchConfig_t cfg = cluster_config(NUM_SMS, C, NT, smem, 0, attr);
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, kernel, &cfg) != cudaSuccess) {
      cudaGetLastError();  // a failed query leaves its error pending: clear that one, not an older one
      n = 0;
    }
    it = cache.emplace(key, n).first;
  }
  *capacity = it->second;
  return B200RNN_OK;
}

// Candidates are ordered by batch rows per cluster; the first one whose clusters are all co-resident
// (one wave => every sequence advances in lock step) wins, else the widest one runs in several waves.
// Template arguments: <MODE, H, C, BS, KL, UPL, RG>; projected: <H, P, C, BS>, H = 128 on 2-CTA clusters of 4 batch rows
// (256 threads), H = 256 on 4-CTA clusters of 8 batch rows (512 threads).
int plan_rec_fwd(const RecFwdParams& p, RecFwdLaunch* L, int w16, int models) {
  int rc = B200RNN_OK;
  L->kernel = nullptr;
  if (p.B <= 0 || p.T <= 0) return rc;
  if (p.P > 0) {
    if (p.mode == B200RNN_LSTM && p.H == 128 && p.P == 32) return pick_proj<128, 32, 2, 4>(p, L);
    if (p.mode == B200RNN_LSTM && p.H == 128 && p.P == 64) return pick_proj<128, 64, 2, 4>(p, L);
    if (p.mode == B200RNN_LSTM && p.H == 256 && p.P == 64) return pick_proj<256, 64, 4, 8>(p, L);
    if (p.mode == B200RNN_LSTM && p.H == 256 && p.P == 128) return pick_proj<256, 128, 4, 8>(p, L);
    set_error("recurrence: unsupported projection (mode=%d, hidden_size=%d, proj_size=%d); built for the LSTM with "
              "proj_size hidden_size/4 or hidden_size/2", p.mode, p.H, p.P);
    return B200RNN_ERR_UNSUPPORTED;
  }
  // the Elman modes and several models in one launch run the runtime-sized kernels at every hidden size, 128 and 256
  // included (rnn_anyh.cu)
  if (is_elman(p.mode) || models > 1) return plan_anyh_fwd(p, L, w16, models);
  // One config per shape plus a wider-batch fallback that runs in several waves when the batch needs more clusters
  // than fit the chip.
  if (p.mode == B200RNN_GRU && p.H == 256) {
    // 4-CTA clusters of 2, 4 or 8 batch rows; each takes 4 * ceil(B / BS) SMs:
    //   bs2 <4,2,16,8,0>: all three gate blocks in shared memory, 4 warps per CTA
    //   bs4 <4,4,16,4,1> batch-paired (rnn_core.cuh dots_chunk2b): two gate blocks in shared memory, one in registers,
    //       8 warps per CTA
    //   tc8 8 batch rows, the contraction on the tensor cores (rec_fwd_tc_kernel, mma.sync 3xTF32), 8 warps per CTA
    // A cluster cannot span GPCs, and H100 SXM GPCs are floor-swept unevenly, so the number of co-resident 4-CTA clusters
    // (30 on a 132-SM card measured) comes from the driver (pick_clustered), never from the SM count. Measured per layer
    // launch at T = 120 (DESIGN.md): a config in one wave beats the next wider one, and tc8 in one wave beats bs4 in two.
    if (pick_fwd<B200RNN_GRU, 256, 4, 2, 16, 8, 0>(p, false, L, &rc)) return rc;
    if (pick_fwd<B200RNN_GRU, 256, 4, 4, 16, 4, 1, true>(p, false, L, &rc)) return rc;
    // the widest clusters: one wave up to B = 8 x the 4-CTA cluster capacity, several waves beyond
    return pick_fwd_tc(p, L);
  }
  if (p.mode == B200RNN_GRU && p.H == 128) {
    if (pick_fwd<B200RNN_GRU, 128, 2, 4, 16, 4, 1>(p, false, L, &rc)) return rc;
    pick_fwd<B200RNN_GRU, 128, 4, 8, 32, 4, 1>(p, true, L, &rc);
    return rc;
  }
  if (p.mode == B200RNN_LSTM && p.H == 256) {
    // scalar FFMA: the batch-paired form needs more registers than sm_90 leaves this config (it spills)
    if (pick_fwd<B200RNN_LSTM, 256, 4, 4, 16, 4, 1>(p, false, L, &rc)) return rc;
    pick_fwd<B200RNN_LSTM, 256, 8, 8, 16, 2, 1>(p, true, L, &rc);
    return rc;
  }
  if (p.mode == B200RNN_LSTM && p.H == 128) {
    // the no-grad fused forward (no initial state, default precision): fp16 pairs on the tensor cores, half the CTAs
    // of the FFMA config below at the same batch
    if (p.shell_nograd && !p.tf32) return pick_fwd_tcl(p, L);
    // scalar FFMA
    if (pick_fwd<B200RNN_LSTM, 128, 2, 4, 16, 4, 1>(p, false, L, &rc)) return rc;
    pick_fwd<B200RNN_LSTM, 128, 4, 8, 16, 2, 1>(p, true, L, &rc);
    return rc;
  }
  // every other hidden size: the runtime-sized kernels of rnn_anyh.cu
  if (anyh_hidden_size(p.H)) return plan_anyh_fwd(p, L, w16);
  set_error("recurrence: unsupported (mode=%d, hidden_size=%d); built for hidden_size 128 and 256", p.mode,
            p.H);
  return B200RNN_ERR_UNSUPPORTED;
}

// The same rule and projected configs as the forward
int plan_rec_bwd(const RecBwdParams& p, RecBwdLaunch* L, int w16, int models) {
  int rc = B200RNN_OK;
  L->kernel = nullptr;
  if (p.B <= 0 || p.T <= 0) return rc;
  if (p.P > 0) {
    if (p.mode == B200RNN_LSTM && p.H == 128 && p.P == 32) return pick_proj<128, 32, 2, 4>(p, L);
    if (p.mode == B200RNN_LSTM && p.H == 128 && p.P == 64) return pick_proj<128, 64, 2, 4>(p, L);
    if (p.mode == B200RNN_LSTM && p.H == 256 && p.P == 64) return pick_proj<256, 64, 4, 8>(p, L);
    if (p.mode == B200RNN_LSTM && p.H == 256 && p.P == 128) return pick_proj<256, 128, 4, 8>(p, L);
    set_error("recurrence backward: unsupported projection (mode=%d, hidden_size=%d, proj_size=%d)", p.mode, p.H, p.P);
    return B200RNN_ERR_UNSUPPORTED;
  }
  if (is_elman(p.mode) || models > 1) return plan_anyh_bwd(p, L, w16, models);
  // K across all 32 lanes with 8 units per lane halves the redundant reads of the [BS][G*H] gradient vector, which
  // (not the weights) dominates the shared-memory traffic of the backward contraction
  if (p.mode == B200RNN_GRU && p.H == 256) {
    if (pick_bwd<B200RNN_GRU, 256, 4, 2, 16, 8, 0>(p, false, L, &rc)) return rc;
    if (pick_bwd<B200RNN_GRU, 256, 4, 4, 32, 8, 1>(p, false, L, &rc)) return rc;
    pick_bwd<B200RNN_GRU, 256, 8, 8, 32, 4, 1>(p, true, L, &rc);
    return rc;
  }
  if (p.mode == B200RNN_GRU && p.H == 128) {
    if (pick_bwd<B200RNN_GRU, 128, 2, 4, 32, 8, 1>(p, false, L, &rc)) return rc;
    pick_bwd<B200RNN_GRU, 128, 4, 8, 32, 4, 1>(p, true, L, &rc);
    return rc;
  }
  if (p.mode == B200RNN_LSTM && p.H == 256) {
    if (pick_bwd<B200RNN_LSTM, 256, 4, 4, 32, 8, 1>(p, false, L, &rc)) return rc;
    pick_bwd<B200RNN_LSTM, 256, 8, 8, 32, 4, 1>(p, true, L, &rc);
    return rc;
  }
  if (p.mode == B200RNN_LSTM && p.H == 128) {
    if (pick_bwd<B200RNN_LSTM, 128, 2, 4, 32, 8, 1>(p, false, L, &rc)) return rc;
    pick_bwd<B200RNN_LSTM, 128, 4, 8, 32, 4, 1>(p, true, L, &rc);
    return rc;
  }
  if (anyh_hidden_size(p.H)) return plan_anyh_bwd(p, L, w16);
  set_error("recurrence backward: unsupported (mode=%d, hidden_size=%d)", p.mode, p.H);
  return B200RNN_ERR_UNSUPPORTED;
}

int prep_whh_h16(const float* w_hh, void* img, cudaStream_t s) {
  using L = h16::Gru256;
  whh_h16_prep_kernel<<<L::G * L::H / 8, 256, 0, s>>>(w_hh, static_cast<unsigned char*>(img));
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

int launch_rec_fwd(const RecFwdLaunch& L, const RecFwdParams& p, cudaStream_t s) {
  if (p.B <= 0 || p.T <= 0) return B200RNN_OK;
  if (p.ready && p.D != 1) {  // GiReady walks the row tiles in increasing t
    set_error("recurrence: a streamed x-projection needs a unidirectional layer");
    return B200RNN_ERR_INVALID;
  }
  if (p.shell_nograd && p.h_0) {  // the fp16-pair state scale assumes |h| <= 1
    set_error("recurrence: the no-grad fused forward takes no initial state");
    return B200RNN_ERR_INVALID;
  }
  if (L.anyh && (p.ready || p.y_pool || p.shell_nograd)) {
    set_error("recurrence: hidden_size %d takes no streamed x-projection, y_pool or no-grad fused forward", p.H);
    return B200RNN_ERR_UNSUPPORTED;
  }
  return launch_clustered(L, p, PROF_REC_FWD, p.ready != nullptr, s);
}

int launch_rec_tangent(const RecTanParams& p, int directions, cudaStream_t s) {
  if (p.B <= 0 || p.T <= 0) return B200RNN_OK;
  RecTanLaunch L;
  const int rc = plan_anyh_tangent(p, &L, directions);
  if (rc != B200RNN_OK) return rc;
  return launch_clustered(L, p, PROF_REC_FWD, false, s);
}

namespace {

// The backward's W_hh for a C-CTA cluster, transposed and contiguous per CTA: CTA r's block starts at G * j0_r * H and
// holds out[G*j0_r*H + (g*n_r + u)*H + jj] = W_hh[g*H + jj][j0_r + u] (anyh_units). For the fixed configs (C divides
// H / 8) this is the [C ranks][G][H / C][H] layout rec_bwd_kernel copies with TMA.
template <typename T>
__device__ __forceinline__ void whh_prep_body(const T* __restrict__ w_hh, T* __restrict__ out, int G, int H, int C) {
  __shared__ T tile[32][33];
  const int nt = (H + 31) / 32;
  for (int tix = blockIdx.x; tix < G * nt * nt; tix += gridDim.x) {
    const int g = tix / (nt * nt), rem = tix - g * nt * nt;
    const int tj = rem / nt, tk = rem - tj * nt;  // row tile of the gate block, column tile
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
      const int r = tj * 32 + i, k = tk * 32 + threadIdx.x;
      tile[i][threadIdx.x] = (r < H && k < H) ? w_hh[((size_t)g * H + r) * H + k] : T(0);
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

__global__ void whh_prep_kernel(const float* __restrict__ w_hh, float* __restrict__ out, int G, int H, int C) {
  whh_prep_body<float>(w_hh, out, G, H, C);
}

// the same transpose of a 16-bit weight_hh, bit for bit (the 16-bit runtime-sized backward stages it as it lies)
__global__ void whh_prep16_kernel(const uint16_t* __restrict__ w_hh, uint16_t* __restrict__ out, int G, int H, int C) {
  whh_prep_body<uint16_t>(w_hh, out, G, H, C);
}

}  // namespace

int launch_rec_bwd(RecBwdParams& p, cudaStream_t s, int w16, const void* const* whh16, const RecModels* models) {
  RecBwdLaunch L;
  if (!whh16) w16 = 0;
  const int rc = plan_rec_bwd(p, &L, w16, models ? models->M : 1);
  if (rc != B200RNN_OK || L.kernel == nullptr) return rc;
  if (models) L.models = *models;
  const RecModels& ms = L.models;
  if (p.P == 0) {  // the unprojected kernels read W_hh transposed for the chosen cluster width
    for (int d = 0; d < p.D; ++d)
      for (int m = 0; m < ms.M; ++m) {  // once per distinct weight_hh: a shared one once
        if (m > 0 && ms.whh[d] == 0) break;
        if (L.anyh && w16)
          whh_prep16_kernel<<<NUM_SMS, dim3(32, 8), 0, s>>>(static_cast<const uint16_t*>(whh16[d]),
                                                            reinterpret_cast<uint16_t*>(p.w_prep[d]), gates_of(p.mode),
                                                            p.H, L.C);
        else
          whh_prep_kernel<<<NUM_SMS, dim3(32, 8), 0, s>>>(p.w_hh[d] + m * ms.whh[d], p.w_prep[d] + m * ms.wprep[d],
                                                          gates_of(p.mode), p.H, L.C);
        if (cudaGetLastError() != cudaSuccess) {
          set_error("whh_prep launch failed");
          return B200RNN_ERR_CUDA;
        }
        count_launch();
      }
  }
  p.nslices_out = L.nslices;
  return launch_clustered(L, p, PROF_REC_BWD, false, s);
}

}  // namespace b200rnn
