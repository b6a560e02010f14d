// cell.cu — one-step GRUCell / LSTMCell / RNNCell kernels for sm_90a (torch.nn.GRUCell / LSTMCell / RNNCell, rnn.py).
//
// Forward, cell_fwd_kernel, one launch per call:
//   * a CTA owns UNITS = 16 hidden units with all G gate rows of them (one m16 tile per gate) and NB = 8 * ntn batch
//     rows (ntn n-tiles of 8), so the whole cell epilogue stays in the CTA: lane (g, t) of the mma accumulator fragment
//     holds units g, g + 8 for batch rows 2t, 2t + 1 of every gate, and applies the cell to those 4 outputs.
//   * the contraction over K = I + H runs on the tensor cores, warp-level mma.sync m16n8k8 with N = 8 batch rows per
//     n-tile as in tc8 (rnn_rec.cu): 3xTF32 (ptx::split_tf32, hi*hi and the two cross terms on their own accumulators),
//     or single-pass TF32 on operands rounded to nearest (B200RNN_FLAG_TF32). The x-part and the h-part have separate
//     accumulators (the GRU's n gate needs W_hn h + b_hn alone). Each tensor-core chain restarts at every ring stage,
//     at most 4 hi*hi or 8 cross-term MMAs long: within the 12 MMAs gemm_tc.cu allows.
//   * the weights are not resident: W_ih, then W_hh, and the matching columns of x and h are streamed through an
//     NSTAGE-deep shared-memory ring of KC-wide k-slices with cp.async (L2 after the first call). Rows that are not
//     16-byte aligned take 4-byte copies; rows past H or B and columns past K are zero-filled, nothing is read past a
//     row. Without h (hx = None) the W_hh half is skipped.
//   * 4 warps: ntn of them own one n-tile each, the other warps split the k-steps of every stage with them (small
//     batches stream the weights with all 4 warps); their partial sums meet in shared memory in a fixed order.
// Backward, cell_bwd_kernel: one elementwise pass over the saved gates (the gradient GEMMs run in api.cu).
// RNNCell: elman_cell_fwd_kernel runs the same step (cell_fwd) with one gate tile and saves h' alone;
// elman_cell_bwd_kernel is its elementwise backward (dpre from the saved h').
#include "cell_kernels.cuh"
#include "profile.cuh"
#include "ptx.cuh"
#include "rnn_cell.cuh"

namespace b200rnn {

namespace {

constexpr int UNITS = 16;                // hidden units per CTA: one m16 tile per gate
constexpr int NWARP = 4, NT = NWARP * 32;
constexpr int KC = 32;                   // k per ring stage: 4 k-steps of 8
constexpr int KSTEPS = KC / 8;
constexpr int LDS = KC + 4;              // row pitch (floats): conflict-free fragment loads, 16-byte aligned rows
constexpr int NSTAGE = 3;
constexpr int A_ROWS = 4 * UNITS;        // G * UNITS weight rows (LSTM)
constexpr int B_ROWS = 8 * NWARP;        // up to one n-tile per warp
constexpr int STAGE_FLOATS = (A_ROWS + B_ROWS) * LDS;
constexpr size_t FWD_SMEM = (size_t)NSTAGE * STAGE_FLOATS * sizeof(float);
static_assert(FWD_SMEM <= 48 * 1024, "the ring fits the default dynamic shared-memory limit");
static_assert(NWARP * 2 * 4 * 4 * 32 <= NSTAGE * STAGE_FLOATS, "the k-split partial sums fit the ring");
constexpr int BWD_ROWS = 32;             // batch rows per slice of the backward's bias partial sums

__device__ __forceinline__ float round_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

// Stage rows [0, nrows) x columns [k0, k0 + KC) of an operand into dst (pitch LDS): row r is src + row(r) * ld, or
// zeros when row(r) < 0; columns at or past K are zeros. vec: src and ld allow 16-byte copies.
template <typename RowFn>
__device__ __forceinline__ void stage_rows(float* dst, const float* src, long long ld, int nrows, RowFn row, int k0,
                                           int K, bool vec, int tid) {
  if (vec) {
    for (int i = tid; i < nrows * (KC / 4); i += NT) {
      const int r = i / (KC / 4), k = k0 + (i % (KC / 4)) * 4;
      const long long gr = row(r);
      const uint32_t bytes = (gr >= 0 && k < K) ? 4u * (uint32_t)min(4, K - k) : 0u;
      ptx::cp_async16(dst + r * LDS + (k - k0), bytes ? src + gr * ld + k : src, bytes);
    }
  } else {
    for (int i = tid; i < nrows * KC; i += NT) {
      const int r = i / KC, k = k0 + i % KC;
      const long long gr = row(r);
      const uint32_t bytes = (gr >= 0 && k < K) ? 4u : 0u;
      ptx::cp_async4(dst + r * LDS + (k - k0), bytes ? src + gr * ld + k : src, bytes);
    }
  }
}

__device__ __forceinline__ bool vec_rows(const float* p, long long ld) {
  return (reinterpret_cast<uintptr_t>(p) & 15u) == 0 && ld % 4 == 0;
}

// One cell step of the CTA's units and batch rows, the body of cell_fwd_kernel and elman_cell_fwd_kernel. MODE
// B200RNN_RNN_TANH stands for both Elman modes: the nonlinearity is read from p.mode (warp-uniform).
template <int MODE, bool TF32>
__device__ __forceinline__ void cell_fwd(const CellFwdParams& p, const int ntn) {
  constexpr int G = gates_of(MODE);
  extern __shared__ __align__(16) float smem[];
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int kw = NWARP / ntn;              // warps per n-tile, splitting the k-steps of a stage
  const int nt = w % ntn, kslice = w / ntn;
  const int j0 = blockIdx.x * UNITS, b0 = blockIdx.y * 8 * ntn;
  const int H = p.H;
  const int nq_x = (p.I + KC - 1) / KC;
  const int nq = nq_x + (p.h ? (H + KC - 1) / KC : 0);
  const bool vec_wih = vec_rows(p.w_ih, p.I), vec_whh = vec_rows(p.w_hh, H);
  const bool vec_x = vec_rows(p.x, p.x_ld), vec_h = p.h && vec_rows(p.h, p.h_ld);

  // ring stage q: k-slice q of [x | h] against the same k-slice of [W_ih | W_hh]
  auto load_stage = [&](int q) {
    float* As = smem + (q % NSTAGE) * STAGE_FLOATS;
    float* Bs = As + A_ROWS * LDS;
    const bool xp = q < nq_x;
    const int K = xp ? p.I : H, k0 = (xp ? q : q - nq_x) * KC;
    stage_rows(As, xp ? p.w_ih : p.w_hh, K, G * UNITS,
               [&](int r) { return j0 + r % UNITS < H ? (long long)(r / UNITS) * H + j0 + r % UNITS : -1LL; }, k0, K,
               xp ? vec_wih : vec_whh, tid);
    stage_rows(Bs, xp ? p.x : p.h, xp ? p.x_ld : p.h_ld, 8 * ntn,
               [&](int r) { return b0 + r < p.B ? (long long)(b0 + r) : -1LL; }, k0, K, xp ? vec_x : vec_h, tid);
  };

  const int fg = lane >> 2, ft = lane & 3;
  float accx[G][4], acch[G][4];
#pragma unroll
  for (int g = 0; g < G; ++g)
#pragma unroll
    for (int i = 0; i < 4; ++i) accx[g][i] = acch[g][i] = 0.f;

#pragma unroll
  for (int s = 0; s < NSTAGE - 1; ++s) {
    if (s < nq) load_stage(s);
    ptx::cp_async_commit();
  }
  for (int q = 0; q < nq; ++q) {
    ptx::cp_async_wait<NSTAGE - 2>();
    __syncthreads();  // stage q has landed for every thread; stage q - 1's slot is free again
    if (q + NSTAGE - 1 < nq) load_stage(q + NSTAGE - 1);
    ptx::cp_async_commit();
    const float* As = smem + (q % NSTAGE) * STAGE_FLOATS + fg * LDS + ft;
    const float* Bs = smem + (q % NSTAGE) * STAGE_FLOATS + (A_ROWS + nt * 8 + fg) * LDS + ft;
    float d[G][2][4];  // [gate tile][lo*hi + hi*lo, hi*hi]; TF32: [gate tile][-, the single product]
#pragma unroll
    for (int g = 0; g < G; ++g)
#pragma unroll
      for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int i = 0; i < 4; ++i) d[g][m][i] = 0.f;
    for (int ks = kslice; ks < KSTEPS; ks += kw) {
      const float bv[2] = {Bs[ks * 8], Bs[ks * 8 + 4]};
#pragma unroll
      for (int g = 0; g < G; ++g) {
        const float* ap = As + g * UNITS * LDS + ks * 8;
        const float av[4] = {ap[0], ap[8 * LDS], ap[4], ap[8 * LDS + 4]};
        if constexpr (TF32) {
          const uint32_t a[4] = {__float_as_uint(round_tf32(av[0])), __float_as_uint(round_tf32(av[1])),
                                 __float_as_uint(round_tf32(av[2])), __float_as_uint(round_tf32(av[3]))};
          const uint32_t b[2] = {__float_as_uint(round_tf32(bv[0])), __float_as_uint(round_tf32(bv[1]))};
          ptx::mma_tf32_m16n8k8(d[g][1], a, b);
        } else {
          uint32_t ah[4], al[4], bh[2], bl[2];
#pragma unroll
          for (int e = 0; e < 4; ++e) ptx::split_tf32(av[e], ah[e], al[e]);
#pragma unroll
          for (int e = 0; e < 2; ++e) ptx::split_tf32(bv[e], bh[e], bl[e]);
          ptx::mma_tf32_m16n8k8(d[g][0], al, bh);
          ptx::mma_tf32_m16n8k8(d[g][0], ah, bl);
          ptx::mma_tf32_m16n8k8(d[g][1], ah, bh);
        }
      }
    }
    if (q < nq_x) {
#pragma unroll
      for (int g = 0; g < G; ++g)
#pragma unroll
        for (int i = 0; i < 4; ++i) accx[g][i] += TF32 ? d[g][1][i] : d[g][0][i] + d[g][1][i];
    } else {
#pragma unroll
      for (int g = 0; g < G; ++g)
#pragma unroll
        for (int i = 0; i < 4; ++i) acch[g][i] += TF32 ? d[g][1][i] : d[g][0][i] + d[g][1][i];
    }
  }
  ptx::cp_async_wait<0>();
  __syncthreads();  // the ring is free: it holds the k-split partial sums

  if (kw > 1) {
    float* red = smem;  // [warp - ntn][2 * G * 4 values][32 lanes]
    if (kslice > 0) {
      float* mine = red + (w - ntn) * 2 * G * 4 * 32 + lane;
#pragma unroll
      for (int g = 0; g < G; ++g)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          mine[(g * 4 + i) * 32] = accx[g][i];
          mine[((G + g) * 4 + i) * 32] = acch[g][i];
        }
    }
    __syncthreads();
    if (kslice > 0) return;
    for (int k = 1; k < kw; ++k) {  // fixed order: deterministic
      const float* part = red + ((k - 1) * ntn + nt) * 2 * G * 4 * 32 + lane;
#pragma unroll
      for (int g = 0; g < G; ++g)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          accx[g][i] += part[(g * 4 + i) * 32];
          acch[g][i] += part[((G + g) * 4 + i) * 32];
        }
    }
  }

  // ---- cell epilogue: accumulator element i is unit fg + 8 * (i / 2), batch row 2 * ft + i % 2 of the n-tile --------
  const size_t GH = (size_t)G * H;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int j = j0 + fg + 8 * (i >> 1), b = b0 + nt * 8 + 2 * ft + (i & 1);
    if (j >= H || b >= p.B) continue;
    float gi[G], pre[G], bhn = 0.f;
#pragma unroll
    for (int g = 0; g < G; ++g) {
      const float bi = p.b_ih ? p.b_ih[g * H + j] : 0.f;
      const float bh = p.b_hh ? p.b_hh[g * H + j] : 0.f;
      // as the sequence path's input projection folds them: b_ih, and b_hh except the GRU's n block
      const bool fold = MODE != B200RNN_GRU || g < 2;
      gi[g] = fold ? accx[g][i] + bi + bh : accx[g][i] + bi;
      if (!fold) bhn = bh;
      pre[g] = acch[g][i];
    }
    float* gp = p.gates ? p.gates + (size_t)b * GH + j : nullptr;
    if constexpr (MODE == B200RNN_GRU) {
      const float hp = p.h ? p.h[(long long)b * p.h_ld + j] : 0.f;
      const GruStep st = gru_cell_fwd(gi, pre, bhn, hp);
      p.h_out[(size_t)b * H + j] = st.h;
      if (gp) {
        gp[0] = st.r; gp[H] = st.z; gp[2 * H] = st.n;
        p.extra[(size_t)b * H + j] = st.hn;
      }
    } else if constexpr (MODE == B200RNN_LSTM) {
      const float cp = p.c ? p.c[(long long)b * p.c_ld + j] : 0.f;
      const LstmStep st = lstm_cell_fwd(gi, pre, cp);
      p.h_out[(size_t)b * H + j] = st.h;
      p.c_out[(size_t)b * H + j] = st.c;
      if (gp) {
        gp[0] = st.i; gp[H] = st.f; gp[2 * H] = st.g; gp[3 * H] = st.o;
        p.extra[(size_t)b * H + j] = st.c;
      }
    } else {  // Elman: h' alone is saved
      const float h = elman_cell_fwd(gi[0], pre[0], p.mode == B200RNN_RNN_RELU);
      p.h_out[(size_t)b * H + j] = h;
      if (gp) gp[0] = h;
    }
  }
}

template <int MODE, bool TF32>
__global__ void __launch_bounds__(NT) cell_fwd_kernel(const CellFwdParams p, const int ntn) {
  cell_fwd<MODE, TF32>(p, ntn);
}

// RNNCell, tanh or relu (p.mode)
template <bool TF32>
__global__ void __launch_bounds__(NT) elman_cell_fwd_kernel(const CellFwdParams p, const int ntn) {
  cell_fwd<B200RNN_RNN_TANH, TF32>(p, ntn);
}

// thread = unit j of slice blockIdx.y (BWD_ROWS batch rows), rows in increasing order: the bias partial sums are
// deterministic
template <int MODE>
__global__ void __launch_bounds__(128) cell_bwd_kernel(const CellBwdParams p) {
  constexpr int G = MODE == B200RNN_GRU ? 3 : 4;
  const int H = p.H, j = blockIdx.x * 128 + threadIdx.x;
  if (j >= H) return;
  const size_t GH = (size_t)G * H;
  const int slice = blockIdx.y, bend = min(p.B, (slice + 1) * BWD_ROWS);
  float bsum[G + 1];
#pragma unroll
  for (int g = 0; g <= G; ++g) bsum[g] = 0.f;
  for (int b = slice * BWD_ROWS; b < bend; ++b) {
    float sv[G], dg[G], dhn = 0.f, direct;
    const float* gp = p.gates + (size_t)b * GH + j;
#pragma unroll
    for (int g = 0; g < G; ++g) sv[g] = gp[g * H];
    const float sx = p.extra[(size_t)b * H + j];
    const float dh = p.dh_out ? p.dh_out[(size_t)b * H + j] : 0.f;
    if constexpr (MODE == B200RNN_GRU) {
      const float hp = p.h ? p.h[(long long)b * p.h_ld + j] : 0.f;
      direct = gru_cell_bwd(sv, sx, hp, dh, dg, dhn);
    } else {
      const float cp = p.c ? p.c[(long long)b * p.c_ld + j] : 0.f;
      const float dc = p.dc_out ? p.dc_out[(size_t)b * H + j] : 0.f;
      direct = lstm_cell_bwd(sv, sx, cp, dh, dc, dg);
    }
#pragma unroll
    for (int g = 0; g < G; ++g) {
      p.dg_x[(size_t)b * GH + g * H + j] = dg[g];
      if (MODE == B200RNN_GRU) p.dg_h[(size_t)b * GH + g * H + j] = g == 2 ? dhn : dg[g];
      bsum[g] += dg[g];
    }
    bsum[G] += dhn;
    if (p.direct) p.direct[(size_t)b * H + j] = direct;
  }
  float* part = p.part + (size_t)slice * (G + 1) * H + j;
#pragma unroll
  for (int g = 0; g <= G; ++g) part[g * H] = bsum[g];
}

// thread = unit j of slice blockIdx.y (BWD_ROWS batch rows), rows in increasing order; part is [slices][H]
__global__ void __launch_bounds__(128) elman_cell_bwd_kernel(const CellBwdParams p) {
  const int H = p.H, j = blockIdx.x * 128 + threadIdx.x;
  if (j >= H) return;
  const bool relu = p.mode == B200RNN_RNN_RELU;
  const int slice = blockIdx.y, bend = min(p.B, (slice + 1) * BWD_ROWS);
  float bsum = 0.f;
  for (int b = slice * BWD_ROWS; b < bend; ++b) {
    const float dh = p.dh_out ? p.dh_out[(size_t)b * H + j] : 0.f;
    const float dg = elman_cell_bwd(p.gates[(size_t)b * H + j], dh, relu);
    p.dg_x[(size_t)b * H + j] = dg;
    bsum += dg;
  }
  p.part[(size_t)slice * H + j] = bsum;
}

}  // namespace

int launch_cell_fwd(const CellFwdParams& p, cudaStream_t stream) {
  ProfScope prof(PROF_MISC, stream);
  const int ntn = p.B <= 8 ? 1 : p.B <= 16 ? 2 : 4;
  const dim3 grid((p.H + UNITS - 1) / UNITS, (p.B + 8 * ntn - 1) / (8 * ntn));
  const bool gru = p.mode == B200RNN_GRU;
  void (*k)(const CellFwdParams, int) =
      is_elman(p.mode) ? (p.tf32 ? elman_cell_fwd_kernel<true> : elman_cell_fwd_kernel<false>)
      : gru            ? (p.tf32 ? cell_fwd_kernel<B200RNN_GRU, true> : cell_fwd_kernel<B200RNN_GRU, false>)
                       : (p.tf32 ? cell_fwd_kernel<B200RNN_LSTM, true> : cell_fwd_kernel<B200RNN_LSTM, false>);
  k<<<grid, NT, FWD_SMEM, stream>>>(p, ntn);
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

int cell_bwd_slices(int B) { return (B + BWD_ROWS - 1) / BWD_ROWS; }

int launch_cell_bwd(const CellBwdParams& p, cudaStream_t stream) {
  ProfScope prof(PROF_MISC, stream);
  const dim3 grid((p.H + 127) / 128, cell_bwd_slices(p.B));
  if (is_elman(p.mode))
    elman_cell_bwd_kernel<<<grid, 128, 0, stream>>>(p);
  else if (p.mode == B200RNN_GRU)
    cell_bwd_kernel<B200RNN_GRU><<<grid, 128, 0, stream>>>(p);
  else
    cell_bwd_kernel<B200RNN_LSTM><<<grid, 128, 0, stream>>>(p);
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

}  // namespace b200rnn
