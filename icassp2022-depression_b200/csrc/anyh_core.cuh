// anyh_core.cuh — the cluster slice, exchange protocol and contraction shared by the runtime-sized recurrence kernels:
// the GRU / LSTM ones of rnn_anyh.cu and the Elman ones of rnn_elman.cu (DESIGN.md §4 "Every other hidden size").
#pragma once
#include <stdint.h>

#include "ptx.cuh"
#include "rnn_kernels.cuh"

namespace b200rnn {

template <typename P>
using AnyhKernel = void (*)(P, int);
// the Elman kernels of one launch shape (rnn_elman.cu): ragged or not, W_hh on chip or read from L2
AnyhKernel<RecFwdParams> elman_kernel(const RecFwdParams&, bool vl, bool onchip);
AnyhKernel<RecBwdParams> elman_kernel(const RecBwdParams&, bool vl, bool onchip);

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

// The units of CTA r of a C-CTA cluster: the H / 8 groups of 8 units split as evenly as possible, [j0, j0 + n). Every
// CTA owns at least one group when C <= H / 8; a slice of a state row is a whole number of 16-byte chunks.
__host__ __device__ __forceinline__ void anyh_units(int H, int C, int r, int& j0, int& n) {
  const int g = H / 8, a = r * g / C, e = (r + 1) * g / C;
  j0 = 8 * a;
  n = 8 * (e - a);
}
__host__ __device__ __forceinline__ int anyh_max_units(int H, int C) { return 8 * ((H / 8 + C - 1) / C); }

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
  const int cid = blockIdx.x / s.C;
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
// tier, from global memory (read-only for the whole launch)
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

}  // namespace b200rnn
