// rnn_core.cuh — the per-step contraction shared by the persistent forward and backward kernels.
//
// A warp multiplies UPW = CL*UPL rows of a weight slice (row-major, length KLEN) per row-group with BS vectors
// of length KLEN that sit in shared memory. Its 32 lanes form a CL x KL grid: the KL "k-lanes" split the
// contraction dimension (each owns 4 consecutive k per 4*KL-wide chunk, so every shared-memory read is a
// conflict-free 16-byte load), the CL "column-lanes" own different rows. The cross-lane sum over the KL lanes is
// a transposing butterfly: every stage halves the number of live partial sums per lane (UPL*BS == KL, so exactly
// one sum per row-group is left per lane), i.e. about one SHFL+FADD per accumulator instead of log2(KL).
//
// To keep every register index static, the *data* a register slot holds is permuted per lane:
//   slot (au, ab) of k-lane kl accumulates   unit = au ^ p(kl),  batch = ab ^ q(kl)
// with p = the top log2(UPL) bits of kl and q = its low log2(BS) bits. Row / vector addresses are computed per
// lane (free: rows differ by multiples of KLEN floats, i.e. the same banks), and each butterfly stage becomes
// "slot[i] += shfl_xor(slot[i + half])" with compile-time i.
//
// The last RG row-groups can be register resident (loaded once per kernel): they cost no shared-memory
// bandwidth in the time loop, which is what bounds the loop once the FFMA pipe is fed.
#pragma once
#include "common.cuh"

namespace b200rnn {

template <int V>
struct Log2 {
  static constexpr int value = 1 + Log2<V / 2>::value;
};
template <>
struct Log2<1> {
  static constexpr int value = 0;
};

template <int KL, int UPL, int BS>
struct LaneMap {
  static constexpr int LK = Log2<KL>::value;
  static constexpr int LU = Log2<UPL>::value;
  static constexpr int LB = Log2<BS>::value;
  static_assert((1 << LK) == KL && (1 << LU) == UPL && (1 << LB) == BS, "KL, UPL, BS must be powers of two");
  static_assert(UPL * BS == KL && KL <= 32, "one reduced value per lane needs UPL*BS == KL <= 32");
  static constexpr int CL = 32 / KL;     // column-lanes
  static constexpr int UPW = CL * UPL;   // rows (units) per warp and row-group
  __device__ static __forceinline__ int kl(int lane) { return lane & (KL - 1); }
  __device__ static __forceinline__ int cl(int lane) { return lane >> LK; }
  __device__ static __forceinline__ int p(int lane) { return kl(lane) >> LB; }
  __device__ static __forceinline__ int q(int lane) { return lane & (BS - 1); }
  // unit (within the warp) and batch (within the slice) this lane owns after the butterfly
  __device__ static __forceinline__ int unit(int lane) { return cl(lane) * UPL + p(lane); }
  // lane that owns (unit u of the warp, batch b)
  __device__ static __forceinline__ int lane_of(int u, int b) {
    return ((u >> LU) << LK) | ((u & (UPL - 1)) << LB) | b;
  }
};

// The contraction dimension is processed in chunks of CW = 4*KL floats. `rot` rotates the chunk order per CTA
// (chunk c of the loop works on actual chunk ca = (c + rot) % NCH) so that a CTA starts with the slice of the
// state vector it produced itself while its peers' slices are still in flight; register-resident weights are
// loaded in that rotated order, so their register indices stay compile-time constants.

// Load the register-resident row-groups: wreg[r][au][c*4 + e] = W[row][ca*CW + kl*4 + e].
//   Wg : global weight matrix, row-major, leading dimension KLEN; row of (group r, unit u) = grow0 + r*gstride + u
template <int RG, int KL, int UPL, int BS, int KLEN>
__device__ __forceinline__ void load_resident(const float* __restrict__ Wg, long long gstride_rows, long long grow0,
                                              int rot, int lane, float (&wreg)[RG > 0 ? RG : 1][UPL][KLEN / KL]) {
  using LM = LaneMap<KL, UPL, BS>;
  constexpr int NCH = KLEN / (4 * KL);
  const int kl = LM::kl(lane), p = LM::p(lane), cgrp = LM::cl(lane);
#pragma unroll
  for (int r = 0; r < RG; ++r)
#pragma unroll
    for (int au = 0; au < UPL; ++au) {
      const float* row = Wg + (grow0 + (long long)r * gstride_rows + cgrp * UPL + (au ^ p)) * KLEN;
#pragma unroll
      for (int c = 0; c < NCH; ++c) {
        const int ca = (c + rot) % NCH;
        const float4 v = __ldg(reinterpret_cast<const float4*>(row + ca * 4 * KL + kl * 4));
        wreg[r][au][c * 4 + 0] = v.x;
        wreg[r][au][c * 4 + 1] = v.y;
        wreg[r][au][c * 4 + 2] = v.z;
        wreg[r][au][c * 4 + 3] = v.w;
      }
    }
}

// One chunk of the contraction:
//   acc[r][au][ab] += sum_{k in chunk ca, this lane} W[row(r, au^p)][k] * vec[ab^q][k]
//   W_s   : shared-memory weights of the first NR-RG row-groups, row-major [.][KLEN];
//           row of (group r, unit u of this warp) = r*group_stride + row0 + u
//   wreg  : the last RG row-groups, register resident (see load_resident), indexed by the LOOP chunk index c
//   vec_s : BS vectors, VSTRIDE floats apart
template <int NR, int RG, int KL, int UPL, int BS, int KLEN, int VSTRIDE>
__device__ __forceinline__ void dots_chunk(const float* __restrict__ W_s, int group_stride, int row0,
                                           const float (&wreg)[RG > 0 ? RG : 1][UPL][KLEN / KL],
                                           const float* __restrict__ vec_s, int c, int ca, int lane,
                                           float (&acc)[NR][UPL][BS]) {
  using LM = LaneMap<KL, UPL, BS>;
  static_assert(KLEN % (4 * KL) == 0, "contraction length must be a multiple of 4*KL");
  const int kl = LM::kl(lane), p = LM::p(lane), q = LM::q(lane), cgrp = LM::cl(lane);
  const int koff = ca * 4 * KL + kl * 4;
  float4 hv[BS];
#pragma unroll
  for (int ab = 0; ab < BS; ++ab) hv[ab] = *reinterpret_cast<const float4*>(&vec_s[(ab ^ q) * VSTRIDE + koff]);
#pragma unroll
  for (int r = 0; r < NR; ++r) {
#pragma unroll
    for (int au = 0; au < UPL; ++au) {
      float4 wv;
      if (r < NR - RG) {
        const int row = r * group_stride + row0 + cgrp * UPL + (au ^ p);
        wv = *reinterpret_cast<const float4*>(&W_s[row * KLEN + koff]);
      } else {
        const int ri = (r - (NR - RG)) > 0 ? (r - (NR - RG)) : 0;
        wv = make_float4(wreg[ri][au][c * 4 + 0], wreg[ri][au][c * 4 + 1], wreg[ri][au][c * 4 + 2],
                         wreg[ri][au][c * 4 + 3]);
      }
#pragma unroll
      for (int ab = 0; ab < BS; ++ab) {
        float a = acc[r][au][ab];
        a = fmaf(wv.x, hv[ab].x, a);
        a = fmaf(wv.y, hv[ab].y, a);
        a = fmaf(wv.z, hv[ab].z, a);
        a = fmaf(wv.w, hv[ab].w, a);
        acc[r][au][ab] = a;
      }
    }
  }
}

// Two independent round-to-nearest FMAs on the halves of a float2. sm_90 has no packed fp32 FMA, so this is two FFMA;
// each half rounds exactly like fma.rn.f32, so the paired contractions below give the same bits as scalar FMA chains.
__device__ __forceinline__ float2 fma2_rn(float2 a, float2 b, float2 c) {
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}

// Same chunk contraction with a float2 accumulator per (row, batch) holding the even-k and odd-k partial sums (two
// independent FMA chains, operands are the naturally 64-bit aligned halves of the 16-byte shared-memory loads);
// fold_pairs() adds the two halves before the butterfly.
template <int NR, int RG, int KL, int UPL, int BS, int KLEN, int VSTRIDE>
__device__ __forceinline__ void dots_chunk2(const float* __restrict__ W_s, int group_stride, int row0,
                                            const float (&wreg)[RG > 0 ? RG : 1][UPL][KLEN / KL],
                                            const float* __restrict__ vec_s, int c, int ca, int lane,
                                            float2 (&acc)[NR][UPL][BS]) {
  using LM = LaneMap<KL, UPL, BS>;
  const int kl = LM::kl(lane), p = LM::p(lane), q = LM::q(lane), cgrp = LM::cl(lane);
  const int koff = ca * 4 * KL + kl * 4;
  float4 hv[BS];
#pragma unroll
  for (int ab = 0; ab < BS; ++ab) hv[ab] = *reinterpret_cast<const float4*>(&vec_s[(ab ^ q) * VSTRIDE + koff]);
#pragma unroll
  for (int r = 0; r < NR; ++r) {
#pragma unroll
    for (int au = 0; au < UPL; ++au) {
      float4 wv;
      if (r < NR - RG) {
        const int row = r * group_stride + row0 + cgrp * UPL + (au ^ p);
        wv = *reinterpret_cast<const float4*>(&W_s[row * KLEN + koff]);
      } else {
        const int ri = (r - (NR - RG)) > 0 ? (r - (NR - RG)) : 0;
        wv = make_float4(wreg[ri][au][c * 4 + 0], wreg[ri][au][c * 4 + 1], wreg[ri][au][c * 4 + 2],
                         wreg[ri][au][c * 4 + 3]);
      }
#pragma unroll
      for (int ab = 0; ab < BS; ++ab) {
        float2 a = acc[r][au][ab];
        a = fma2_rn(make_float2(wv.x, wv.y), make_float2(hv[ab].x, hv[ab].y), a);
        a = fma2_rn(make_float2(wv.z, wv.w), make_float2(hv[ab].z, hv[ab].w), a);
        acc[r][au][ab] = a;
      }
    }
  }
}

template <int NR, int UPL, int BS>
__device__ __forceinline__ void fold_pairs(const float2 (&acc2)[NR][UPL][BS], float (&acc)[NR][UPL][BS]) {
#pragma unroll
  for (int r = 0; r < NR; ++r)
#pragma unroll
    for (int au = 0; au < UPL; ++au)
#pragma unroll
      for (int ab = 0; ab < BS; ++ab) acc[r][au][ab] = acc2[r][au][ab].x + acc2[r][au][ab].y;
}

// ---- batch-paired packed contraction (forward GRU) --------------------------------------------------------------
// dots_chunk2 pairs two k of ONE (row, batch), which costs a float2 accumulator per (row, batch) (96 registers for the
// GRU) and a pair fold before the butterfly. Pairing two BATCH rows instead makes both halves of the float2 final
// outputs: half the accumulator registers, no fold, and one weight serves both halves. For that the two batch values
// of one k must be an aligned 64-bit word in shared memory (one 8-byte load), so the state vector is kept in a paired
// layout:
//   index(j, b) = ((((j / CW) * 4 + j % 4) * (BS/2) + b / 2) * KL + (j % CW) / 4) * 2 + b % 2,   CW = 4*KL
// i.e. for a fixed (chunk, e = k % 4, batch pair) the KL k-lanes read KL consecutive 8-byte words (conflict free).
// Slot am of a lane holds batch pair am ^ (q >> 1); the low bit of q is resolved by the last butterfly stage.
template <int KL, int BS>
__device__ __forceinline__ int paired_index(int j, int b) {
  constexpr int CW = 4 * KL;
  return ((((j / CW) * 4 + (j & 3)) * (BS / 2) + (b >> 1)) * KL + (j % CW) / 4) * 2 + (b & 1);
}

template <int NR, int RG, int KL, int UPL, int BS, int KLEN>
__device__ __forceinline__ void dots_chunk2b(const float* __restrict__ W_s, int group_stride, int row0,
                                             const float (&wreg)[RG > 0 ? RG : 1][UPL][KLEN / KL],
                                             const float* __restrict__ vec_s, int c, int ca, int lane,
                                             float2 (&acc)[NR][UPL][BS / 2]) {
  using LM = LaneMap<KL, UPL, BS>;
  constexpr int NP = BS / 2;
  const int kl = LM::kl(lane), p = LM::p(lane), qh = LM::q(lane) >> 1, cgrp = LM::cl(lane);
  const int koff = ca * 4 * KL + kl * 4;
  float2 hp[4][NP];
#pragma unroll
  for (int e = 0; e < 4; ++e)
#pragma unroll
    for (int am = 0; am < NP; ++am)
      hp[e][am] = *reinterpret_cast<const float2*>(&vec_s[(((ca * 4 + e) * NP + (am ^ qh)) * KL + kl) * 2]);
#pragma unroll
  for (int r = 0; r < NR; ++r) {
#pragma unroll
    for (int au = 0; au < UPL; ++au) {
      float4 wv;
      if (r < NR - RG) {
        const int row = r * group_stride + row0 + cgrp * UPL + (au ^ p);
        wv = *reinterpret_cast<const float4*>(&W_s[row * KLEN + koff]);
      } else {
        const int ri = (r - (NR - RG)) > 0 ? (r - (NR - RG)) : 0;
        wv = make_float4(wreg[ri][au][c * 4 + 0], wreg[ri][au][c * 4 + 1], wreg[ri][au][c * 4 + 2],
                         wreg[ri][au][c * 4 + 3]);
      }
#pragma unroll
      for (int am = 0; am < NP; ++am) {
        float2 a = acc[r][au][am];
        a = fma2_rn(make_float2(wv.x, wv.x), hp[0][am], a);
        a = fma2_rn(make_float2(wv.y, wv.y), hp[1][am], a);
        a = fma2_rn(make_float2(wv.z, wv.z), hp[2][am], a);
        a = fma2_rn(make_float2(wv.w, wv.w), hp[3][am], a);
        acc[r][au][am] = a;
      }
    }
  }
}

// Butterfly of the batch-paired accumulators: the same stages as warp_transpose_reduce over units and batch PAIRS, then
// one last exchange with lane ^ 1 in which the even lane keeps the pair's first batch and the odd lane its second.
// out[r] = full sum for unit LaneMap::unit(lane), batch LaneMap::q(lane).
template <int NR, int KL, int UPL, int BS>
__device__ __forceinline__ void warp_transpose_reduce2b(float2 (&acc)[NR][UPL][BS / 2], float (&out)[NR], int lane) {
  constexpr unsigned FULL = 0xffffffffu;
  constexpr int NP = BS / 2;
  const bool odd = (lane & 1) != 0;
#pragma unroll
  for (int r = 0; r < NR; ++r) {
    int off = KL / 2;
#pragma unroll
    for (int s = UPL / 2; s >= 1; s >>= 1) {
#pragma unroll
      for (int au = 0; au < s; ++au)
#pragma unroll
        for (int am = 0; am < NP; ++am) {
          acc[r][au][am].x += __shfl_xor_sync(FULL, acc[r][au + s][am].x, off);
          acc[r][au][am].y += __shfl_xor_sync(FULL, acc[r][au + s][am].y, off);
        }
      off >>= 1;
    }
#pragma unroll
    for (int s = NP / 2; s >= 1; s >>= 1) {
#pragma unroll
      for (int am = 0; am < s; ++am) {
        acc[r][0][am].x += __shfl_xor_sync(FULL, acc[r][0][am + s].x, off);
        acc[r][0][am].y += __shfl_xor_sync(FULL, acc[r][0][am + s].y, off);
      }
      off >>= 1;
    }
    const float mine = odd ? acc[r][0][0].y : acc[r][0][0].x;
    const float send = odd ? acc[r][0][0].x : acc[r][0][0].y;
    out[r] = mine + __shfl_xor_sync(FULL, send, 1);
  }
}

// Transposing butterfly over the KL k-lanes. On return acc[r][0][0] of a lane holds the full sum for
// unit LaneMap::unit(lane), batch LaneMap::q(lane).
template <int NR, int KL, int UPL, int BS>
__device__ __forceinline__ void warp_transpose_reduce(float (&acc)[NR][UPL][BS]) {
  constexpr unsigned FULL = 0xffffffffu;
#pragma unroll
  for (int r = 0; r < NR; ++r) {
    int off = KL / 2;
#pragma unroll
    for (int s = UPL / 2; s >= 1; s >>= 1) {
#pragma unroll
      for (int au = 0; au < s; ++au)
#pragma unroll
        for (int ab = 0; ab < BS; ++ab) acc[r][au][ab] += __shfl_xor_sync(FULL, acc[r][au + s][ab], off);
      off >>= 1;
    }
#pragma unroll
    for (int s = BS / 2; s >= 1; s >>= 1) {
#pragma unroll
      for (int ab = 0; ab < s; ++ab) acc[r][0][ab] += __shfl_xor_sync(FULL, acc[r][0][ab + s], off);
      off >>= 1;
    }
  }
}

}  // namespace b200rnn
