// rec_h16_layout.cuh — shared-memory layout of the fp16-pair forward recurrences (rec_fwd_tc_body, rnn_rec.cu): where the
// staging loop puts each weight, where the lane that produces h_t puts each state element, and which 16 bytes a lane
// reads or hands to the peers. Host and device code: tests/test_h16_layout_cpu.py (GRU-256) and
// tests/test_lstm_h16_layout_cpu.py (LSTM-128) compile these helpers into a host program and check every offset against
// the regions below and the mma.sync fragment definitions.
//
// Geometry (Geom<H, C, G, RING_IN_TILE>): H units, C CTAs per cluster, HS = H / C units per CTA, BS = 8 batch rows,
// G gate tiles, HS / 16 unit groups of 16 units, two warps per unit group (k halves). The contraction runs as
// mma.sync m16n8k16 f16 -> f32 (ptx.cuh mma_f16_m16n8k16) over H / 16 k-blocks of 16, each operand a (hi, lo) pair of
// fp16. Two geometries are built: the GRU-256 one (H = 256, C = 4, G = 3; rec_fwd_h16_kernel), whose names the plain
// h16:: constants and functions below keep, and the LSTM-128 one (H = 128, C = 2, G = 4; lstm_fwd_h16_kernel).
//
// k order inside a k-block: fragment position p (the k index of the PTX fragments) holds unit kk = h16_perm(p) of the
// block, bits 2 and 3 swapped. Lane (g, t) of the B fragment then holds units {0,1,4,5} (t = 0), {2,3,6,7} (t = 1),
// {8,9,12,13} (t = 2), {10,11,14,15} (t = 3): the lanes t < 2 hold the first 8 units of the block, the lanes t >= 2 the
// last 8. A and B use the same order, so the product is unchanged.
#pragma once
#include <math.h>

namespace b200rnn {
namespace h16 {

// Row scale 2^e of the weight split: max |w| of the row times 2^e lies in [2^14, 2^15), so hi = RN_f16(w 2^e) is normal
// for every weight within 2^-28 of the row's maximum. e = 0 for a row whose maximum is 0 or not finite: zeros stay exact,
// and an Inf weight gives hi = Inf, lo = NaN, NaN outputs, as the 3xTF32 split does. e <= 112 keeps 2^e and the unscale
// 2^-(e + 14) normal fp32 numbers; a row whose maximum is below 2^-98 is scaled less (its hi loses bits, at an absolute
// error below 2^-120).
__host__ __device__ inline int scale_exp(float m) {
  if (!(m > 0.f) || !(m <= 3.40282347e38f)) return 0;
  int x = 0;
  frexpf(m, &x);  // m = f 2^x, f in [0.5, 1)
  return 15 - x < 112 ? 15 - x : 112;
}
// the state scale: |h| <= 1 without an initial state, so |h| 2^14 <= 2^14 < 65504 (GRU: h is a convex combination of
// h_{t-1} and tanh; LSTM: h = o tanh(c) with o in (0, 1))
constexpr float STATE_SCALE = 16384.f;

__host__ __device__ constexpr int perm(int p) { return (p & 3) | ((p >> 3) & 1) << 2 | ((p >> 2) & 1) << 3; }

// B fragment of m16n8k16 (PTX ISA), lane (g, t): register 0 = {B[2t][g], B[2t + 1][g]}, 1 = {B[2t + 8][g], B[2t + 9][g]}
// (B[k][n], n = batch row). 16-byte slot of lane `lane` in a k-block: the slots of the lanes holding the first 8 units
// of the block come first, so that the 8 units a warp finishes are 256 contiguous bytes (see exchange_chunk)
__host__ __device__ constexpr int state_slot(int lane) { return ((lane & 3) >> 1) * 16 + (lane >> 2) * 2 + (lane & 1); }

// the exchange: after the warp finishing units k0 .. k0 + 7 (k0 % 8 == 0) has written them, lane l < 16 sends the
// 16-byte chunk with this index (in 16-byte units of the state buffer) to every peer
__host__ __device__ constexpr int exchange_chunk(int k0, int lane) { return (k0 / 16) * 32 + ((k0 % 16) / 8) * 16 + lane; }

// The x-projection ring (rnn_rec.cu, rec_fwd_tc_body): slot s holds one step's gates of the CTA, [G][BS][RING_ROW]
// floats, unit u of gate g, batch slot q at ring_index(g, q, u). A row is one 256-byte bulk copy; rows are padded to 68
// floats so that the rows 2t, 2t + 1 the lanes t = 0..3 of a warp read fall in different banks.
constexpr int RING_SLOTS = 4, RING_ROW = 68;

// RING_IN_TILE: the ring lives in dead weight space. The GRU-256 kernel reads the n tile's A fragments into registers in
// the prologue, so the n-tile region of unit group s (16 KB, one contiguous block of the weight region) is dead
// afterwards and holds slot s. Otherwise (LSTM-128: 128 KB of weights leave room) the ring has a region of its own,
// behind the weight region, the two state buffers and the k-half swap buffer [NW][2 G][32] floats.
template <int H_, int C_, int G_, bool RING_IN_TILE_>
struct Geom {
  static constexpr int H = H_, C = C_, HS = H / C, BS = 8, G = G_, NUG = HS / 16, NW = 2 * NUG;
  static constexpr bool RING_IN_TILE = RING_IN_TILE_;
  static constexpr int KB = H / 16;    // k-blocks of the contraction
  static constexpr int KBC = HS / 16;  // k-blocks per source slice
  // weights: [NUG][G][KB][hi, lo][32 lanes] of 16 bytes (4 f16x2 A-fragment registers): a lane's hi (lo) registers of
  // one (tile, k-block) are one LDS.128, a warp's are 512 contiguous bytes
  static constexpr int W_HALVES = NUG * G * KB * 2 * 32 * 8;
  // state: [KB][32 slots] of 16 bytes {hi b0, hi b1, lo b0, lo b1} per buffer
  static constexpr int S_HALVES = KB * 32 * 8;
  static constexpr int RED_BYTES = NW * 2 * G * 32 * 4;
  static constexpr int RING_SLOT_BYTES = G * BS * RING_ROW * 4;
  static_assert(W_HALVES * 2 == G * HS * H * 4, "the fp16 pairs fill exactly the bytes of the fp32 weight tiles");
  static_assert(S_HALVES * 2 == BS * H * 4, "the fp16 pairs fill exactly the bytes of an fp32 state buffer");
  static_assert(HS * 4 == 256, "one ring row is one 256-byte copy");

  // A fragment of m16n8k16 (PTX ISA), lane (g, t) = (lane / 4, lane % 4), register r, element e (low half first):
  //   r = 0: A[g][2t + e], 1: A[g + 8][2t + e], 2: A[g][2t + 8 + e], 3: A[g + 8][2t + 8 + e]
  // half index in the weight region of (unit group ug, tile gt, k-block kb, hl = 0 hi / 1 lo, lane, register, element)
  __host__ __device__ static constexpr int w_half(int ug, int gt, int kb, int hl, int lane, int r, int e) {
    return (((((ug * G + gt) * KB + kb) * 2 + hl) * 32 + lane) * 4 + r) * 2 + e;
  }
  // half index of weight row (gate gt, unit u of the CTA's slice), column k, part hl: where the staging loop writes it
  __host__ __device__ static constexpr int w_index(int gt, int u, int k, int hl) {
    return w_half(u / 16, gt, k / 16, hl, (u % 8) * 4 + (perm(k % 16) % 8) / 2, (u % 16) / 8 + 2 * (perm(k % 16) / 8),
                  perm(k % 16) % 2);
  }
  // half index of state element (unit k of the layer, batch row b), part hl, in one state buffer
  __host__ __device__ static constexpr int state_index(int k, int b, int hl) {
    // position of unit kk = k % 16 in the fragment: p = perm(kk); lane t = (p % 8) / 2, register p / 8, element p % 2
    return ((k / 16 * 32 + state_slot(b * 4 + (perm(k % 16) % 8) / 2)) * 4 + 2 * hl + perm(k % 16) / 8) * 2 +
           perm(k % 16) % 2;
  }
  __host__ __device__ static constexpr int ring_index(int g, int q, int u) { return (g * BS + q) * RING_ROW + u; }
  // byte offset of slot s in the shared-memory block (the weight region starts at 0)
  __host__ __device__ static constexpr int ring_byte(int s) {
    return RING_IN_TILE ? w_half(s, G - 1, 0, 0, 0, 0, 0) * 2 : W_HALVES * 2 + 2 * S_HALVES * 2 + RED_BYTES + s * RING_SLOT_BYTES;
  }
  // Weight cache image of W_hh (b200rnn_prepare_weights, prep_whh_h16): per CTA rank, the weight region exactly as the
  // prologue of the fp16-pair kernel stages it (W_HALVES halves), then the row scales 2^e_r, e_r = scale_exp(max_k
  // |w_rk|), of its G * HS rows as fp32 [G][HS], padded to 256 bytes
  static constexpr int CACHE_SCALE_BYTES = (G * HS * 4 + 255) / 256 * 256;
  static constexpr int CACHE_RANK_BYTES = W_HALVES * 2 + CACHE_SCALE_BYTES;
  static constexpr int CACHE_BYTES = C * CACHE_RANK_BYTES;
  __host__ __device__ static constexpr int cache_rank_byte(int rank) { return rank * CACHE_RANK_BYTES; }
  static_assert(CACHE_RANK_BYTES % 256 == 0 && (G * HS * 4) % 16 == 0, "16-byte copies, 256-byte aligned ranks");
  static_assert(!RING_IN_TILE || RING_SLOTS <= NUG, "one slot per unit group's n-tile region");
  static_assert(!RING_IN_TILE || RING_SLOT_BYTES <= KB * 2 * 32 * 8 * 2, "a slot fits the n-tile region of one unit group");
  static_assert((RING_ROW * 4) % 16 == 0 && ring_byte(0) % 128 == 0 && ring_byte(1) % 128 == 0,
                "bulk-copy destinations are 16-byte aligned");
};
using Gru256 = Geom<256, 4, 3, true>;
using Lstm128 = Geom<128, 2, 4, false>;

// the GRU-256 geometry under its plain names
constexpr int H = Gru256::H, C = Gru256::C, HS = Gru256::HS, BS = Gru256::BS, G = Gru256::G, NUG = Gru256::NUG,
              NW = Gru256::NW;
constexpr int KB = Gru256::KB, KBC = Gru256::KBC;
constexpr int W_HALVES = Gru256::W_HALVES, S_HALVES = Gru256::S_HALVES;
constexpr int RING_SLOT_BYTES = Gru256::RING_SLOT_BYTES;
__host__ __device__ constexpr int w_half(int ug, int gt, int kb, int hl, int lane, int r, int e) {
  return Gru256::w_half(ug, gt, kb, hl, lane, r, e);
}
__host__ __device__ constexpr int w_index(int gt, int u, int k, int hl) { return Gru256::w_index(gt, u, k, hl); }
__host__ __device__ constexpr int state_index(int k, int b, int hl) { return Gru256::state_index(k, b, hl); }
__host__ __device__ constexpr int ring_index(int g, int q, int u) { return Gru256::ring_index(g, q, u); }
__host__ __device__ constexpr int ring_byte(int s) { return Gru256::ring_byte(s); }

}  // namespace h16
}  // namespace b200rnn
