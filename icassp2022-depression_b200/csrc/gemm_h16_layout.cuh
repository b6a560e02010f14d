// gemm_h16_layout.cuh — where the fp16-pair input projection (gemm_f16x3_kernel, gemm_tc.cu) finds its split weight,
// and where the weight cache of b200rnn_prepare_weights (api.cu) puts every split. Host and device code:
// tests/test_gemm_h16_layout_cpu.py compiles these helpers into a host program and checks that every region is in
// bounds, 256-byte aligned and disjoint from every other.
//
// Split weight of one GEMM (W = weight_ih [N][K], N % 128 == 0, K % 64 == 0), from a 256-byte aligned base:
//   hi  [N][K] fp16   row n = RN_f16(w 2^e_n)
//   lo  [N][K] fp16   RN_f16(w 2^e_n - hi)
//   exp [N]    int    e_n = h16::scale_exp(max_k |w[n][k]|)
// Weight cache, per (layer l, direction k) in this order: the TF32 hi and lo splits of weight_ih as dense fp32 [N][K_l]
// (read by the autograd / TF32 forwards of a frozen module), then the fp16-pair split above (the no-grad forward).
// A unidirectional GRU-256 (D = 1, GH = 3 DH, DH = 256) then has, per layer, weight_hh as the fp16-pair recurrence
// stages it (rec_h16_layout.cuh, h16::Gru256::CACHE_BYTES).
#pragma once
#include <stddef.h>
#include <string.h>

#include "rec_h16_layout.cuh"

namespace b200rnn {
namespace g16 {

constexpr int BK = 64;           // k-block of the fp16-pair GEMM: 4 wgmma k16 steps, one 128-byte fp16 W row
constexpr size_t ALIGN = 256;    // every region starts on a 256-byte boundary
constexpr int MAX_LAYERS = 8;

__host__ __device__ constexpr size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// h16::scale_exp(m) for m >= 0 (a max of |x|) from the exponent bits alone, without frexpf's branches: e = 15 - x for
// m = f 2^x, f in [0.5, 1), capped at 112 (which covers every subnormal m); 0 for m == 0 and for Inf / NaN
__host__ __device__ inline int scale_exp_bits(float m) {
  unsigned u;
  memcpy(&u, &m, sizeof u);
  const int be = (int)((u >> 23) & 0xffu);
  return (m > 0.f && be < 255) ? (141 - be < 112 ? 141 - be : 112) : 0;
}
// 2^e as a float for |e| <= 126, exact
__host__ __device__ inline float exp2i(int e) {
  const unsigned u = (unsigned)(e + 127) << 23;
  float f;
  memcpy(&f, &u, sizeof f);
  return f;
}

// the shapes the fp16-pair GEMM takes (the alignment rules of the fp32-A kernel are checked by its launcher)
__host__ __device__ constexpr bool shape_ok(int N, int K) { return N > 0 && N % 128 == 0 && K >= BK && K % BK == 0; }

// byte offsets of one split weight from its base, and its extent
struct W16 {
  size_t hi, lo, exp, bytes;
};
__host__ __device__ constexpr W16 w16_layout(int N, int K) {
  return W16{0, align_up((size_t)N * K * 2, ALIGN), 2 * align_up((size_t)N * K * 2, ALIGN),
             2 * align_up((size_t)N * K * 2, ALIGN) + align_up((size_t)N * 4, ALIGN)};
}
// the fp16 split fits the room the per-call TF32 hi / lo split of W had in the GEMM workspace (8 N K bytes)
static_assert(w16_layout(128, 64).bytes <= (size_t)8 * 128 * 64, "fp16 pairs + exponents fit the TF32 hi/lo room");
static_assert(w16_layout(768, 256).lo % ALIGN == 0 && w16_layout(768, 256).exp % ALIGN == 0, "256-byte aligned");

// weight cache: byte offsets of each (layer, direction)'s regions. GH = gates x hidden (rows of weight_ih), I = input
// size of layer 0, DH = directions x hidden (input size of every later layer)
struct WCache {
  size_t hi[MAX_LAYERS][2], lo[MAX_LAYERS][2], h16[MAX_LAYERS][2];
  bool has_whh16;  // the GRU-256 weight_hh images below exist
  size_t whh16[MAX_LAYERS];
  size_t total;
};
inline WCache wcache_layout(int L, int D, int I, int DH, int GH) {
  WCache w = {};
  size_t off = 0;
  for (int l = 0; l < L && l < MAX_LAYERS; ++l) {
    const int Il = l == 0 ? I : DH;
    for (int k = 0; k < D; ++k) {
      w.hi[l][k] = off;
      off += align_up((size_t)GH * Il * 4, ALIGN);
      w.lo[l][k] = off;
      off += align_up((size_t)GH * Il * 4, ALIGN);
      w.h16[l][k] = off;
      if (shape_ok(GH, Il)) off += w16_layout(GH, Il).bytes;
    }
  }
  w.has_whh16 = D == 1 && DH == h16::Gru256::H && GH == h16::Gru256::G * DH;
  for (int l = 0; w.has_whh16 && l < L && l < MAX_LAYERS; ++l) {
    w.whh16[l] = off;
    off += align_up((size_t)h16::Gru256::CACHE_BYTES, ALIGN);
  }
  w.total = off;
  return w;
}

}  // namespace g16
}  // namespace b200rnn
