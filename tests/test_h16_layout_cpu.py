"""The fp16-pair GRU-256 forward recurrence (rec_fwd_h16_kernel) without a GPU: its shared-memory layout and its weight
split.

Layout: csrc/rec_h16_layout.cuh is compiled with nvcc into a host program, which checks for every (unit group, tile,
k-block, hi/lo, lane, register, element) that the offsets stay inside their regions, that the staging loop's and the state
writers' stores are bijections onto the weight and state regions, that the exchange chunks tile the state buffer and each
warp sends exactly the units it wrote, and that contracting the fragments as mma.sync m16n8k16 defines them gives the
plain matrix product.

Split: a float64 emulation of the row-scaled hi/lo split reproduces an fp32 dot to within 2^-21 of sum |w h| when the
three products are accumulated exactly."""
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "icassp2022-depression_b200", "csrc")
nvcc = shutil.which("nvcc") or (shutil.which("/usr/local/cuda/bin/nvcc"))

PROGRAM = r"""
#include <stdio.h>
#include <stdlib.h>
#include <vector>
#include "rec_h16_layout.cuh"
using namespace b200rnn::h16;

static int fails = 0;
#define CHECK(c, ...) do { if (!(c)) { if (fails++ < 20) { printf("FAIL %s:%d ", __FILE__, __LINE__); printf(__VA_ARGS__); printf("\n"); } } } while (0)

int main() {
  // weights: every (gate tile, unit, k, hi/lo) lands on its own half of the region
  std::vector<int> wcount(W_HALVES, 0);
  for (int g = 0; g < G; ++g)
    for (int u = 0; u < HS; ++u)
      for (int k = 0; k < H; ++k)
        for (int hl = 0; hl < 2; ++hl) {
          const int i = w_index(g, u, k, hl);
          CHECK(i >= 0 && i < W_HALVES, "w_index(%d,%d,%d,%d) = %d", g, u, k, hl, i);
          if (i >= 0 && i < W_HALVES) ++wcount[i];
          // the staging loop stores k, k+1 (k even) as one f16x2: adjacent halves, 4-byte aligned
          if (k % 2 == 0) CHECK(w_index(g, u, k + 1, hl) == i + 1 && i % 2 == 0, "pair %d %d %d", g, u, k);
        }
  for (int i = 0; i < W_HALVES; ++i) CHECK(wcount[i] == 1, "weight half %d written %d times", i, wcount[i]);
  // every fragment load of the step loop (and of the register tile) reads inside the region, 16-byte aligned
  for (int ug = 0; ug < NUG; ++ug)
    for (int g = 0; g < G; ++g)
      for (int kb = 0; kb < KB; ++kb)
        for (int hl = 0; hl < 2; ++hl)
          for (int lane = 0; lane < 32; ++lane) {
            const int i0 = w_half(ug, g, kb, hl, lane, 0, 0);
            CHECK(i0 % 8 == 0 && i0 >= 0 && i0 + 8 <= W_HALVES, "w_half %d", i0);
            CHECK(w_half(ug, g, kb, 1, lane, 0, 0) == w_half(ug, g, kb, 0, lane, 0, 0) + 32 * 8, "lo is 32 chunks on");
          }
  // state: the writers (every unit of the layer, every batch row) cover each buffer exactly once
  std::vector<int> scount(S_HALVES, 0);
  for (int k = 0; k < H; ++k)
    for (int b = 0; b < BS; ++b)
      for (int hl = 0; hl < 2; ++hl) {
        const int i = state_index(k, b, hl);
        CHECK(i >= 0 && i < S_HALVES, "state_index(%d,%d,%d) = %d", k, b, hl, i);
        if (i >= 0 && i < S_HALVES) ++scount[i];
      }
  for (int i = 0; i < S_HALVES; ++i) CHECK(scount[i] == 1, "state half %d written %d times", i, scount[i]);
  // the exchange: warp (CTA r, unit group ug, k half kh) finishes units k0 = r*HS + ug*16 + kh*8 .. k0 + 7; lanes
  // 0..15 send one 16-byte chunk each. The chunks of all warps of the cluster tile the buffer, and a warp's chunks are
  // exactly the halves its lanes wrote
  std::vector<int> ccount(S_HALVES / 8, 0);
  for (int r = 0; r < C; ++r)
    for (int w = 0; w < NW; ++w) {
      const int ug = w % NUG, kh = w / NUG, k0 = r * HS + ug * 16 + kh * 8;
      std::vector<int> sent(S_HALVES, 0);
      for (int lane = 0; lane < 16; ++lane) {
        const int ch = exchange_chunk(k0, lane);
        CHECK(ch == k0 / 8 * 16 + lane, "exchange chunk %d (the kernel sends float4 %d)", ch, k0 / 8 * 16 + lane);
        CHECK(ch >= 0 && ch < S_HALVES / 8, "chunk %d", ch);
        if (ch < 0 || ch >= S_HALVES / 8) continue;
        ++ccount[ch];
        for (int e = 0; e < 8; ++e) sent[ch * 8 + e] = 1;
      }
      for (int u = 0; u < 8; ++u)
        for (int b = 0; b < BS; ++b)
          for (int hl = 0; hl < 2; ++hl) CHECK(sent[state_index(k0 + u, b, hl)], "unit %d row %d not sent", k0 + u, b);
    }
  for (int i = 0; i < S_HALVES / 8; ++i) CHECK(ccount[i] == 1, "chunk %d sent %d times", i, ccount[i]);

  // the contraction: values stored by the layout functions, read back as the fragments of mma.sync m16n8k16 (PTX ISA)
  // and multiplied as the instruction does, give W x h for every gate row and batch row (small integers: exact)
  std::vector<int> Wv(G * HS * H), hv(BS * H);
  for (size_t i = 0; i < Wv.size(); ++i) Wv[i] = (int)(i * 7919 % 13) - 6;
  for (size_t i = 0; i < hv.size(); ++i) hv[i] = (int)(i * 104729 % 11) - 5;
  std::vector<long> Ws(W_HALVES, 0), Ss(S_HALVES, 0);
  for (int g = 0; g < G; ++g)
    for (int u = 0; u < HS; ++u)
      for (int k = 0; k < H; ++k)
        for (int hl = 0; hl < 2; ++hl) Ws[w_index(g, u, k, hl)] = (hl + 1) * Wv[(g * HS + u) * H + k];
  for (int k = 0; k < H; ++k)
    for (int b = 0; b < BS; ++b)
      for (int hl = 0; hl < 2; ++hl) Ss[state_index(k, b, hl)] = (hl + 1) * hv[b * H + k];
  for (int ug = 0; ug < NUG; ++ug)
    for (int g = 0; g < G; ++g)
      for (int hw = 0; hw < 2; ++hw)
        for (int hs = 0; hs < 2; ++hs) {
          long D[16][8] = {};
          for (int kb = 0; kb < KB; ++kb) {
            long A[16][16], B[16][8];
            for (int lane = 0; lane < 32; ++lane) {
              const int fg = lane / 4, t = lane % 4;
              for (int r = 0; r < 4; ++r)
                for (int e = 0; e < 2; ++e)
                  A[fg + 8 * (r % 2)][2 * t + 8 * (r / 2) + e] = Ws[w_half(ug, g, kb, hw, lane, r, e)];
              const int s = (kb * 32 + state_slot(lane)) * 8;
              for (int r = 0; r < 2; ++r)
                for (int e = 0; e < 2; ++e) B[2 * t + 8 * r + e][fg] = Ss[s + (2 * hs + r) * 2 + e];
            }
            for (int m = 0; m < 16; ++m)
              for (int n = 0; n < 8; ++n)
                for (int kk = 0; kk < 16; ++kk) D[m][n] += A[m][kk] * B[kk][n];
          }
          for (int m = 0; m < 16; ++m)
            for (int n = 0; n < 8; ++n) {
              long want = 0;
              for (int k = 0; k < H; ++k) want += (long)Wv[(g * HS + ug * 16 + m) * H + k] * hv[n * H + k];
              want *= (hw + 1) * (hs + 1);
              CHECK(D[m][n] == want, "ug %d tile %d hi/lo %d%d D[%d][%d] = %ld, want %ld", ug, g, hw, hs, m, n,
                    D[m][n], want);
            }
        }
  // the state scale and the row scale exponent
  CHECK(STATE_SCALE * 1.0f <= 16384.f && 16384.f * STATE_SCALE < 65504.f * 16384.f, "state scale");
  const float ms[] = {1.f, 0.75f, 3e-5f, 1e30f, 1e-30f, 1.5e-45f, 3.4e38f};
  for (float m : ms) {
    const int e = scale_exp(m);
    const double s = m * ldexp(1.0, e);
    CHECK(e <= 112 && e >= -113, "scale_exp(%g) = %d", m, e);
    CHECK(e == 112 ? s < 32768.0 : (s >= 16384.0 && s < 32768.0), "scale_exp(%g) = %d: %g", m, e, s);
  }
  CHECK(scale_exp(0.f) == 0 && scale_exp(1.f / 0.f) == 0 && scale_exp(0.f / 0.f) == 0, "zero / inf / nan rows");
  printf(fails ? "FAILED %d\n" : "OK\n", fails);
  return fails ? 1 : 0;
}
"""


@pytest.mark.skipif(nvcc is None, reason="nvcc not available")
def test_h16_layout_offsets_and_fragments(tmp_path):
    src = tmp_path / "h16_layout.cu"
    src.write_text(PROGRAM)
    exe = tmp_path / "h16_layout"
    proc = subprocess.run([nvcc, "-std=c++17", "-O1", "-I", CSRC, str(src), "-o", str(exe)], capture_output=True,
                          text=True, timeout=600)
    assert proc.returncode == 0, proc.stdout + proc.stderr
    run = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
    assert run.returncode == 0 and run.stdout.strip().endswith("OK"), run.stdout + run.stderr


cuobjdump = shutil.which("cuobjdump") or shutil.which("/usr/local/cuda/bin/cuobjdump")


@pytest.mark.skipif(cuobjdump is None, reason="cuobjdump not available")
def test_h16_kernel_runs_on_hmma_16816_without_local_memory():
    """Both instantiations (fixed length, ragged) contract with HMMA.16816.F32 only, keep the register tile in
    registers, and split nothing in the step loop (no HMMA.1688)."""
    import re

    from b200rnn import _lib

    txt = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    out, name = {}, None
    for line in txt.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1) if "rec_fwd_h16_kernel" in m.group(1) else None
            if name:
                out[name] = []
        elif name is not None:
            m = re.search(r"\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]*)", line)
            if m:
                out[name].append(m.group(1))
    assert len(out) == 2, sorted(out)
    for name, ops in out.items():
        assert sum(o == "HMMA.16816.F32" for o in ops) == 72, name  # 8 k-blocks x 3 tiles x 3 products per step
        assert not [o for o in ops if o.startswith("HMMA.1688")], name
        assert not sorted({o for o in ops if o.startswith(("LDL", "STL"))}), name


# ---- the weight split, emulated --------------------------------------------------------------------------------------

def _scale_exp(m):
    """h16::scale_exp"""
    if not (m > 0) or not np.isfinite(m):
        return 0
    _, x = np.frexp(np.float32(m))
    return min(15 - int(x), 112)


def _split(v):
    """hi = RN_f16(v), lo = RN_f16(v - hi), v fp32; v - hi is exact in fp32"""
    v = np.asarray(v, dtype=np.float32)
    hi = v.astype(np.float16)
    lo = (v - hi.astype(np.float32)).astype(np.float16)
    return hi.astype(np.float64), lo.astype(np.float64)


def _f16x3_dot(w, h):
    """the three products of the fp16-pair contraction, accumulated exactly (float64), unscaled"""
    e = _scale_exp(float(np.max(np.abs(w))) if np.all(np.isfinite(w)) else np.inf)
    with np.errstate(invalid="ignore", over="ignore"):
        wh, wl = _split(np.float32(w) * np.float32(2.0 ** e))
        hh, hl = _split(np.float32(h) * np.float32(16384.0))
        return (wh @ hh + (wl @ hh + wh @ hl)) * 2.0 ** -(e + 14)


def _rows(rng):
    yield "random", rng.standard_normal(256).astype(np.float32) * 0.06
    yield "zero", np.zeros(256, np.float32)
    yield "tiny", (rng.standard_normal(256) * 1e-30).astype(np.float32)
    yield "huge", (rng.standard_normal(256) * 1e30).astype(np.float32)
    w = rng.standard_normal(256).astype(np.float32)
    w[::7] = np.float32(1e-41)   # fp32 subnormals beside normal weights
    yield "subnormal", w
    w = rng.standard_normal(256).astype(np.float32)
    w[::5] *= np.float32(2.0 ** -20)   # weights far below the row maximum
    yield "spread", w


@pytest.mark.parametrize("seed", range(4))
def test_scaled_f16_split_reproduces_the_fp32_dot(seed):
    rng = np.random.default_rng(seed)
    for name, w in _rows(rng):
        for h in (np.tanh(rng.standard_normal(256)).astype(np.float32),
                  (rng.uniform(-1, 1, 256) * (rng.uniform(size=256) < 0.5)).astype(np.float32),
                  np.float32(1e-20) * rng.standard_normal(256).astype(np.float32)):
            exact = w.astype(np.float64) @ h.astype(np.float64)
            scale = np.abs(w.astype(np.float64)) @ np.abs(h.astype(np.float64))
            got = _f16x3_dot(w, h)
            # the row's hi is normal, lo is exact to 2^-11 of itself; h near 0 has absolute error below 2^-38 per term
            tol = 2.0 ** -21 * scale + 256 * 2.0 ** -38 * np.abs(w.astype(np.float64)).max()
            assert abs(got - exact) <= tol, (name, got, exact, tol)


def test_non_finite_rows_give_nan():
    w = np.zeros(256, np.float32)
    w[3] = np.inf
    h = np.full(256, 0.5, np.float32)
    assert np.isnan(_f16x3_dot(w, h))
    w[3] = np.nan
    assert np.isnan(_f16x3_dot(w, h))
