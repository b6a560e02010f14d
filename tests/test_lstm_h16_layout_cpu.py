"""The fp16-pair LSTM-128 forward recurrence (lstm_fwd_h16_kernel, the no-grad forward of b200rnn_forward_fused) without
a GPU.

Layout: the LSTM-128 geometry of csrc/rec_h16_layout.cuh (h16::Lstm128: 2-CTA clusters, 64 units x 4 gate tiles per
CTA, 8 k-blocks) is compiled with nvcc into a host program, which checks that the offsets stay inside their regions,
that the staging loop's and the state writers' stores are bijections onto the weight and state regions, that the
exchange chunks tile the state buffer and each warp sends exactly the units it wrote, that the x-projection ring lies
outside every region the step loop reads, and that contracting the fragments as mma.sync m16n8k16 defines them gives
the plain matrix product.

SASS: both instantiations (fixed length, ragged) contract with HMMA.16816.F32 only and use no stack and no local
memory."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "icassp2022-depression_b200", "csrc")
LIB = os.path.join(ROOT, "icassp2022-depression_b200", "lib", "libb200rnn.so")
nvcc = shutil.which("nvcc") or (shutil.which("/usr/local/cuda/bin/nvcc"))
cuobjdump = shutil.which("cuobjdump") or shutil.which("/usr/local/cuda/bin/cuobjdump")

PROGRAM = r"""
#include <stdio.h>
#include <vector>
#include "rec_h16_layout.cuh"
using namespace b200rnn::h16;
using Lg = Lstm128;

static int fails = 0;
#define CHECK(c, ...) do { if (!(c)) { if (fails++ < 20) { printf("FAIL %s:%d ", __FILE__, __LINE__); printf(__VA_ARGS__); printf("\n"); } } } while (0)

int main() {
  CHECK(Lg::H == 128 && Lg::C == 2 && Lg::HS == 64 && Lg::BS == 8 && Lg::G == 4 && Lg::NW == 8 && Lg::KB == 8 &&
        Lg::KBC == 4, "geometry");
  CHECK(Lg::W_HALVES * 2 == 128 * 1024, "128 KB of weight pairs");
  // weights: every (gate tile, unit, k, hi/lo) lands on its own half of the region
  std::vector<int> wcount(Lg::W_HALVES, 0);
  for (int g = 0; g < Lg::G; ++g)
    for (int u = 0; u < Lg::HS; ++u)
      for (int k = 0; k < Lg::H; ++k)
        for (int hl = 0; hl < 2; ++hl) {
          const int i = Lg::w_index(g, u, k, hl);
          CHECK(i >= 0 && i < Lg::W_HALVES, "w_index(%d,%d,%d,%d) = %d", g, u, k, hl, i);
          if (i >= 0 && i < Lg::W_HALVES) ++wcount[i];
          if (k % 2 == 0) CHECK(Lg::w_index(g, u, k + 1, hl) == i + 1 && i % 2 == 0, "pair %d %d %d", g, u, k);
        }
  for (int i = 0; i < Lg::W_HALVES; ++i) CHECK(wcount[i] == 1, "weight half %d written %d times", i, wcount[i]);
  for (int ug = 0; ug < Lg::NUG; ++ug)
    for (int g = 0; g < Lg::G; ++g)
      for (int kb = 0; kb < Lg::KB; ++kb)
        for (int lane = 0; lane < 32; ++lane) {
          const int i0 = Lg::w_half(ug, g, kb, 0, lane, 0, 0);
          CHECK(i0 % 8 == 0 && i0 >= 0 && i0 + 8 <= Lg::W_HALVES, "w_half %d", i0);
          CHECK(Lg::w_half(ug, g, kb, 1, lane, 0, 0) == i0 + 32 * 8, "lo is 32 chunks on");
        }
  // state: the writers (every unit of the layer, every batch row) cover each buffer exactly once
  std::vector<int> scount(Lg::S_HALVES, 0);
  for (int k = 0; k < Lg::H; ++k)
    for (int b = 0; b < Lg::BS; ++b)
      for (int hl = 0; hl < 2; ++hl) {
        const int i = Lg::state_index(k, b, hl);
        CHECK(i >= 0 && i < Lg::S_HALVES, "state_index(%d,%d,%d) = %d", k, b, hl, i);
        if (i >= 0 && i < Lg::S_HALVES) ++scount[i];
      }
  for (int i = 0; i < Lg::S_HALVES; ++i) CHECK(scount[i] == 1, "state half %d written %d times", i, scount[i]);
  // the exchange: the chunks of all warps of the cluster tile the buffer, a warp's chunks are the halves it wrote
  std::vector<int> ccount(Lg::S_HALVES / 8, 0);
  for (int r = 0; r < Lg::C; ++r)
    for (int w = 0; w < Lg::NW; ++w) {
      const int ug = w % Lg::NUG, kh = w / Lg::NUG, k0 = r * Lg::HS + ug * 16 + kh * 8;
      std::vector<int> sent(Lg::S_HALVES, 0);
      for (int lane = 0; lane < 16; ++lane) {
        const int ch = exchange_chunk(k0, lane);
        CHECK(ch == k0 / 8 * 16 + lane, "exchange chunk %d (the kernel sends float4 %d)", ch, k0 / 8 * 16 + lane);
        CHECK(ch >= 0 && ch < Lg::S_HALVES / 8, "chunk %d", ch);
        if (ch < 0 || ch >= Lg::S_HALVES / 8) continue;
        ++ccount[ch];
        for (int e = 0; e < 8; ++e) sent[ch * 8 + e] = 1;
      }
      for (int u = 0; u < 8; ++u)
        for (int b = 0; b < Lg::BS; ++b)
          for (int hl = 0; hl < 2; ++hl)
            CHECK(sent[Lg::state_index(k0 + u, b, hl)], "unit %d row %d not sent", k0 + u, b);
    }
  for (int i = 0; i < Lg::S_HALVES / 8; ++i) CHECK(ccount[i] == 1, "chunk %d sent %d times", i, ccount[i]);
  // the ring: its own region behind the weights, both state buffers and the swap buffer; slots disjoint and aligned,
  // so no byte of a fragment, a state buffer or a partial sum the step loop reads belongs to a slot
  CHECK(!Lg::RING_IN_TILE, "the LSTM ring has a region of its own");
  const int read_end = Lg::W_HALVES * 2 + 2 * Lg::S_HALVES * 2 + Lg::RED_BYTES;
  for (int s = 0; s < RING_SLOTS; ++s) {
    const int b0 = Lg::ring_byte(s);
    CHECK(b0 >= read_end && b0 % 128 == 0, "slot %d at %d", s, b0);
    if (s > 0) CHECK(b0 >= Lg::ring_byte(s - 1) + Lg::RING_SLOT_BYTES, "slots %d and %d overlap", s - 1, s);
  }
  for (int ug = 0; ug < Lg::NUG; ++ug)
    for (int g = 0; g < Lg::G; ++g)
      for (int kb = 0; kb < Lg::KB; ++kb)
        for (int hl = 0; hl < 2; ++hl)
          for (int lane = 0; lane < 32; ++lane)
            CHECK(Lg::w_half(ug, g, kb, hl, lane, 0, 0) * 2 + 16 <= Lg::ring_byte(0), "fragment in the ring");
  std::vector<int> rcount(Lg::RING_SLOT_BYTES / 4, 0);
  for (int g = 0; g < Lg::G; ++g)
    for (int q = 0; q < Lg::BS; ++q) {
      CHECK((Lg::ring_index(g, q, 0) * 4) % 16 == 0, "row %d %d not 16-byte aligned", g, q);
      for (int u = 0; u < Lg::HS; ++u) {
        const int i = Lg::ring_index(g, q, u);
        CHECK(i >= 0 && i < Lg::RING_SLOT_BYTES / 4, "ring_index(%d,%d,%d) = %d", g, q, u, i);
        if (i >= 0 && i < Lg::RING_SLOT_BYTES / 4) ++rcount[i];
      }
    }
  for (int i = 0; i < Lg::RING_SLOT_BYTES / 4; ++i) CHECK(rcount[i] <= 1, "ring float %d written %d times", i, rcount[i]);
  for (int u0 = 0; u0 < Lg::HS; u0 += 8)
    for (int g = 0; g < Lg::G; ++g)
      for (int jb = 0; jb < 2; ++jb) {
        int banks = 0;
        for (int lane = 0; lane < 32; ++lane)
          banks |= 1 << (Lg::ring_index(g, 2 * (lane & 3) + jb, u0 + (lane >> 2)) % 32);
        CHECK(banks == -1, "units %d gate %d jb %d: bank conflict (mask %08x)", u0, g, jb, banks);
      }

  // the contraction: values stored by the layout functions, read back as the fragments of mma.sync m16n8k16 (PTX ISA)
  // and multiplied as the instruction does, give W x h for every gate row and batch row (small integers: exact)
  std::vector<int> Wv(Lg::G * Lg::HS * Lg::H), hv(Lg::BS * Lg::H);
  for (size_t i = 0; i < Wv.size(); ++i) Wv[i] = (int)(i * 7919 % 13) - 6;
  for (size_t i = 0; i < hv.size(); ++i) hv[i] = (int)(i * 104729 % 11) - 5;
  std::vector<long> Ws(Lg::W_HALVES, 0), Ss(Lg::S_HALVES, 0);
  for (int g = 0; g < Lg::G; ++g)
    for (int u = 0; u < Lg::HS; ++u)
      for (int k = 0; k < Lg::H; ++k)
        for (int hl = 0; hl < 2; ++hl) Ws[Lg::w_index(g, u, k, hl)] = (hl + 1) * Wv[(g * Lg::HS + u) * Lg::H + k];
  for (int k = 0; k < Lg::H; ++k)
    for (int b = 0; b < Lg::BS; ++b)
      for (int hl = 0; hl < 2; ++hl) Ss[Lg::state_index(k, b, hl)] = (hl + 1) * hv[b * Lg::H + k];
  for (int ug = 0; ug < Lg::NUG; ++ug)
    for (int g = 0; g < Lg::G; ++g)
      for (int hw = 0; hw < 2; ++hw)
        for (int hs = 0; hs < 2; ++hs) {
          long D[16][8] = {};
          for (int kb = 0; kb < Lg::KB; ++kb) {
            long A[16][16], B[16][8];
            for (int lane = 0; lane < 32; ++lane) {
              const int fg = lane / 4, t = lane % 4;
              for (int r = 0; r < 4; ++r)
                for (int e = 0; e < 2; ++e)
                  A[fg + 8 * (r % 2)][2 * t + 8 * (r / 2) + e] = Ws[Lg::w_half(ug, g, kb, hw, lane, r, e)];
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
              for (int k = 0; k < Lg::H; ++k) want += (long)Wv[(g * Lg::HS + ug * 16 + m) * Lg::H + k] * hv[n * Lg::H + k];
              want *= (hw + 1) * (hs + 1);
              CHECK(D[m][n] == want, "ug %d tile %d hi/lo %d%d D[%d][%d] = %ld, want %ld", ug, g, hw, hs, m, n,
                    D[m][n], want);
            }
        }
  printf(fails ? "FAILED %d\n" : "OK\n", fails);
  return fails ? 1 : 0;
}
"""


@pytest.mark.skipif(nvcc is None, reason="nvcc not available")
def test_lstm_h16_layout_offsets_ring_and_fragments(tmp_path):
    src = tmp_path / "lstm_h16_layout.cu"
    src.write_text(PROGRAM)
    exe = tmp_path / "lstm_h16_layout"
    proc = subprocess.run([nvcc, "-std=c++17", "-O1", "-I", CSRC, str(src), "-o", str(exe)], capture_output=True,
                          text=True, timeout=600)
    assert proc.returncode == 0, proc.stdout + proc.stderr
    run = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
    assert run.returncode == 0 and run.stdout.strip().endswith("OK"), run.stdout + run.stderr


@pytest.mark.skipif(cuobjdump is None, reason="cuobjdump not available")
def test_lstm_h16_kernel_runs_on_hmma_16816_without_local_memory():
    """48 HMMA.16816.F32 per warp and step (2 slices x 2 k-blocks x 4 tiles x 3 products), no HMMA.1688, no
    local-memory traffic, and -res-usage reports no stack and no local memory"""
    txt = subprocess.run([cuobjdump, "-sass", LIB], capture_output=True, text=True, timeout=300).stdout
    out, name = {}, None
    for line in txt.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1) if "lstm_fwd_h16_kernel" in m.group(1) else None
            if name:
                out[name] = []
        elif name is not None:
            m = re.search(r"\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]*)", line)
            if m:
                out[name].append(m.group(1))
    assert len(out) == 2, sorted(out)
    for name, ops in out.items():
        assert sum(o == "HMMA.16816.F32" for o in ops) == 48, name
        assert not [o for o in ops if o.startswith("HMMA.1688")], name
        assert not sorted({o for o in ops if o.startswith(("LDL", "STL"))}), name
    res = subprocess.run([cuobjdump, "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    seen, name = {}, None
    for line in res.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1) if "lstm_fwd_h16_kernel" in m.group(1) else None
            continue
        m = re.search(r"STACK:(\d+) .*LOCAL:(\d+)", line)
        if m and name:
            seen[name] = (int(m.group(1)), int(m.group(2)))
    assert len(seen) == 2 and all(v == (0, 0) for v in seen.values()), seen
