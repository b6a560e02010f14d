"""The x-projection ring of the fp16-pair GRU-256 forward recurrence (rec_fwd_h16_kernel) without a GPU.

Its slots live in the weight region, in the n-tile A fragments that the prologue reads into registers. A host program
compiled from csrc/rec_h16_layout.cuh checks that every slot lies inside the weight region and overlaps no fragment
the step loop still reads (the r and z tiles of every unit group), that the slots are disjoint and every row is a
16-byte-aligned 256-byte bulk-copy destination inside its slot, and that the six values a compute warp reads per step
(one gate and batch row of each lane) fall in 32 different banks."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "icassp2022-depression_b200", "csrc")
nvcc = shutil.which("nvcc") or (shutil.which("/usr/local/cuda/bin/nvcc"))

PROGRAM = r"""
#include <stdio.h>
#include <vector>
#include "rec_h16_layout.cuh"
using namespace b200rnn::h16;

static int fails = 0;
#define CHECK(c, ...) do { if (!(c)) { if (fails++ < 20) { printf("FAIL %s:%d ", __FILE__, __LINE__); printf(__VA_ARGS__); printf("\n"); } } } while (0)

int main() {
  const int W_BYTES = W_HALVES * 2;
  std::vector<int> owner(W_BYTES, -1);  // which slot covers each byte of the weight region
  for (int s = 0; s < RING_SLOTS; ++s) {
    const int b0 = ring_byte(s);
    CHECK(b0 >= 0 && b0 + RING_SLOT_BYTES <= W_BYTES && b0 % 16 == 0, "slot %d at %d", s, b0);
    for (int b = b0; b < b0 + RING_SLOT_BYTES && b < W_BYTES; ++b) {
      CHECK(owner[b] == -1, "slots %d and %d overlap at byte %d", owner[b], s, b);
      owner[b] = s;
    }
  }
  // no byte the step loop reads (the A fragments of the r and z tiles, 16 bytes per lane) belongs to a slot
  for (int ug = 0; ug < NUG; ++ug)
    for (int g = 0; g < G - 1; ++g)
      for (int kb = 0; kb < KB; ++kb)
        for (int hl = 0; hl < 2; ++hl)
          for (int lane = 0; lane < 32; ++lane) {
            const int b0 = w_half(ug, g, kb, hl, lane, 0, 0) * 2;
            for (int b = b0; b < b0 + 16; ++b)
              CHECK(owner[b] == -1, "step-loop fragment ug %d tile %d kb %d byte %d is in slot %d", ug, g, kb, b, owner[b]);
          }
  // every slot byte was an n-tile byte (read once into registers in the prologue)
  std::vector<char> ntile(W_BYTES, 0);
  for (int ug = 0; ug < NUG; ++ug)
    for (int kb = 0; kb < KB; ++kb)
      for (int hl = 0; hl < 2; ++hl)
        for (int lane = 0; lane < 32; ++lane)
          for (int b = 0; b < 16; ++b) ntile[w_half(ug, G - 1, kb, hl, lane, 0, 0) * 2 + b] = 1;
  for (int b = 0; b < W_BYTES; ++b) CHECK(owner[b] == -1 || ntile[b], "slot byte %d is not in an n tile", b);
  // rows: one 256-byte, 16-byte-aligned copy each, disjoint, inside the slot
  std::vector<int> rcount(RING_SLOT_BYTES / 4, 0);
  for (int g = 0; g < G; ++g)
    for (int q = 0; q < BS; ++q) {
      CHECK((ring_index(g, q, 0) * 4) % 16 == 0, "row %d %d not 16-byte aligned", g, q);
      for (int u = 0; u < HS; ++u) {
        const int i = ring_index(g, q, u);
        CHECK(i >= 0 && i < RING_SLOT_BYTES / 4, "ring_index(%d,%d,%d) = %d", g, q, u, i);
        if (i >= 0 && i < RING_SLOT_BYTES / 4) ++rcount[i];
        if (u > 0) CHECK(i == ring_index(g, q, u - 1) + 1, "row %d %d not contiguous", g, q);
      }
    }
  for (int i = 0; i < RING_SLOT_BYTES / 4; ++i) CHECK(rcount[i] <= 1, "ring float %d written %d times", i, rcount[i]);
  // the compute lanes' reads: lane (fg, ft) of the warp finishing units u0 .. u0 + 7 reads unit u0 + fg, row 2 ft + jb
  for (int u0 = 0; u0 < HS; u0 += 8)
    for (int g = 0; g < G; ++g)
      for (int jb = 0; jb < 2; ++jb) {
        int banks = 0;
        for (int lane = 0; lane < 32; ++lane) banks |= 1 << (ring_index(g, 2 * (lane & 3) + jb, u0 + (lane >> 2)) % 32);
        CHECK(banks == -1, "units %d gate %d jb %d: bank conflict (mask %08x)", u0, g, jb, banks);
      }
  printf(fails ? "FAILED %d\n" : "OK\n", fails);
  return fails ? 1 : 0;
}
"""


@pytest.mark.skipif(nvcc is None, reason="nvcc not available")
def test_h16_ring_slots_stay_out_of_the_step_loop_reads(tmp_path):
    src = tmp_path / "h16_ring.cu"
    src.write_text(PROGRAM)
    exe = tmp_path / "h16_ring"
    proc = subprocess.run([nvcc, "-std=c++17", "-O1", "-I", CSRC, str(src), "-o", str(exe)], capture_output=True,
                          text=True, timeout=600)
    assert proc.returncode == 0, proc.stdout + proc.stderr
    run = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
    assert run.returncode == 0 and run.stdout.strip().endswith("OK"), run.stdout + run.stderr
