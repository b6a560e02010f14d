"""The weight_hh image of the weight cache (b200rnn_prepare_weights, prep_whh_h16) without a GPU.

A frozen unidirectional GRU-256 keeps each layer's weight_hh as the fp16-pair recurrence (rec_fwd_h16_kernel) stages it,
so the kernel's prologue is a copy. The cache layout (gemm_h16_layout.cuh wcache_layout) and the per-rank image
(rec_h16_layout.cuh, h16::Gru256 CACHE_*) are compiled into a host program that checks: the image exists exactly for
D = 1, G * H = 3 * 256; it lies behind every other region, 256-byte aligned, inside the reported total; each rank's
weights and row scales lie inside its own block, and the prep kernel's stores (w_index of every row, k and half, and the
scale slot of every row) cover each rank's weight region and scale slots exactly once."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "icassp2022-depression_b200", "csrc")
nvcc = shutil.which("nvcc") or shutil.which("/usr/local/cuda/bin/nvcc")

PROGRAM = r"""
#include <stdio.h>
#include <vector>
#include "gemm_h16_layout.cuh"
using namespace b200rnn;
using Lg = h16::Gru256;

static int fails = 0;
#define CHECK(c, ...) do { if (!(c)) { if (fails++ < 20) { printf("FAIL %s:%d ", __FILE__, __LINE__); printf(__VA_ARGS__); printf("\n"); } } } while (0)

int main() {
  CHECK(Lg::CACHE_RANK_BYTES == 196608 + 768 && Lg::CACHE_BYTES == 4 * Lg::CACHE_RANK_BYTES, "image size");
  // which caches hold the image: (L, D, I, DH, GH)
  const int cfg[][6] = {{2, 1, 256, 256, 768, 1}, {2, 1, 36, 256, 768, 1}, {1, 1, 256, 256, 768, 1},
                        {2, 2, 256, 512, 768, 0}, {2, 1, 256, 256, 1024, 0}, {2, 1, 128, 128, 384, 0},
                        {2, 2, 1024, 256, 512, 0}};
  for (auto& c : cfg) {
    const int L = c[0], D = c[1], I = c[2], DH = c[3], GH = c[4];
    const g16::WCache w = g16::wcache_layout(L, D, I, DH, GH);
    CHECK(w.has_whh16 == (c[5] != 0), "has_whh16 L=%d D=%d DH=%d GH=%d", L, D, DH, GH);
    if (!w.has_whh16) continue;
    size_t end_other = 0;
    for (int l = 0; l < L; ++l) {
      const int Il = l == 0 ? I : DH;
      size_t e = w.h16[l][0] + (g16::shape_ok(GH, Il) ? g16::w16_layout(GH, Il).bytes : 0);
      end_other = e > end_other ? e : end_other;
      e = w.lo[l][0] + (size_t)GH * Il * 4;
      end_other = e > end_other ? e : end_other;
    }
    for (int l = 0; l < L; ++l) {
      CHECK(w.whh16[l] % g16::ALIGN == 0, "layer %d image at %zu", l, w.whh16[l]);
      CHECK(w.whh16[l] >= end_other, "layer %d image overlaps the weight_ih regions", l);
      CHECK(w.whh16[l] + Lg::CACHE_BYTES <= w.total, "layer %d image past the total", l);
      if (l > 0) CHECK(w.whh16[l] >= w.whh16[l - 1] + Lg::CACHE_BYTES, "images %d and %d overlap", l - 1, l);
    }
  }
  // the prep kernel's stores: row = g * H + j, rank j / HS, unit j % HS
  std::vector<int> cnt(Lg::CACHE_BYTES / 2, 0);
  for (int g = 0; g < Lg::G; ++g)
    for (int j = 0; j < Lg::H; ++j) {
      const int rank = j / Lg::HS, u = j % Lg::HS;
      const int base = Lg::cache_rank_byte(rank) / 2;
      for (int k = 0; k < Lg::H; ++k)
        for (int hl = 0; hl < 2; ++hl) {
          const int i = Lg::w_index(g, u, k, hl);
          CHECK(i >= 0 && i < Lg::W_HALVES, "w_index %d", i);
          if (i >= 0 && i < Lg::W_HALVES) ++cnt[base + i];
        }
      const int sb = Lg::cache_rank_byte(rank) + Lg::W_HALVES * 2 + (g * Lg::HS + u) * 4;
      CHECK(sb + 4 <= Lg::cache_rank_byte(rank) + Lg::CACHE_RANK_BYTES, "scale slot past the rank block");
      cnt[sb / 2] += 1;
      cnt[sb / 2 + 1] += 1;
    }
  for (int r = 0; r < Lg::C; ++r) {
    const int base = Lg::cache_rank_byte(r) / 2;
    for (int i = 0; i < Lg::W_HALVES + Lg::G * Lg::HS * 2; ++i)
      CHECK(cnt[base + i] == 1, "rank %d half %d written %d times", r, i, cnt[base + i]);
  }
  printf(fails ? "FAILED %d\n" : "OK\n", fails);
  return fails ? 1 : 0;
}
"""


@pytest.mark.skipif(nvcc is None, reason="nvcc not available")
def test_whh_cache_image_is_in_bounds_and_covered_once(tmp_path):
    src = tmp_path / "whh_cache.cu"
    src.write_text(PROGRAM)
    exe = tmp_path / "whh_cache"
    proc = subprocess.run([nvcc, "-std=c++17", "-O1", "-I", CSRC, str(src), "-o", str(exe)], capture_output=True,
                          text=True, timeout=600)
    assert proc.returncode == 0, proc.stdout + proc.stderr
    run = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
    assert run.returncode == 0 and run.stdout.strip().endswith("OK"), run.stdout + run.stderr
