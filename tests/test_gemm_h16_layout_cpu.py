"""The fp16-pair input projection's memory layout without a GPU: csrc/gemm_h16_layout.cuh is compiled with nvcc into a host
program, which checks for the split weight of every GEMM shape and for the weight cache of every (layer, direction) that
each region is in bounds, 256-byte aligned and disjoint from every other region, and that the per-call split fits the
room of the TF32 hi / lo weight split in the GEMM workspace. The kernel's branch-free row exponent (g16::scale_exp_bits)
is checked against h16::scale_exp over every exponent field."""
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
#include <algorithm>
#include <math.h>
#include <string.h>
#include "gemm_h16_layout.cuh"
#include "rec_h16_layout.cuh"
using namespace b200rnn::g16;

static int fails = 0;
#define CHECK(c, ...) do { if (!(c)) { if (fails++ < 20) { printf("FAIL line %d: ", __LINE__); printf(__VA_ARGS__); printf("\n"); } } } while (0)

struct R { size_t b, e; const char* what; };

static void disjoint(std::vector<R> v, size_t total, const char* ctx) {
  std::sort(v.begin(), v.end(), [](const R& x, const R& y) { return x.b < y.b; });
  for (size_t i = 0; i < v.size(); ++i) {
    CHECK(v[i].b % ALIGN == 0, "%s: %s at %zu not 256-byte aligned", ctx, v[i].what, v[i].b);
    CHECK(v[i].e <= total, "%s: %s ends at %zu past %zu", ctx, v[i].what, v[i].e, total);
    if (i) CHECK(v[i - 1].e <= v[i].b, "%s: %s overlaps %s", ctx, v[i - 1].what, v[i].what);
  }
}

int main() {
  const int Ns[] = {128, 256, 512, 768, 1024, 1536, 4096};
  const int Ks[] = {64, 128, 192, 256, 512, 1024, 4096};
  for (int N : Ns)
    for (int K : Ks) {
      const W16 l = w16_layout(N, K);
      char ctx[64];
      snprintf(ctx, sizeof ctx, "w16 N=%d K=%d", N, K);
      disjoint({{l.hi, l.hi + (size_t)N * K * 2, "hi"}, {l.lo, l.lo + (size_t)N * K * 2, "lo"},
                {l.exp, l.exp + (size_t)N * 4, "exp"}}, l.bytes, ctx);
      CHECK(l.bytes <= (size_t)8 * N * K, "%s: %zu bytes exceed the TF32 hi/lo room", ctx, l.bytes);
    }
  // weight caches of the model shapes: GRU-256 (G*H = 768), BiLSTM-128 (512), and a few others
  const int cfg[][5] = {{2, 1, 256, 256, 768}, {2, 2, 1024, 256, 512}, {3, 2, 100, 512, 1024}, {8, 2, 64, 128, 256},
                        {1, 1, 96, 128, 384}, {2, 1, 36, 256, 768}};
  for (auto& c : cfg) {
    const int L = c[0], D = c[1], I = c[2], DH = c[3], GH = c[4];
    const WCache w = wcache_layout(L, D, I, DH, GH);
    std::vector<R> v;
    char ctx[96];
    snprintf(ctx, sizeof ctx, "wcache L=%d D=%d I=%d DH=%d GH=%d", L, D, I, DH, GH);
    for (int l = 0; l < L; ++l)
      for (int k = 0; k < D; ++k) {
        const int Il = l == 0 ? I : DH;
        const size_t f = (size_t)GH * Il * 4;
        v.push_back({w.hi[l][k], w.hi[l][k] + f, "tf32 hi"});
        v.push_back({w.lo[l][k], w.lo[l][k] + f, "tf32 lo"});
        if (shape_ok(GH, Il)) {
          const W16 l16 = w16_layout(GH, Il);
          v.push_back({w.h16[l][k] + l16.hi, w.h16[l][k] + l16.hi + (size_t)GH * Il * 2, "f16 hi"});
          v.push_back({w.h16[l][k] + l16.lo, w.h16[l][k] + l16.lo + (size_t)GH * Il * 2, "f16 lo"});
          v.push_back({w.h16[l][k] + l16.exp, w.h16[l][k] + l16.exp + (size_t)GH * 4, "f16 exp"});
        }
      }
    disjoint(v, w.total, ctx);
  }
  // the kernel's branch-free row exponent is h16::scale_exp, and exp2i(e) is 2^e, over every exponent field and a
  // spread of mantissas (zero, subnormals, normals, the largest finite value, Inf, NaN)
  const unsigned mants[] = {0u, 1u, 2u, 0x12345u, 0x400000u, 0x7fffffu};
  for (unsigned be = 0; be < 256; ++be)
    for (unsigned mt : mants) {
      const unsigned u = (be << 23) | mt;
      float m;
      memcpy(&m, &u, sizeof m);
      CHECK(scale_exp_bits(m) == b200rnn::h16::scale_exp(m), "scale_exp_bits(%a) = %d, scale_exp = %d", m,
            scale_exp_bits(m), b200rnn::h16::scale_exp(m));
    }
  for (int e = -126; e <= 126; ++e) CHECK(exp2i(e) == ldexpf(1.f, e), "exp2i(%d)", e);
  printf("fails %d\n", fails);
  return fails != 0;
}
"""


@pytest.mark.skipif(nvcc is None, reason="nvcc not available")
def test_layout_regions_are_in_bounds_aligned_and_disjoint(tmp_path):
    src = tmp_path / "layout.cu"
    src.write_text(PROGRAM)
    exe = tmp_path / "layout"
    subprocess.run([nvcc, "-std=c++17", "-I", CSRC, str(src), "-o", str(exe)], check=True, capture_output=True,
                   timeout=300)
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0, out.stdout
    assert "fails 0" in out.stdout


def test_cache_keeps_the_tf32_offsets_first():
    """the TF32 hi / lo blocks a frozen module's autograd and TF32 forwards read stay where they were: at the start of
    each (layer, direction) entry, hi then lo"""
    text = open(os.path.join(CSRC, "gemm_h16_layout.cuh")).read()
    body = text[text.index("inline WCache wcache_layout"):]
    assert body.index("w.hi[l][k] = off") < body.index("w.lo[l][k] = off") < body.index("w.h16[l][k] = off")
