"""The no-grad forward's fp16-pair input projection (gemm_f16x3_kernel) on the GPU.

* Every element against float64 within kappa u S + F (tests/gemm_h16_bound.py derives the bound), at the audio and text
  shapes, K in {64, 128, 256, 1024} and M tails; on sharp operands as well as random ones.
* A NaN or Inf in a row of A reaches only that row, where the 3xTF32 fp32-A path gives non-finite values too.
* Streamed runs (ready counters, 4-CTA clusters) equal serial runs bitwise; runs repeat bitwise; CUDA-graph replay equals
  eager.
* The fused no-grad forward runs it and the module forward does not (B200RNN_DEBUG). That the cached
  (b200rnn_prepare_weights) and uncached weights give bit-identical outputs is tests/test_gpu_models.py's frozen-cache
  test, which now runs this kernel."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT
from b200rnn import _lib
from gemm_h16_bound import bound

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)

_ARGT = [ctypes.c_int] * 3 + [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int] + [ctypes.c_void_p] * 4 + \
    [ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]


def _fn(name):
    f = getattr(_lib.load(), name)
    f.restype = ctypes.c_int
    f.argtypes = _ARGT
    return f


def _gemm(A, W, bias, h16=True, ready=None, clusters=0, C=None):
    M, K = A.shape
    N = W.shape[0]
    if C is None:
        C = torch.full((M, N), float("nan"), device=DEV)
    sbytes = 8 * (M + N) * K + 4096
    scratch = torch.empty(sbytes, dtype=torch.uint8, device=DEV)
    f = _fn("b200rnn_debug_gemm_f16a" if h16 else "b200rnn_debug_gemm_f32a")
    rc = f(M, N, K, A.data_ptr(), K, 0, 0, W.data_ptr(), C.data_ptr(), bias.data_ptr(),
           None if ready is None else ready.data_ptr(), clusters, scratch.data_ptr(), sbytes,
           torch.cuda.current_stream(DEV).cuda_stream)
    _lib.check(rc, "debug gemm")
    return C


def _operands(M, N, K, kind, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "sharp":
        A = torch.rand(M, K, generator=g, dtype=torch.float64).add(1).half().double() * (1 + 2.0 ** -12)
        W = torch.rand(N, K, generator=g, dtype=torch.float64).add(1).half().double() * (1 + 2.0 ** -12)
        A = A * torch.exp2(torch.randint(-20, 21, (M, 1), generator=g).double())
        W = W * torch.exp2(torch.randint(-20, 21, (N, 1), generator=g).double())
        A, W = A.float(), W.float()
    else:
        A = torch.randn(M, K, generator=g)
        W = torch.randn(N, K, generator=g) / K ** 0.5
    b = torch.randn(N, generator=g)
    return A.to(DEV), W.to(DEV), b.to(DEV)


def _check_bound(C, A, W, b):
    C64, bnd = bound(A.cpu().numpy(), W.cpu().numpy(), b.cpu().numpy())
    err = np.abs(C.cpu().double().numpy() - C64)
    ratio = float((err / bnd).max())
    assert np.isfinite(ratio) and ratio <= 1.0, ratio
    return ratio


@pytest.mark.parametrize("M,N,K", [(15360, 768, 256), (3840, 512, 1024), (3840, 512, 256), (1000, 768, 64),
                                   (200, 256, 128), (129, 128, 1024)])
@pytest.mark.parametrize("kind", ["random", "sharp"])
def test_against_float64(M, N, K, kind):
    A, W, b = _operands(M, N, K, kind, M + K)
    C = _gemm(A, W, b)
    torch.cuda.synchronize()
    _check_bound(C, A, W, b)


def test_non_finite_rows_stay_in_their_row():
    M, N, K = 300, 256, 256
    A, W, b = _operands(M, N, K, "random", 1)
    A[5, 17] = float("nan")
    A[140, 200] = float("inf")
    A[299, 0] = float("-inf")
    C = _gemm(A, W, b)
    C32 = _gemm(A, W, b, h16=False)
    torch.cuda.synchronize()
    bad = ~torch.isfinite(C)
    rows = [5, 140, 299]
    assert bad[rows].all()
    assert torch.equal(bad, ~torch.isfinite(C32))
    keep = [m for m in range(M) if m not in rows]
    _check_bound(C[keep], A[keep], W, b)


def test_streamed_equals_serial_and_repeats():
    M, N, K = 15360, 768, 256
    A, W, b = _operands(M, N, K, "random", 2)
    C0 = _gemm(A, W, b)
    C1 = _gemm(A, W, b)
    ready = torch.zeros(M // 128, dtype=torch.int32, device=DEV)
    Cs = _gemm(A, W, b, ready=ready, clusters=8)
    torch.cuda.synchronize()
    assert torch.equal(C0, C1)
    assert torch.equal(C0, Cs)
    assert (ready == N // 128).all()


def test_graph_replay_equals_eager():
    M, N, K = 3840, 512, 1024
    A, W, b = _operands(M, N, K, "random", 3)
    eager = _gemm(A, W, b)
    C = torch.zeros(M, N, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        _gemm(A, W, b, C=C)
    C.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(C, eager)


_FWD = r"""
import sys, torch
sys.path[:0] = [{root!r}, {pkg!r}]
import b200rnn
torch.manual_seed(0)
dev = torch.device("cuda", 0)
gru = b200rnn.from_torch(torch.nn.GRU(256, 256, num_layers=2, batch_first=True)).to(dev).eval()
x = torch.randn(128, 30, 256, device=dev)
ln = torch.nn.LayerNorm(256).to(dev)
with torch.no_grad():
    gru(x)
    print("MARK fused", file=sys.stderr, flush=True)
    gru.forward_ln_sum(x, ln)
"""


def test_fused_nograd_forward_runs_fp16_pairs_and_the_module_forward_does_not():
    code = _FWD.format(root=ROOT, pkg=os.path.join(ROOT, "icassp2022-depression_b200"))
    proc = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, B200RNN_DEBUG="1"), capture_output=True,
                          text=True, timeout=600)
    assert proc.returncode == 0, proc.stderr[-2000:]
    module, fused = proc.stderr.split("MARK fused")
    pick = lambda txt: [ln for ln in txt.splitlines() if "forward x-projection:" in ln]  # noqa: E731
    # the module's own forward is not the fused entry: it keeps 3xTF32; the fused no-grad one takes fp16 pairs
    assert pick(module) and all("math=3xtf32" in ln for ln in pick(module)), pick(module)
    assert pick(fused) and all("math=f16x3" in ln for ln in pick(fused)), pick(fused)
