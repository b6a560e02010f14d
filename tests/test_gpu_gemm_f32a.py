"""The input projection's fp32-A GEMM: A is read in fp32 by TMA (in place through its row map) and split into TF32
hi / lo in shared memory. The MMAs see exactly the operands of the presplit path, so C must be bitwise equal to the
generic GEMM entry (which splits A in a separate pass), plain and streamed, for dense and batch-first A."""
import ctypes

import pytest
import torch

from b200rnn import _lib

pytestmark = pytest.mark.gpu

# audio layer 0, text layer 0, and a row count that is not a multiple of the 128-row tile
SHAPES = [(15360, 768, 256), (3840, 512, 1024), (1000, 384, 256)]


def _gemm_f32a(A, W, bias, M, a_st, a_sb=0, a_batch=0, streamed=False):
    lib = _lib.load()
    fn = lib.b200rnn_debug_gemm_f32a
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64,
                   ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
                   ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    N, K = W.shape
    dev = W.device
    out = torch.empty(M, N, device=dev)
    sbytes = 8 * (M + N) * K + 4096
    scratch = torch.empty(sbytes, dtype=torch.uint8, device=dev)
    tiles_m = (M + 127) // 128
    ready = torch.zeros(tiles_m, dtype=torch.int32, device=dev) if streamed else None
    rc = fn(M, N, K, A.data_ptr(), a_st, a_sb, a_batch, W.data_ptr(), out.data_ptr(), bias.data_ptr(),
            ready.data_ptr() if streamed else None, 8 if streamed else 0, scratch.data_ptr(), sbytes,
            torch.cuda.current_stream(dev).cuda_stream)
    _lib.check(rc, "b200rnn_debug_gemm_f32a")
    torch.cuda.synchronize()
    if streamed:  # every row tile published once per column tile
        assert torch.equal(ready.cpu(), torch.full((tiles_m,), N // 128, dtype=torch.int32))
    return out


def _inputs(M, N, K, seed):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(M, K, generator=g)
    W = torch.randn(N, K, generator=g) / K ** 0.5
    bias = torch.randn(N, generator=g)
    dev = torch.device("cuda:0")
    return A.to(dev), W.to(dev), bias.to(dev)


@pytest.mark.parametrize("streamed", [False, True])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_f32a_matches_presplit_bitwise(M, N, K, streamed):
    import b200rnn

    A, W, bias = _inputs(M, N, K, M + N + K)
    ref = b200rnn.gemm(A, W, bias=bias)  # generic entry: split pass, then the presplit GEMM
    out = _gemm_f32a(A, W, bias, M, a_st=K, streamed=streamed)
    assert torch.equal(out, ref), (out - ref).abs().max().item()
    exact = (A.double() @ W.double().t() + bias.double())
    assert (out.double() - exact).abs().max().item() < 5e-6 * exact.abs().max().item()


@pytest.mark.parametrize("streamed", [False, True])
@pytest.mark.parametrize("B,T,N,K", [(128, 120, 768, 256), (128, 30, 512, 1024), (32, 37, 384, 256), (256, 5, 768, 256)])
def test_f32a_batch_first_in_place_matches_dense_copy(B, T, N, K, streamed):
    """x [B][T][K] batch-first, rows m = t * B + b: the 3-D tensor map reads it in place."""
    import b200rnn

    M = T * B
    _, W, bias = _inputs(1, N, K, B + T)
    g = torch.Generator().manual_seed(B * T)
    x = torch.randn(B, T, K, generator=g).to(W.device)
    dense = x.transpose(0, 1).contiguous().view(M, K)
    ref = _gemm_f32a(dense, W, bias, M, a_st=K)
    out = _gemm_f32a(x, W, bias, M, a_st=K, a_sb=T * K, a_batch=B, streamed=streamed)
    assert torch.equal(out, ref), (out - ref).abs().max().item()
    assert torch.equal(ref, b200rnn.gemm(dense, W, bias=bias))
