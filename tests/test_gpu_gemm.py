"""GPU parity of the fp32 time-parallel GEMM (K1/K6) through the C-ABI, against torch CPU float64."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("M,N,K", [(7680, 768, 256), (1920, 1024, 1024), (100, 37, 53), (1, 512, 1024),
                                   (768, 256, 7680), (130, 130, 16), (64, 64, 1)])
@pytest.mark.parametrize("a_kc,b_kc", [(True, True), (True, False), (False, False), (False, True)])
def test_gemm_layouts(M, N, K, a_kc, b_kc):
    import b200rnn

    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(M * 31 + N * 7 + K)
    A = torch.randn(M, K, generator=g)
    B = torch.randn(K, N, generator=g)
    bias = torch.randn(N, generator=g)
    ref = (A.double() @ B.double() + bias.double()).float()
    a_in = (A if a_kc else A.t().contiguous()).to(dev)
    b_in = (B.t().contiguous() if b_kc else B).to(dev)
    out = b200rnn.gemm(a_in, b_in, a_kcontig=a_kc, b_kcontig=b_kc, bias=bias.to(dev))
    torch.cuda.synchronize()
    err = (out.cpu() - ref).abs().max().item()
    scale = ref.abs().max().item()
    # 4e-6 of the largest output: fp32 FFMA sits near 1e-6, the tensor-core 3xTF32 path (truncating fp32 accumulate
    # inside each k-block) a little above; plain TF32 would be ~1e-3
    assert err <= 4e-6 * scale * max(1.0, (K / 256) ** 0.5) + 1e-5, (err, scale)


def test_gemm_accumulate_and_no_splitk():
    import b200rnn

    dev = torch.device("cuda:0")
    A = torch.randn(300, 2048, device=dev)
    B = torch.randn(2048, 200, device=dev)
    C0 = torch.randn(300, 200, device=dev)
    out = C0.clone()
    b200rnn.gemm(A, B, b_kcontig=False, out=out, accumulate=True)
    out2 = C0.clone()
    b200rnn.gemm(A, B, b_kcontig=False, out=out2, accumulate=True, use_splitk=False)
    ref = (C0.double() + A.double() @ B.double()).float()
    assert (out - ref).abs().max().item() < 5e-4
    assert (out2 - ref).abs().max().item() < 5e-4


@pytest.mark.parametrize("M,N,K", [(15360, 768, 256), (3840, 512, 1024), (130, 384, 512), (1, 128, 32), (257, 1024, 256)])
def test_tcgen05_3xtf32_input_projection(M, N, K):
    """Eligible shapes (A, W k-contiguous, K % 32 == 0, N % 128 == 0) run on wgmma with the 3xTF32 split; the
    result must stay within fp32-FFMA-like error of the float64 product (plain TF32 would be ~1e-3 relative)."""
    import b200rnn

    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(M + N + K)
    A = torch.randn(M, K, generator=g)
    W = torch.randn(N, K, generator=g) / K ** 0.5
    bias = torch.randn(N, generator=g)
    ref = (A.double() @ W.double().t() + bias.double())
    out = b200rnn.gemm(A.to(dev), W.to(dev), bias=bias.to(dev))
    out_ffma = b200rnn.gemm(A.to(dev), W.to(dev), bias=bias.to(dev), use_splitk=False)  # no workspace => FFMA path
    torch.cuda.synchronize()
    err_tc = (out.cpu().double() - ref).abs().max().item()
    err_ffma = (out_ffma.cpu().double() - ref).abs().max().item()
    assert err_ffma < 5e-6 * ref.abs().max().item()
    assert err_tc < 5e-6 * ref.abs().max().item(), (err_tc, err_ffma)
