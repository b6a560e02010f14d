"""Property test (hypothesis) over the nn.GRU / nn.LSTM argument space the drop-in supports (SURVEY.md §4):
random B in [1,130], T in [1,40], input widths that hit both GEMM paths (tensor cores: I % 32 == 0; FFMA: anything else),
H in {128, 256}, 1-2 layers, 1-2 directions, batch_first or not, ragged batch tails, B=1, T=1 — forward outputs and
all gradients against stock torch on CPU."""
import pytest
import torch
from hypothesis import HealthCheck, given, settings, strategies as st

pytestmark = pytest.mark.gpu


@settings(max_examples=14, deadline=None, derandomize=True,
          suppress_health_check=[HealthCheck.too_slow, HealthCheck.function_scoped_fixture])
@given(kind=st.sampled_from(["gru", "lstm"]), B=st.integers(1, 130), T=st.integers(1, 40),
       I=st.sampled_from([1, 5, 37, 64, 96, 256, 300, 1024]), H=st.sampled_from([128, 256]),
       L=st.integers(1, 2), bi=st.booleans(), bf=st.booleans(), seed=st.integers(0, 2 ** 16))
def test_random_configurations_match_torch_cpu(kind, B, T, I, H, L, bi, bf, seed):
    import b200rnn

    dev = torch.device("cuda:0")
    torch.manual_seed(seed)
    cls = torch.nn.GRU if kind == "gru" else torch.nn.LSTM
    ref = cls(I, H, num_layers=L, bidirectional=bi, batch_first=bf).eval()
    mine = b200rnn.from_torch(ref).to(dev).eval()
    x = torch.randn((B, T, I) if bf else (T, B, I))
    xr = x.clone().requires_grad_(True)
    xm = x.clone().to(dev).requires_grad_(True)
    outr, outm = ref(xr), mine(xm)
    yr, ym = outr[0], outm[0]
    sr = outr[1] if isinstance(outr[1], tuple) else (outr[1],)
    sm = outm[1] if isinstance(outm[1], tuple) else (outm[1],)
    assert (ym.cpu() - yr).abs().max().item() <= 1e-5
    w = torch.randn(yr.shape)
    lr_, lm_ = (yr * w).sum(), (ym * w.to(dev)).sum()
    for a, b in zip(sm, sr):
        assert (a.cpu() - b).abs().max().item() <= 1e-5
        ws = torch.randn(b.shape)
        lr_, lm_ = lr_ + (b * ws).sum(), lm_ + (a * ws.to(dev)).sum()
    lr_.backward()
    lm_.backward()
    torch.cuda.synchronize()

    def close(a, b):
        # 1e-4 of the largest entry, with an absolute floor of 1e-6: a 1-element gradient that is itself the
        # cancelling sum of hundreds of terms (B=T=I=1) has an fp32 noise floor of ~1e-7 whatever its magnitude
        return (a - b).abs().max().item() <= 1e-4 * b.abs().max().item() + 1e-6

    assert close(xm.grad.cpu(), xr.grad)
    for (n, pr), (_, pm) in zip(ref.named_parameters(), mine.named_parameters()):
        assert close(pm.grad.cpu(), pr.grad), n
