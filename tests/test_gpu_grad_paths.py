"""The backward's tensor-core fallbacks, against stock ``torch.nn.GRU`` / ``torch.nn.LSTM`` on CPU.

Every layer here (I = 256, H = 128) is tensor-core eligible, so each case takes a gradient GEMM off the tensor cores or
drops it: a gradient sink whose views sit 4 bytes off 16-byte alignment and already hold a gradient (the weight
gradients run on the FFMA GEMM and accumulate), a frozen ``weight_ih_l0`` (no dW_ih for layer 0), and an input that
does not require grad (no dX at layer 0). Gradients within 1e-4 relative to the largest entry, as
tests/test_gpu_proj.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GRAD_RTOL = 1e-4
I, H, L, B, T = 256, 128, 2, 6, 11


def _models(kind, bi):
    import b200rnn

    torch.manual_seed(0)
    cls = torch.nn.GRU if kind == "gru" else torch.nn.LSTM
    ref = cls(I, H, num_layers=L, bidirectional=bi, batch_first=True)
    return ref, b200rnn.from_torch(ref).to(DEV)


def _inputs(bi, seed=5):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, T, I, generator=g), torch.randn(B, T, (2 if bi else 1) * H, generator=g)


def _backward(model, x, wy, x_grad):
    """x.grad (None when x does not require grad) after sum(y * wy).backward()"""
    dev = next(model.parameters()).device
    xx = x.clone().to(dev).requires_grad_(x_grad)
    (model(xx)[0] * wy.to(dev)).sum().backward()
    return xx.grad


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


@pytest.mark.parametrize("kind", ["gru", "lstm"])
@pytest.mark.parametrize("bi", [False, True])
def test_misaligned_grad_sink_accumulates(kind, bi):
    ref, mine = _models(kind, bi)
    x, wy = _inputs(bi)
    names = [n for n, _ in mine.named_parameters()]
    params = dict(mine.named_parameters())
    # every view starts one float past a 256-byte boundary: none is 16-byte aligned
    offs, total = [], 0
    for n in names:
        offs.append(total + 1)
        total += (params[n].numel() + 1 + 63) // 64 * 64
    flat = torch.empty(total, device=DEV)
    views = {n: flat[o:o + params[n].numel()].view_as(params[n]) for n, o in zip(names, offs)}
    g = torch.Generator().manual_seed(9)
    before = {n: 0.5 * torch.randn(params[n].shape, generator=g) for n in names}
    for n in names:
        views[n].copy_(before[n])
        assert views[n].data_ptr() % 16 == 4
    by_ptr = {params[n].data_ptr(): views[n] for n in names}
    mine._grad_sink = lambda weights: [by_ptr[w.data_ptr()] for w in weights]

    dx = _backward(mine, x, wy, True)
    rdx = _backward(ref, x, wy, True)
    assert _rel(dx.cpu(), rdx) <= GRAD_RTOL
    for n, q in ref.named_parameters():
        assert params[n].grad is None, n  # the gradient went to the sink only
        assert _rel(views[n].cpu() - before[n], q.grad) <= GRAD_RTOL, n


@pytest.mark.parametrize("kind", ["gru", "lstm"])
@pytest.mark.parametrize("bi", [False, True])
def test_frozen_weight_ih_l0(kind, bi):
    ref, mine = _models(kind, bi)
    x, wy = _inputs(bi)
    for m in (ref, mine):
        m.weight_ih_l0.requires_grad_(False)
    dx = _backward(mine, x, wy, True)
    rdx = _backward(ref, x, wy, True)
    assert _rel(dx.cpu(), rdx) <= GRAD_RTOL
    assert mine.weight_ih_l0.grad is None
    params = dict(mine.named_parameters())
    for n, q in ref.named_parameters():
        if q.requires_grad:
            assert _rel(params[n].grad.cpu(), q.grad) <= GRAD_RTOL, n


@pytest.mark.parametrize("kind", ["gru", "lstm"])
@pytest.mark.parametrize("bi", [False, True])
def test_input_without_grad(kind, bi):
    ref, mine = _models(kind, bi)
    x, wy = _inputs(bi)
    assert _backward(mine, x, wy, False) is None
    _backward(ref, x, wy, False)
    params = dict(mine.named_parameters())
    for n, q in ref.named_parameters():
        assert _rel(params[n].grad.cpu(), q.grad) <= GRAD_RTOL, n
