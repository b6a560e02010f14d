"""CPU tests of oracle.stacked, the layered reference of tests/test_gpu_stacked_f64.py: with no dropout the chain of stock
one-layer modules is stock ``nn.GRU`` / ``nn.LSTM`` (also with ``proj_size``) / ``nn.RNN(num_layers=L)`` in float64 -
outputs, final states and every gradient, fixed-length and packed, with hx - and with masks it is the per-layer
composition test_gpu_shell_f64.py checks the inter-layer dropout against."""
import numpy as np
import pytest
import torch

from oracle import philox
from oracle.stacked import chained, split_layers

CASES = {
    "gru_bi": (torch.nn.GRU, dict(), True),
    "lstm": (torch.nn.LSTM, dict(), False),
    "lstm_proj_bi": (torch.nn.LSTM, dict(proj_size=5), True),
    "rnn_tanh_bi": (torch.nn.RNN, dict(nonlinearity="tanh"), True),
    "rnn_relu": (torch.nn.RNN, dict(nonlinearity="relu"), False),
}


def _stock(name, L, I=7, H=9, dropout=0.0):
    cls, kw, bi = CASES[name]
    torch.manual_seed(0)
    return cls(I, H, num_layers=L, bidirectional=bi, dropout=dropout, **kw).double()


def _inputs(ref, T, B, ragged, seed=1):
    g = torch.Generator().manual_seed(seed)
    D, HO = (2 if ref.bidirectional else 1), (ref.proj_size or ref.hidden_size)
    x = torch.randn(T, B, ref.input_size, generator=g, dtype=torch.float64)
    hx = [torch.randn(ref.num_layers * D, B, HO, generator=g, dtype=torch.float64)]
    if isinstance(ref, torch.nn.LSTM):
        hx.append(torch.randn(ref.num_layers * D, B, ref.hidden_size, generator=g, dtype=torch.float64))
    lens = torch.tensor([T, 1] + [int(v) for v in torch.randint(1, T + 1, (B - 2,), generator=g)]) if ragged else None
    wy = torch.randn(T, B, D * HO, generator=g, dtype=torch.float64)
    ws = [torch.randn(s.shape, generator=g, dtype=torch.float64) for s in hx]
    return x, hx, lens, wy, ws


def _grads(loss, tensors):
    return [g for g in torch.autograd.grad(loss, tensors)]


@pytest.mark.parametrize("ragged", [False, True], ids=["fixed", "packed"])
@pytest.mark.parametrize("L", [2, 3])
@pytest.mark.parametrize("name", list(CASES))
def test_chain_without_dropout_is_the_stock_stack(name, L, ragged):
    ref = _stock(name, L)
    layers = split_layers(ref)
    assert len(layers) == L and all(m.num_layers == 1 for m in layers)
    T, B = 6, 5
    x, hx, lens, wy, ws = _inputs(ref, T, B, ragged)
    xs = [x.clone().requires_grad_(True) for _ in range(2)]
    hs = [[s.clone().requires_grad_(True) for s in hx] for _ in range(2)]
    inp = xs[0] if lens is None else torch.nn.utils.rnn.pack_padded_sequence(xs[0], lens, enforce_sorted=False)
    out, st = ref(inp, tuple(hs[0]) if len(hx) == 2 else hs[0][0])
    y0 = out if lens is None else torch.nn.utils.rnn.pad_packed_sequence(out, total_length=T)[0]
    st0 = st if isinstance(st, tuple) else (st,)
    y1, st1 = chained(layers, xs[1], lens, tuple(hs[1]) if len(hx) == 2 else hs[1][0])
    for a, b in zip((y0, *st0), (y1, *st1)):
        assert a.shape == b.shape and (a - b).abs().max().item() <= 1e-12
    losses = [(y * wy).sum() + sum((s * w).sum() for s, w in zip(sts, ws)) for y, sts in ((y0, st0), (y1, st1))]
    g0 = _grads(losses[0], [xs[0], *hs[0], *ref.parameters()])
    params1 = [getattr(layers[int(n.split("_l")[1][0])], n.split("_l")[0] + "_l0" + n.split("_l")[1][1:])
               for n, _ in ref.named_parameters()]
    g1 = _grads(losses[1], [xs[1], *hs[1], *params1])
    for a, b in zip(g0, g1):
        assert (a - b).abs().max().item() <= 1e-12


@pytest.mark.parametrize("ragged", [False, True], ids=["fixed", "packed"])
@pytest.mark.parametrize("name", ["gru_bi", "lstm", "lstm_proj_bi", "rnn_tanh_bi"])
def test_chain_with_masks_is_the_per_layer_composition(name, ragged):
    """the Philox factors of each layer (stream = layer index) multiply that layer's output, as in
    test_gpu_shell_f64.py::test_inter_layer_dropout_masks_are_the_oracles, in float64 and in fp32"""
    L, T, B, p = 3, 6, 5, 0.3
    ref = _stock(name, L, dropout=p)
    D, HO = (2 if ref.bidirectional else 1), (ref.proj_size or ref.hidden_size)
    n = T * B * D * HO
    masks = [torch.from_numpy(philox.dropout_factor(0xC0FFEE, 99, l, n, p).reshape(T, B, D * HO)).double()
             for l in range(L - 1)]
    x, _, lens, _, _ = _inputs(ref, T, B, ragged)
    for dtype in (torch.float64, torch.float32):
        stock = ref.to(dtype)
        per = split_layers(stock)
        h = x.to(dtype)
        for l, m in enumerate(per):   # the composition of test_gpu_shell_f64.py
            if ragged:
                h = torch.nn.utils.rnn.pad_packed_sequence(
                    m(torch.nn.utils.rnn.pack_padded_sequence(h, lens, enforce_sorted=False))[0], total_length=T)[0]
            else:
                h = m(h)[0]
            if l < L - 1:
                h = h * masks[l].to(dtype)
        y, _ = chained(per, x.to(dtype), lens, masks=[mk.to(dtype) for mk in masks])
        assert torch.equal(y, h), dtype
    dropped = sum(int((mk == 0).sum()) for mk in masks)
    assert 0.2 * n * (L - 1) < dropped < 0.4 * n * (L - 1)
    assert np.isclose(masks[0].max().item(), 1 / 0.7, rtol=1e-6)
