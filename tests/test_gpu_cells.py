"""GRUCell / LSTMCell on the GPU.

A cell is exactly one step, so the per-step float64 bound of test_gpu_numerics_f64.py applies unchanged: every element
of h' (and c') must satisfy |kernel - step64| <= KAPPA * u * S, with S the magnitude oracle.rnn_numpy.gru_step /
lstm_step return, KAPPA = 24, u = 2^-24 (3xTF32) or 2^-11 (TF32 mode). Gradients are compared with float64 autograd on
the CPU within the sequence tests' relative budget. Also: rows that are not 16-byte aligned, B = 0, the accumulate flag of
the C ABI, determinism, CUDA-graph capture, and 120 steps against the sequence module with the same weights."""
import contextlib
import ctypes

import numpy as np
import pytest
import torch

import b200rnn
from b200rnn import _lib
from oracle.rnn_numpy import gru_step, lstm_step

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KAPPA = 24.0
U32, U_TF32 = 2.0 ** -24, 2.0 ** -11
GRAD_RTOL = 1e-4        # tests/test_gpu_parity.py
TF32_GRAD_RTOL = 4e-3   # single-pass TF32 operands: 2^-11 per product instead of ~2^-22
STOCK = {"gru": torch.nn.GRUCell, "lstm": torch.nn.LSTMCell}
BATCHES = (1, 7, 8, 9, 130, 1024)
SHAPES = ((1, 1), (3, 5), (256, 256), (1024, 128), (40, 1000), (257, 129))
# (bias, hx given, TF32 mode): each flag both ways
VARIANTS = ((True, True, False), (False, False, False), (True, False, True), (False, True, True))


@contextlib.contextmanager
def _tf32(on):
    old = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "tf32" if on else "ieee"
    try:
        yield
    finally:
        torch.backends.cuda.matmul.fp32_precision = old


def _pair(kind, I, H, bias, scale=1.0, seed=0):
    """stock cell (CPU, fp32) and its b200rnn twin on the GPU; scale > 1: saturating weights and biases U(-3, 3)"""
    torch.manual_seed(seed)
    stock = STOCK[kind](I, H, bias=bias)
    with torch.no_grad():
        for n, p in stock.named_parameters():
            if scale != 1.0:
                p.copy_(p * scale if n.startswith("weight") else torch.empty_like(p).uniform_(-3, 3))
    return stock, b200rnn.from_torch(stock).to(DEV)


def _np(t):
    return t.detach().double().cpu().numpy()


def _params(stock, G, H):
    b = [stock.bias_ih, stock.bias_hh] if stock.bias else [torch.zeros(G * H)] * 2
    return [_np(stock.weight_ih), _np(stock.weight_hh), _np(b[0]), _np(b[1])]


def _check_step(kind, stock, x, hx, out, u):
    """out of the kernel against the float64 step from the same inputs, elementwise within KAPPA * u * S"""
    H = stock.hidden_size
    B = x.shape[0]
    h = _np(hx[0] if kind == "lstm" else hx) if hx is not None else np.zeros((B, H))
    if kind == "gru":
        want, S = gru_step(_np(x), h, *_params(stock, 3, H))
        pairs = [(out, want, S)]
    else:
        c = _np(hx[1]) if hx is not None else np.zeros((B, H))
        hw, cw, Sh, Sc = lstm_step(_np(x), h, c, *_params(stock, 4, H))
        pairs = [(out[0], hw, Sh), (out[1], cw, Sc)]
    for got, want, S in pairs:
        ratio = np.abs(_np(got) - want) / (KAPPA * u * S)
        assert ratio.max(initial=0.0) <= 1.0, ratio.max()


def _inputs(kind, B, I, H, hx_given, seed=1, x_scale=1.0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, I, generator=g) * x_scale
    if not hx_given:
        return x, None
    h = torch.rand(B, H, generator=g) * 2 - 1
    return x, (h if kind == "gru" else (h, torch.randn(B, H, generator=g)))


def _dev(hx):
    if hx is None:
        return None
    return tuple(s.to(DEV) for s in hx) if isinstance(hx, tuple) else hx.to(DEV)


@pytest.mark.parametrize("kind", ["gru", "lstm"])
@pytest.mark.parametrize("IH", SHAPES, ids=lambda s: f"I{s[0]}H{s[1]}")
@pytest.mark.parametrize("B", BATCHES)
def test_one_step_against_float64(kind, IH, B):
    I, H = IH
    for bias, hx_given, tf32 in VARIANTS:
        stock, mine = _pair(kind, I, H, bias)
        x, hx = _inputs(kind, B, I, H, hx_given)
        with torch.no_grad(), _tf32(tf32):
            out = mine(x.to(DEV), _dev(hx))
            if B == 1:  # unbatched: the same step
                hx1 = None if hx is None else (tuple(s[0] for s in _dev(hx)) if kind == "lstm" else _dev(hx)[0])
                out1 = mine(x[0].to(DEV), hx1)
        torch.cuda.synchronize()
        _check_step(kind, stock, x, hx, out, U_TF32 if tf32 else U32)
        if B == 1:
            want = out if kind == "gru" else out[0]
            got = out1 if kind == "gru" else out1[0]
            assert got.shape == (H,) and torch.equal(got, want[0])


@pytest.mark.parametrize("kind", ["gru", "lstm"])
@pytest.mark.parametrize("bias", [True, False])
def test_saturating_weights_against_float64(kind, bias):
    for I, H in ((256, 256), (257, 129), (40, 1000)):
        stock, mine = _pair(kind, I, H, bias, scale=4.0)
        x, hx = _inputs(kind, 130, I, H, True, x_scale=2.0)
        for tf32 in (False, True):
            with torch.no_grad(), _tf32(tf32):
                out = mine(x.to(DEV), _dev(hx))
            _check_step(kind, stock, x, hx, out, U_TF32 if tf32 else U32)


def _relmax(a, b):
    return (np.abs(_np(a) - _np(b)).max() / max(np.abs(_np(b)).max(), 1e-30))


def _grads(kind, cell, x, hx, dout):
    """forward + backward of `cell` (any device / dtype) on leaf copies; returns the gradients by name"""
    dev, dt = cell.weight_ih.device, cell.weight_ih.dtype
    x = x.to(dev, dt).requires_grad_(True)
    hx = None if hx is None else tuple(s.to(dev, dt).requires_grad_(True) for s in
                                       (hx if isinstance(hx, tuple) else (hx,)))
    out = cell(x, hx if hx is None or kind == "lstm" else hx[0])
    outs = out if kind == "lstm" else (out,)
    loss = sum((o * d.to(dev, dt)).sum() for o, d in zip(outs, dout))
    loss.backward()
    g = {"x": x.grad}
    for i, s in enumerate(hx or ()):
        g[f"hx{i}"] = s.grad
    for n, p in cell.named_parameters():
        g[n] = p.grad
    return g


@pytest.mark.parametrize("kind", ["gru", "lstm"])
@pytest.mark.parametrize("IH", SHAPES, ids=lambda s: f"I{s[0]}H{s[1]}")
@pytest.mark.parametrize("B", (1, 9, 130))
def test_gradients_against_float64_autograd(kind, IH, B):
    I, H = IH
    for bias, hx_given, tf32 in VARIANTS:
        stock, mine = _pair(kind, I, H, bias)
        x, hx = _inputs(kind, B, I, H, hx_given)
        g = torch.Generator().manual_seed(7)
        dout = [torch.randn(B, H, generator=g) for _ in range(2 if kind == "lstm" else 1)]
        want = _grads(kind, stock.double(), x, hx, dout)
        with _tf32(tf32):
            got = _grads(kind, mine, x, hx, dout)
        assert sorted(got) == sorted(want)
        for n in want:
            assert _relmax(got[n], want[n]) <= (TF32_GRAD_RTOL if tf32 else GRAD_RTOL), (n, bias, hx_given, tf32)


@pytest.mark.parametrize("kind", ["gru", "lstm"])
def test_rows_that_are_not_16_byte_aligned(kind):
    """input, state and weight rows at an odd float offset into larger buffers"""
    B, I, H = 9, 256, 128
    G = 3 if kind == "gru" else 4
    stock, mine = _pair(kind, I, H, True)
    with torch.no_grad():
        for name in ("weight_ih", "weight_hh"):
            p = getattr(mine, name)
            buf = torch.zeros(p.numel() + 1, device=DEV)
            buf[1:].copy_(p.reshape(-1))
            setattr(mine, name, torch.nn.Parameter(buf[1:].view(G * H, -1)))
            assert getattr(mine, name).data_ptr() % 16 != 0
    x, hx = _inputs(kind, B, I, H, True)

    def shifted(t):
        buf = torch.zeros(t.numel() + 3, device=DEV)
        v = buf[3:].view_as(t)
        v.copy_(t)
        return v

    xs = shifted(x.to(DEV))
    hs = tuple(shifted(s.to(DEV)) for s in hx) if kind == "lstm" else shifted(hx.to(DEV))
    with torch.no_grad():
        out = mine(xs, hs)
    _check_step(kind, stock, x, hx, out, U32)
    # and the gradients through the same views
    g = torch.Generator().manual_seed(7)
    dout = [torch.randn(B, H, generator=g) for _ in range(2 if kind == "lstm" else 1)]
    want = _grads(kind, stock.double(), x, hx, dout)
    got = _grads(kind, mine, x, hx, dout)
    for n in want:
        assert _relmax(got[n], want[n]) <= GRAD_RTOL, n


@pytest.mark.parametrize("kind", ["gru", "lstm"])
def test_empty_batch(kind):
    _, mine = _pair(kind, 12, 20, True)
    x = torch.zeros(0, 12, device=DEV, requires_grad=True)
    out = mine(x)
    outs = out if kind == "lstm" else (out,)
    assert all(o.shape == (0, 20) for o in outs)
    sum(o.sum() for o in outs).backward()
    assert x.grad.shape == (0, 12)
    for n, p in mine.named_parameters():
        assert p.grad is not None and torch.count_nonzero(p.grad).item() == 0, n


def _abi_step(kind, mine, x, h, c, dh_out, dc_out, dparams, accumulate):
    """forward (saving) and backward through the C ABI, gradients into `dparams`"""
    lib = _lib.load()
    B, I = x.shape
    H = mine.hidden_size
    flags = _lib.FLAG_SAVE_FOR_BACKWARD | (_lib.FLAG_ACCUMULATE_GRADS if accumulate else 0)
    desc = _lib.CellDesc(_lib.GRU if kind == "gru" else _lib.LSTM, B, I, H, flags)
    sv, sc = _lib.cell_workspace_bytes(desc)
    saved = torch.empty(sv, dtype=torch.uint8, device=DEV)
    scratch = torch.empty(sc, dtype=torch.uint8, device=DEV)
    params = _lib.ptr_array([p.data_ptr() for p in mine.parameters()])
    h_out = torch.empty(B, H, device=DEV)
    c_out = torch.empty(B, H, device=DEV) if kind == "lstm" else None
    ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.b200rnn_cell_forward(ctypes.byref(desc), x.data_ptr(), I, h.data_ptr(), H, ptr(c), H, params,
                                        h_out.data_ptr(), ptr(c_out), saved.data_ptr(), st), "cell_forward")
    _lib.check(lib.b200rnn_cell_backward(ctypes.byref(desc), x.data_ptr(), I, h.data_ptr(), H, ptr(c), H, params,
                                         dh_out.data_ptr(), ptr(dc_out), saved.data_ptr(), None, None, None,
                                         _lib.ptr_array([t.data_ptr() for t in dparams]), scratch.data_ptr(), st),
               "cell_backward")


@pytest.mark.parametrize("kind", ["gru", "lstm"])
@pytest.mark.parametrize("IH", ((256, 256), (40, 1000)), ids=lambda s: f"I{s[0]}H{s[1]}")
def test_accumulate_flag_adds_into_existing_gradients(kind, IH):
    I, H = IH
    B = 33
    _, mine = _pair(kind, I, H, True)
    g = torch.Generator().manual_seed(3)
    x, h, c, dh, dc = (torch.randn(B, n, generator=g).to(DEV) for n in (I, H, H, H, H))
    c, dc = (c, dc) if kind == "lstm" else (None, None)
    fresh = [torch.empty_like(p) for p in mine.parameters()]
    _abi_step(kind, mine, x, h, c, dh, dc, fresh, accumulate=False)
    base = [torch.randn(p.shape, generator=g).to(DEV) for p in mine.parameters()]
    acc = [b.clone() for b in base]
    _abi_step(kind, mine, x, h, c, dh, dc, acc, accumulate=True)
    torch.cuda.synchronize()
    for a, b, f in zip(acc, base, fresh):
        assert _relmax(a - b, f) <= 1e-5


@pytest.mark.parametrize("kind", ["gru", "lstm"])
def test_two_runs_are_bit_identical(kind):
    B, I, H = 130, 257, 129
    stock, mine = _pair(kind, I, H, True)
    x, hx = _inputs(kind, B, I, H, True)
    g = torch.Generator().manual_seed(7)
    dout = [torch.randn(B, H, generator=g) for _ in range(2 if kind == "lstm" else 1)]
    runs = []
    for _ in range(2):
        mine.zero_grad(set_to_none=True)
        runs.append({k: v.clone() for k, v in _grads(kind, mine, x, hx, dout).items()})
    for k in runs[0]:
        assert torch.equal(runs[0][k], runs[1][k]), k


@pytest.mark.parametrize("kind", ["gru", "lstm"])
def test_captured_step_loop_matches_the_eager_loop_bitwise(kind):
    B, I, H, T = 8, 256, 256, 120
    _, mine = _pair(kind, I, H, True)
    xs = torch.randn(T, B, I, generator=torch.Generator().manual_seed(5)).to(DEV)

    def loop():
        state = None
        for t in range(T):
            state = mine(xs[t], state)
        return state if kind == "lstm" else (state,)

    with torch.no_grad():
        eager = [s.clone() for s in loop()]
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            loop()  # warm-up on the capturing stream's side, as torch.cuda.graphs recommends
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            captured = loop()
        graph.replay()
        torch.cuda.synchronize()
    for a, b in zip(eager, captured):
        assert torch.equal(a, b)


@pytest.mark.parametrize("kind", ["gru", "lstm"])
def test_120_steps_track_the_sequence_module(kind):
    """The cells with the weights of a 1-layer b200rnn.GRU / LSTM follow its output step by step: each step within twice
    the float64 per-step bound (each side's own step error), not bitwise (the contraction orders differ)."""
    B, I, H, T = 16, 256, 256, 120
    torch.manual_seed(0)
    seq = (b200rnn.GRU if kind == "gru" else b200rnn.LSTM)(I, H).to(DEV)
    cell = (b200rnn.GRUCell if kind == "gru" else b200rnn.LSTMCell)(I, H).to(DEV)
    with torch.no_grad():
        for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"):
            getattr(cell, n).copy_(getattr(seq, f"{n}_l0"))
    x = torch.randn(T, B, I, device=DEV)
    params = [_np(getattr(cell, n)) for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
    with torch.no_grad(), _tf32(False):
        y = seq(x)[0]
        state = None
        h_prev, c_prev = np.zeros((B, H)), np.zeros((B, H))
        for t in range(T):
            state = cell(x[t], state)
            h = state if kind == "gru" else state[0]
            if kind == "gru":
                _, S = gru_step(_np(x[t]), h_prev, *params)
            else:
                _, _, S, _ = lstm_step(_np(x[t]), h_prev, c_prev, *params)
                c_prev = _np(state[1])
            ratio = np.abs(_np(h) - _np(y[t])) / (2 * KAPPA * U32 * S)
            assert ratio.max() <= 1.0, (t, ratio.max())
            h_prev = _np(h)
