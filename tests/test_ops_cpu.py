"""The ``b200rnn::`` custom ops without a GPU: schemas and mutation annotations, fake (shape) implementations against
stock torch's modules, the reserve size against ``b200rnn_workspace_bytes``, the autograd wiring and ``torch.export``.

Everything here runs on fake CUDA tensors (``FakeTensorMode``), which torch builds without a driver: the fake
implementations launch nothing and read no pointer. The library is loaded for its host-side workspace arithmetic only.
The two autograd-wiring cases are marked ``gpu``: autograd's engine sets up a device context for CUDA tensors, fake
ones included, and that needs a driver."""
import itertools
import os
import sys

import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "icassp2022-depression_b200"))
import b200rnn  # noqa: E402
from b200rnn import _lib  # noqa: E402
from b200rnn.functional import RNNConfig, _make_desc  # noqa: E402
from b200rnn.ops import _rnn_attrs  # noqa: E402

pytestmark = pytest.mark.skipif(not os.path.exists(_lib.LIB_PATH), reason="libb200rnn.so not built")

DTYPES = (torch.float32, torch.float16, torch.bfloat16)


def _fake():
    return FakeTensorMode(allow_non_fake_inputs=True)


def _same_meta(a: torch.Tensor, b: torch.Tensor):
    assert (tuple(a.shape), a.stride(), a.dtype) == (tuple(b.shape), b.stride(), b.dtype)


def test_ops_registered_with_schemas():
    ops = torch.ops.b200rnn
    fwd = ops.rnn_forward.default._schema
    mutated = [a.name for a in fwd.arguments if a.alias_info is not None and a.alias_info.is_write]
    assert mutated == ["rng_state"]
    assert [a.name for a in fwd.arguments[:6]] == ["x", "weights", "h_0", "c_0", "lengths", "rng_state"]
    assert [a.name for a in fwd.arguments[6:]] == ["kind", "input_size", "hidden_size", "num_layers", "num_dirs",
                                                   "proj_size", "dropout", "training", "batch_first", "tf32", "dtype",
                                                   "save"]
    assert len(fwd.returns) == 4
    for name in ("rnn_backward", "cell_forward", "cell_backward"):
        schema = getattr(ops, name).default._schema
        assert not schema.is_mutable, name
        assert all(a.alias_info is None for a in schema.arguments), name
    assert "bool[] needs" in str(ops.rnn_backward.default._schema)
    assert "bool[] needs" in str(ops.cell_backward.default._schema)
    assert str(ops.rnn_backward.default._schema).endswith("-> (Tensor, Tensor, Tensor, Tensor[])")


# (mode, stock class, kwargs)
_SEQ = [
    ("gru", torch.nn.GRU, {}),
    ("lstm", torch.nn.LSTM, {}),
    ("lstmp", torch.nn.LSTM, {"proj_size": 32}),
    ("tanh", torch.nn.RNN, {"nonlinearity": "tanh"}),
    ("relu", torch.nn.RNN, {"nonlinearity": "relu"}),
]
_OURS = {"gru": b200rnn.GRU, "lstm": b200rnn.LSTM, "lstmp": b200rnn.LSTM, "tanh": b200rnn.RNN, "relu": b200rnn.RNN}


def _seq_cases():
    for (kind, stock, kw), dtype, bf, bidi, L in itertools.product(_SEQ, DTYPES, (False, True), (False, True),
                                                                  (1, 2, 3)):
        if kind == "lstmp" and dtype != torch.float32:
            continue    # proj_size is float32 only
        yield kind, stock, kw, dtype, bf, bidi, L


@pytest.mark.parametrize("kind,stock,kw,dtype,batch_first,bidi,L", list(_seq_cases()))
@pytest.mark.parametrize("with_state,with_lengths", [(False, False), (True, False), (False, True)])
def test_rnn_forward_fake_matches_stock(kind, stock, kw, dtype, batch_first, bidi, L, with_state, with_lengths):
    T, B, I, H = 5, 3, 24, 128
    ref = stock(I, H, num_layers=L, batch_first=batch_first, bidirectional=bidi, **kw).to(dtype)
    D, HO = (2 if bidi else 1), kw.get("proj_size", 0) or H
    x = torch.randn(B, T, I) if batch_first else torch.randn(T, B, I)
    hx = None
    if with_state:
        h0 = torch.zeros(L * D, B, HO, dtype=dtype)
        hx = (h0, torch.zeros(L * D, B, H, dtype=dtype)) if stock is torch.nn.LSTM else h0
    y_ref, st_ref = ref(x.to(dtype), hx)
    h_ref, c_ref = st_ref if stock is torch.nn.LSTM else (st_ref, None)

    with _fake():
        mine = _OURS[kind](I, H, num_layers=L, batch_first=batch_first, bidirectional=bidi, device="cuda",
                           dtype=dtype, **kw)
        cfg = mine._config()
        xf = x.to(device="cuda", dtype=dtype)
        x_tm = xf.transpose(0, 1) if batch_first else xf
        h_0 = c_0 = None
        if with_state:
            h_0 = torch.zeros(L * D, B, HO, dtype=dtype, device="cuda")
            c_0 = torch.zeros(L * D, B, H, dtype=dtype, device="cuda") if stock is torch.nn.LSTM else None
        lengths = torch.full((B,), T, dtype=torch.int32, device="cuda") if with_lengths else None
        for save in (False, True):
            y, h_n, c_n, reserve = torch.ops.b200rnn.rnn_forward(x_tm, mine._flat_weights, h_0, c_0, lengths,
                                                                 mine._rng_state, *_rnn_attrs(cfg), save)
            # shape and dtype of stock torch's; dense like cuDNN's output (stock CPU returns a batch_first y as a
            # transposed view of its time-major buffer)
            assert (tuple(y.shape), y.dtype) == (tuple(y_ref.shape), y_ref.dtype) and y.is_contiguous()
            _same_meta(h_n, h_ref)
            if c_ref is not None:
                _same_meta(c_n, c_ref)
            else:
                assert tuple(c_n.shape) == (0,)
            rbytes, _ = _lib.workspace_bytes(_make_desc(cfg, B, T, save))
            assert reserve.dtype == torch.uint8
            assert reserve.numel() == (rbytes if save else 0)


@pytest.mark.parametrize("B,T", [(0, 4), (3, 0)])
def test_rnn_forward_fake_empty(B, T):
    with _fake():
        m = b200rnn.LSTM(16, 32, num_layers=2, bidirectional=True, device="cuda")
        y, h_n, c_n, reserve = torch.ops.b200rnn.rnn_forward(torch.randn(T, B, 16, device="cuda"), m._flat_weights,
                                                             None, None, None, m._rng_state, *_rnn_attrs(m._config()),
                                                             True)
    assert tuple(y.shape) == (T, B, 64) and tuple(h_n.shape) == tuple(c_n.shape) == (4, B, 32)
    cfg = RNNConfig(_lib.LSTM, 16, 32, 2, 2, 0.0, True, False)
    assert reserve.numel() == _lib.workspace_bytes(_make_desc(cfg, B, T, True))[0]


_CELLS = [(torch.nn.GRUCell, b200rnn.GRUCell, {}), (torch.nn.LSTMCell, b200rnn.LSTMCell, {}),
          (torch.nn.RNNCell, b200rnn.RNNCell, {"nonlinearity": "tanh"}),
          (torch.nn.RNNCell, b200rnn.RNNCell, {"nonlinearity": "relu"})]


@pytest.mark.parametrize("stock,ours,kw", _CELLS)
@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("with_state", [False, True])
def test_cell_forward_fake_matches_stock(stock, ours, kw, bias, with_state):
    B, I, H = 5, 24, 40
    ref = stock(I, H, bias=bias, **kw)
    x = torch.randn(B, I)
    hx = None
    if with_state:
        hx = (torch.zeros(B, H), torch.zeros(B, H)) if stock is torch.nn.LSTMCell else torch.zeros(B, H)
    out_ref = ref(x, hx)
    h_ref, c_ref = out_ref if stock is torch.nn.LSTMCell else (out_ref, None)
    with _fake():
        cell = ours(I, H, bias=bias, device="cuda", **kw)
        weights = [cell.weight_ih, cell.weight_hh] + ([cell.bias_ih, cell.bias_hh] if bias else [])
        h = torch.zeros(B, H, device="cuda") if with_state else None
        c = torch.zeros(B, H, device="cuda") if with_state and stock is torch.nn.LSTMCell else None
        for save in (False, True):
            h_out, c_out, saved = torch.ops.b200rnn.cell_forward(x.cuda(), h, c, weights, cell._mode, I, H, bias,
                                                                 False, save)
            _same_meta(h_out, h_ref)
            if c_ref is not None:
                _same_meta(c_out, c_ref)
            else:
                assert tuple(c_out.shape) == (0,)
            desc = b200rnn.functional._cell_desc(b200rnn.functional.CellConfig(cell._mode, I, H, bias), B, save)
            assert saved.numel() == (_lib.cell_workspace_bytes(desc)[0] if save else 0)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["gru", "lstm", "lstmp"])
def test_rnn_autograd_wiring_fake(kind):
    """backward of the op gives each requested gradient in its input's shape, and None where none is wanted"""
    kw = {"proj_size": 32} if kind == "lstmp" else {}
    with _fake():
        m = _OURS[kind](24, 128, num_layers=2, bidirectional=True, batch_first=True, device="cuda", **kw)
        m.weight_hh_l1.requires_grad_(False)
        x = torch.randn(3, 5, 24, device="cuda", requires_grad=True)
        HO = 32 if kind == "lstmp" else 128
        h_0 = torch.zeros(4, 3, HO, device="cuda", requires_grad=True)
        c_0 = torch.zeros(4, 3, 128, device="cuda") if kind != "gru" else None
        y, h_n, c_n, _ = torch.ops.b200rnn.rnn_forward(x.transpose(0, 1), m._flat_weights, h_0, c_0, None,
                                                       m._rng_state, *_rnn_attrs(m._config()), True)
        (y.sum() + h_n.sum() + c_n.sum()).backward()
    _same_meta(x.grad, x)
    _same_meta(h_0.grad, h_0)
    assert m.weight_hh_l1.grad is None
    for w in m._flat_weights:
        if w.requires_grad:
            _same_meta(w.grad, w)


@pytest.mark.gpu
def test_cell_autograd_wiring_fake():
    with _fake():
        cell = b200rnn.LSTMCell(24, 40, device="cuda")
        x = torch.randn(5, 24, device="cuda")
        h = torch.zeros(5, 40, device="cuda", requires_grad=True)
        c = torch.zeros(5, 40, device="cuda")
        weights = [cell.weight_ih, cell.weight_hh, cell.bias_ih, cell.bias_hh]
        h_out, c_out, _ = torch.ops.b200rnn.cell_forward(x, h, c, weights, _lib.LSTM, 24, 40, True, False, True)
        (h_out.sum() + c_out.sum()).backward()
    assert x.grad is None and c.grad is None
    _same_meta(h.grad, h)
    for w in weights:
        _same_meta(w.grad, w)


def test_export_traces_the_ops():
    with _fake():
        m = b200rnn.GRU(32, 64, num_layers=2, batch_first=True, dropout=0.2, device="cuda")
        cell = b200rnn.GRUCell(32, 64, device="cuda")
        x = torch.randn(3, 5, 32, device="cuda")
        ep = torch.export.export(m, (x,))
        ep_cell = torch.export.export(cell, (x[:, 0],))
    targets = [n.target for n in ep.graph.nodes if n.op == "call_function"]
    assert torch.ops.b200rnn.rnn_forward.default in targets
    assert "b__rng_state" in str(ep.graph)      # the module's Philox state is an input the op mutates
    assert torch.ops.b200rnn.cell_forward.default in [n.target for n in ep_cell.graph.nodes]


def test_export_with_grad_sink_raises():
    with _fake():
        m = b200rnn.GRU(32, 64, num_layers=2, device="cuda")
        m._grad_sink = lambda weights: weights
        with pytest.raises(b200rnn.B200RNNError, match="run it eagerly"):
            torch.export.export(m, (torch.randn(5, 3, 32, device="cuda"),))
