"""GRUCell / LSTMCell without a GPU: the module API against the stock cells (constructor, parameters, init, extra_repr,
state_dict both ways, pickling, from_torch, exception types and messages), host tensors failing loudly, descriptor
validation of the C ABI, and the cell kernels compiled without stack or local memory."""
import ctypes
import io
import math
import os
import re
import shutil
import subprocess

import pytest
import torch

import b200rnn
from b200rnn import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "icassp2022-depression_b200", "lib", "libb200rnn.so")
STOCK = {"gru": torch.nn.GRUCell, "lstm": torch.nn.LSTMCell}
MINE = {"gru": b200rnn.GRUCell, "lstm": b200rnn.LSTMCell}


def _raised(fn):
    try:
        fn()
    except Exception as e:  # noqa: BLE001 - the exception itself is what is compared
        return e
    return None


@pytest.mark.parametrize("kind", ["gru", "lstm"])
@pytest.mark.parametrize("bias", [True, False])
def test_parameters_match_the_stock_cell(kind, bias):
    torch.manual_seed(0)
    stock = STOCK[kind](7, 5, bias=bias)
    mine = MINE[kind](7, 5, bias=bias)
    assert [(n, tuple(p.shape)) for n, p in mine.named_parameters()] == \
           [(n, tuple(p.shape)) for n, p in stock.named_parameters()]
    assert list(mine.state_dict()) == list(stock.state_dict())
    assert (mine.bias_ih is None) == (not bias) and mine.bias == bias
    assert repr(mine).split("(", 1)[1] == repr(stock).split("(", 1)[1]
    assert type(mine).__name__ == type(stock).__name__


@pytest.mark.parametrize("kind", ["gru", "lstm"])
def test_default_init_is_uniform_within_one_over_sqrt_hidden(kind):
    torch.manual_seed(0)
    mine = MINE[kind](64, 100)
    bound = 1 / math.sqrt(100)
    for p in mine.parameters():
        assert p.abs().max() <= bound and p.abs().max() > 0.9 * bound
    torch.manual_seed(3)
    stock = STOCK[kind](64, 100)
    torch.manual_seed(3)
    mine = MINE[kind](64, 100)
    for a, b in zip(mine.parameters(), stock.parameters()):
        assert torch.equal(a, b)  # same draws in the same order


@pytest.mark.parametrize("kind", ["gru", "lstm"])
@pytest.mark.parametrize("bias", [True, False])
def test_state_dict_interchange_pickle_and_from_torch(kind, bias):
    torch.manual_seed(1)
    stock = STOCK[kind](6, 4, bias=bias)
    mine = MINE[kind](6, 4, bias=bias)
    mine.load_state_dict(stock.state_dict())
    back = STOCK[kind](6, 4, bias=bias)
    back.load_state_dict(mine.state_dict())
    for a, b in zip(back.parameters(), stock.parameters()):
        assert torch.equal(a, b)
    buf = io.BytesIO()
    torch.save(mine, buf)
    buf.seek(0)
    again = torch.load(buf, weights_only=False)
    assert type(again) is type(mine)
    for a, b in zip(again.parameters(), stock.parameters()):
        assert torch.equal(a, b)
    stock.eval()
    twin = b200rnn.from_torch(stock)
    assert type(twin) is MINE[kind] and twin.bias == bias and not twin.training
    for a, b in zip(twin.parameters(), stock.parameters()):
        assert torch.equal(a, b)


def test_non_float32_dtype_is_not_implemented():
    for cls in MINE.values():
        with pytest.raises(NotImplementedError):
            cls(4, 4, dtype=torch.float64)


def test_install_leaves_the_cells_alone():
    b200rnn.install()
    try:
        assert torch.nn.GRUCell is STOCK["gru"] and torch.nn.LSTMCell is STOCK["lstm"]
        cell = torch.nn.GRUCell(3, 2)
        assert cell(torch.randn(4, 3)).shape == (4, 2)  # host code keeps running on stock torch
    finally:
        b200rnn.uninstall()


def _hx(kind, *shape):
    h = torch.zeros(*shape)
    return h if kind == "gru" else (h, torch.zeros(*shape))


@pytest.mark.parametrize("kind", ["gru", "lstm"])
@pytest.mark.parametrize("case", [
    # (input shape, hx shape or None)
    ((3, 7), None),          # wrong input size
    ((3, 8), (4, 16)),       # wrong batch
    ((3, 8), (3, 15)),       # wrong hidden size
    ((3, 8), (16,)),         # 1-D state for batched input
    ((8,), (3, 16)),         # 2-D state for unbatched input
    ((8,), (15,)),           # unbatched, wrong hidden size
    ((2, 3, 8), None),       # 3-D input
    ((3, 8), (1, 3, 16)),    # 3-D state
])
def test_shape_errors_match_torch(kind, case):
    xshape, hshape = case
    torch.manual_seed(0)
    stock, mine = STOCK[kind](8, 16), MINE[kind](8, 16)
    x = torch.randn(*xshape)
    args = (x,) if hshape is None else (x, _hx(kind, *hshape))
    want, got = _raised(lambda: stock(*args)), _raised(lambda: mine(*args))
    assert want is not None and got is not None
    assert type(got) is type(want) and str(got) == str(want)


def test_lstm_state_errors_match_torch():
    stock, mine = STOCK["lstm"](8, 16), MINE["lstm"](8, 16)
    x = torch.randn(3, 8)
    for hx in ((torch.zeros(3, 16), torch.zeros(3, 15)), (torch.zeros(3, 16), torch.zeros(2, 16)),
               (torch.zeros(3, 16),), torch.zeros(3, 16)):
        want, got = _raised(lambda: stock(x, hx)), _raised(lambda: mine(x, hx))
        assert want is not None and type(got) is type(want) and str(got) == str(want), hx


@pytest.mark.parametrize("kind", ["gru", "lstm"])
def test_host_tensors_raise_not_implemented(kind):
    mine = MINE[kind](8, 16)
    for args in ((torch.randn(3, 8),), (torch.randn(8),), (torch.randn(3, 8), _hx(kind, 3, 16))):
        e = _raised(lambda: mine(*args))
        assert isinstance(e, NotImplementedError) and isinstance(e, _lib.NoCPUPathError), args[0].shape
        assert "no CPU path" in str(e)


# ---- C ABI ------------------------------------------------------------------------------------------------------


def test_cell_symbols_are_bound():
    lib = _lib.load()
    for name in ("b200rnn_cell_workspace_bytes", "b200rnn_cell_forward", "b200rnn_cell_backward"):
        assert name in _lib.SYMBOLS and getattr(lib, name).argtypes is not None
    assert _lib.ABI_VERSION == lib.b200rnn_version() == 4


@pytest.mark.parametrize("desc,frag", [
    (_lib.CellDesc(7, 4, 16, 16, 0), "mode"),
    (_lib.CellDesc(_lib.GRU, -1, 16, 16, 0), "bad shape"),
    (_lib.CellDesc(_lib.GRU, 4, 0, 16, 0), "bad shape"),
    (_lib.CellDesc(_lib.LSTM, 4, 16, 0, 0), "bad shape"),
    (_lib.CellDesc(_lib.GRU, 4, 16, 16, _lib.FLAG_FUSED_LN), "unknown flags"),
    (_lib.CellDesc(_lib.LSTM, 4, 16, 16, _lib.FLAG_PROJ), "unknown flags"),
    (_lib.CellDesc(_lib.GRU, (1 << 20) + 1, 16, 16, 0), "too large"),
    (_lib.CellDesc(_lib.LSTM, 4, 1 << 20, 1 << 10, 0), "too large"),
])
def test_invalid_cell_descriptors_are_rejected_with_a_message(desc, frag):
    with pytest.raises(_lib.B200RNNError) as ei:
        _lib.cell_workspace_bytes(desc)
    assert frag in str(ei.value)


def test_cell_workspace_holds_one_step_of_the_sequence_reserve():
    # hidden sizes the sequence ABI rejects (test_abi.py: 100) are fine for a cell, and so is bias=False
    for mode, G in ((_lib.GRU, 3), (_lib.LSTM, 4)):
        for flags in (0, _lib.FLAG_NO_BIAS | _lib.FLAG_TF32 | _lib.FLAG_ACCUMULATE_GRADS):
            saved, scratch = _lib.cell_workspace_bytes(_lib.CellDesc(mode, 9, 40, 100, flags))
            gates = (9 * G * 100 + 63) // 64 * 64
            assert saved == 4 * (gates + (9 * 100 + 63) // 64 * 64)
            assert scratch >= 4 * 9 * G * 100
    assert _lib.cell_workspace_bytes(_lib.CellDesc(_lib.GRU, 0, 1, 1, 0))[0] == 0


FAKE = ctypes.c_void_p(256)  # never dereferenced: every call below must fail in its argument checks


def test_cell_entry_points_reject_bad_arguments_before_touching_the_device():
    lib = _lib.load()
    gru = _lib.CellDesc(_lib.GRU, 2, 8, 16, 0)
    nob = _lib.CellDesc(_lib.GRU, 2, 8, 16, _lib.FLAG_NO_BIAS)
    lstm = _lib.CellDesc(_lib.LSTM, 2, 8, 16, _lib.FLAG_SAVE_FOR_BACKWARD)
    params = _lib.ptr_array([256, 512, 768, 1024])
    fwd = lambda d, x, c, c_out, p, saved=None, x_ld=8: lib.b200rnn_cell_forward(  # noqa: E731
        ctypes.byref(d), x, x_ld, None, 0, c, 16, p, FAKE, c_out, saved, None)
    assert fwd(gru, FAKE, FAKE, None, params) == -1 and b"no cell state" in lib.b200rnn_last_error()
    assert fwd(gru, None, None, None, params) == -1 and b"null pointer" in lib.b200rnn_last_error()
    assert fwd(nob, FAKE, None, None, params) == -1 and b"bias pointers" in lib.b200rnn_last_error()
    assert fwd(gru, FAKE, None, None, _lib.ptr_array([256, None, 768, 1024])) == -1
    assert b"null weight" in lib.b200rnn_last_error()
    assert fwd(gru, FAKE, None, None, params, x_ld=4) == -1 and b"row stride" in lib.b200rnn_last_error()
    assert fwd(lstm, FAKE, None, FAKE, params) == -1 and b"saved-state" in lib.b200rnn_last_error()
    dparams = _lib.ptr_array([None, None, FAKE.value, None])
    bwd = lambda d: lib.b200rnn_cell_backward(  # noqa: E731
        ctypes.byref(d), FAKE, 8, None, 0, None, 0, params, None, None, None, None, None, None, dparams, None, None)
    assert bwd(nob) == -1 and b"NO_BIAS" in lib.b200rnn_last_error()
    assert bwd(gru) == -1 and b"null pointer" in lib.b200rnn_last_error()


def _cell_kernels():
    """(STACK, LOCAL) of every cell_* kernel, by mangled name"""
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([cuobjdump, "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    seen, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"STACK:(\d+) .*LOCAL:(\d+)", line)
        if m and name and re.search(r"\d(cell_\w+_kernel)I", name):
            seen[name] = (int(m.group(1)), int(m.group(2)))
    return seen


def test_cell_kernels_use_no_local_memory_and_no_stack():
    seen = _cell_kernels()
    # forward: GRU / LSTM x 3xTF32 / TF32; backward: GRU / LSTM
    assert len(seen) == 6, sorted(seen)
    assert all(v == (0, 0) for v in seen.values()), {n: v for n, v in seen.items() if v != (0, 0)}
