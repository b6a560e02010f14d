"""The Elman RNN (``RNN`` / ``RNNCell``, tanh and relu) on the host side: which descriptors the C ABI takes and refuses,
the workspace sizes of one gate block, the modules' constructor checks, repr, state_dict interchange with the stock
modules, pickling and ``from_torch``, and that the Elman cell and bias kernels (cell.cu, misc_kernels.cu) compile
without stack or local memory. The Elman recurrence runs the runtime-sized kernels, checked in test_any_hidden_cpu.py."""
import ctypes
import os
import pickle
import re
import shutil
import subprocess

import pytest
import torch

import b200rnn
from b200rnn import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "icassp2022-depression_b200", "lib", "libb200rnn.so")
UNSUPPORTED = -2
FAKE = ctypes.c_void_p(256)  # never dereferenced: every call that takes it must fail in its argument checks
ELMAN = [_lib.RNN_TANH, _lib.RNN_RELU]
NONLIN = {"tanh": _lib.RNN_TANH, "relu": _lib.RNN_RELU}


def _round(n):
    return (n + 63) // 64 * 64


@pytest.mark.parametrize("mode", ELMAN)
def test_descriptor_takes_every_multiple_of_16_up_to_1024(mode):
    for H in range(16, 1025, 16):
        reserve, scratch = _lib.workspace_bytes(_lib.Desc(mode, 5, 7, 33, H, 1, 1, 1, 0.0, 0))
        # header, then one saved block [T,B,H]: no second block as the GRU / LSTM keep
        assert reserve == 4 * (64 + _round(7 * 5 * H) + 64)
        assert scratch >= 4 * H * H  # the transposed W_hh of the backward


@pytest.mark.parametrize("mode", ELMAN)
def test_reserve_holds_one_block_per_layer_and_direction_plus_the_layer_outputs(mode):
    T, B, H, L, D = 7, 5, 48, 3, 2
    for p in (0.0, 0.25):
        reserve, _ = _lib.workspace_bytes(_lib.Desc(mode, B, T, 33, H, L, D, 1, p, 0))
        layer_out = (L - 1) * _round(T * B * D * H) * (2 if p > 0 else 1)  # ylayer (and ydrop with dropout)
        assert reserve == 4 * (64 + L * D * _round(T * B * H) + layer_out + 64)


@pytest.mark.parametrize("mode", ELMAN)
@pytest.mark.parametrize("H", [8, 100, 1040, 0, 24 + 1])
def test_other_hidden_sizes_are_rejected_with_a_message(mode, H):
    with pytest.raises(_lib.B200RNNError) as ei:
        _lib.workspace_bytes(_lib.Desc(mode, 4, 4, 16, H, 1, 1, 0, 0.0, 0))
    assert "hidden_size" in str(ei.value)


@pytest.mark.parametrize("mode", ELMAN)
def test_projection_is_rejected(mode):
    d = _lib.Desc(mode, 2, 3, 16, 128, 1, 1, 0, 0.0, _lib.FLAG_PROJ)
    d.proj_size = 32
    with pytest.raises(_lib.B200RNNError, match="proj_size"):
        _lib.workspace_bytes(d)


def test_unknown_modes_are_still_rejected():
    for mode in (4, 7, -1):
        with pytest.raises(_lib.B200RNNError, match="mode"):
            _lib.workspace_bytes(_lib.Desc(mode, 4, 4, 16, 128, 1, 1, 0, 0.0, 0))
        with pytest.raises(_lib.B200RNNError, match="mode"):
            _lib.cell_workspace_bytes(_lib.CellDesc(mode, 4, 16, 16, 0))


@pytest.mark.parametrize("mode", ELMAN)
@pytest.mark.parametrize("H", [128, 256])
def test_model_shell_entry_points_return_unsupported(mode, H):
    lib = _lib.load()
    d = _lib.Desc(mode, 2, 3, 128, H, 1, 1, 0, 0.0, 0)
    n = ctypes.c_size_t(0)
    assert lib.b200rnn_wcache_bytes(ctypes.byref(d), ctypes.byref(n)) == UNSUPPORTED
    assert b"mode" in lib.b200rnn_last_error()
    assert lib.b200rnn_prepare_weights(ctypes.byref(d), FAKE, FAKE, None) == UNSUPPORTED
    # desc, x, xs_t, xs_b, params, y, ys_t, ys_b, h_n, c_n, reserve, scratch, seed, offset, rng_state, ln_gamma,
    # ln_beta, ln_eps, y_pool, lengths, wcache, prologue_done, stream
    assert lib.b200rnn_forward_fused(ctypes.byref(d), None, 0, 0, None, None, 0, 0, None, None, None, None, 0, 0, None,
                                     None, None, 1e-5, None, None, None, None, None) == UNSUPPORTED
    # desc, x, xs_t, xs_b, params, y, ys_t, ys_b, dy, dys_t, dys_b, dy_pool, dy_pool_scale, dh_n, dc_n, reserve,
    # scratch, dx, dxs_t, dxs_b, dparams, lengths, ln_gamma, ln_eps, dln_gamma, dln_beta, stream
    assert lib.b200rnn_backward_fused(ctypes.byref(d), None, 0, 0, None, None, 0, 0, None, 0, 0, None, 1.0, None, None,
                                      None, None, None, 0, 0, None, None, None, 1e-5, None, None, None) == UNSUPPORTED
    assert b"mode" in lib.b200rnn_last_error()


def test_cell_state_is_refused_before_touching_the_device():
    lib = _lib.load()
    params = _lib.ptr_array([256, 512, 768, 1024])
    for mode in ELMAN:
        d = _lib.CellDesc(mode, 2, 8, 16, 0)
        assert lib.b200rnn_cell_forward(ctypes.byref(d), FAKE, 8, None, 0, FAKE, 16, params, FAKE, None, None,
                                        None) == -1
        assert b"no cell state" in lib.b200rnn_last_error()
    # the sequence hx entry point: c_0 is an LSTM's alone
    d = _lib.Desc(_lib.RNN_TANH, 2, 3, 16, 64, 1, 1, 0, 0.0, 0)
    assert lib.b200rnn_forward_hx(ctypes.byref(d), FAKE, 0, 0, params, FAKE, 0, 0, FAKE, FAKE, FAKE, None, None, FAKE,
                                  0, 0, None, None, None) == -1
    assert b"no cell state" in lib.b200rnn_last_error()


@pytest.mark.parametrize("mode", ELMAN)
def test_cell_workspace_holds_one_gate_block(mode):
    for flags in (0, _lib.FLAG_NO_BIAS, _lib.FLAG_NO_BIAS | _lib.FLAG_TF32 | _lib.FLAG_ACCUMULATE_GRADS):
        saved, scratch = _lib.cell_workspace_bytes(_lib.CellDesc(mode, 9, 40, 100, flags))
        assert saved == 4 * _round(9 * 100)  # h' alone
        assert scratch >= 4 * 9 * 100
    assert _lib.cell_workspace_bytes(_lib.CellDesc(mode, 0, 1, 1, 0))[0] == 0


# ---- modules ------------------------------------------------------------------------------------------------------
def _raises_like(fn_stock, fn_mine):
    with pytest.raises(Exception) as e_stock:
        fn_stock()
    with pytest.raises(Exception) as e_mine:
        fn_mine()
    assert type(e_mine.value) is type(e_stock.value)
    assert str(e_mine.value) == str(e_stock.value)


@pytest.mark.parametrize("args, kw", [
    ((10, 32), dict(proj_size=4)),
    ((10, 32), dict(proj_size=0)),
    ((10, 32, 1, "sigmoid"), {}),
    ((10, 32), dict(nonlinearity="gelu")),
    ((10, 32), dict(dropout=1.5)),
    ((10, 32), dict(dropout=True)),
])
def test_constructor_errors_match_torch(args, kw):
    _raises_like(lambda: torch.nn.RNN(*args, **kw), lambda: b200rnn.RNN(*args, **kw))


def test_bias_false_is_not_implemented():
    with pytest.raises(NotImplementedError):
        b200rnn.RNN(10, 32, bias=False)


@pytest.mark.parametrize("args, kw", [
    ((10, 32), {}),
    ((10, 32, 2, "relu"), dict(batch_first=True, dropout=0.5, bidirectional=True)),
    ((10, 64), dict(nonlinearity="relu", num_layers=3)),
])
def test_repr_parameters_and_state_dict_round_trip(args, kw):
    torch.manual_seed(3)
    stock = torch.nn.RNN(*args, **kw)
    mine = b200rnn.RNN(*args, **kw)
    assert repr(mine) == repr(stock)
    assert mine.nonlinearity == stock.nonlinearity
    assert [(n, p.shape) for n, p in mine.named_parameters()] == [(n, p.shape) for n, p in stock.named_parameters()]
    stdv = 1.0 / stock.hidden_size ** 0.5
    assert all(p.abs().max() <= stdv for p in mine.parameters())
    mine.load_state_dict(stock.state_dict())
    back = torch.nn.RNN(*args, **kw)
    back.load_state_dict(mine.state_dict())
    assert all(torch.equal(a, b) for a, b in zip(back.parameters(), stock.parameters()))
    twin = b200rnn.from_torch(stock)
    assert isinstance(twin, b200rnn.RNN) and twin._mode == NONLIN[stock.nonlinearity]
    assert all(torch.equal(a, b) for a, b in zip(twin.parameters(), stock.parameters()))
    again = pickle.loads(pickle.dumps(twin))
    assert again._mode == twin._mode and repr(again) == repr(twin)
    assert all(torch.equal(a, b) for a, b in zip(again.parameters(), stock.parameters()))


@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("nonlinearity", ["tanh", "relu"])
def test_cell_matches_the_stock_cell(bias, nonlinearity):
    torch.manual_seed(4)
    stock = torch.nn.RNNCell(12, 40, bias, nonlinearity)
    mine = b200rnn.RNNCell(12, 40, bias, nonlinearity)
    assert repr(mine) == repr(stock)
    assert [(n, p.shape) for n, p in mine.named_parameters()] == [(n, p.shape) for n, p in stock.named_parameters()]
    mine.load_state_dict(stock.state_dict())
    back = torch.nn.RNNCell(12, 40, bias, nonlinearity)
    back.load_state_dict(mine.state_dict())
    assert all(torch.equal(a, b) for a, b in zip(back.parameters(), stock.parameters()))
    twin = b200rnn.from_torch(stock)
    assert isinstance(twin, b200rnn.RNNCell) and twin.nonlinearity == nonlinearity and twin.bias == bias
    again = pickle.loads(pickle.dumps(twin))
    assert repr(again) == repr(stock)
    assert all(torch.equal(a, b) for a, b in zip(again.parameters(), stock.parameters()))


def test_cell_shape_and_nonlinearity_errors_match_torch():
    for make_input in (lambda: torch.randn(2, 3, 12), lambda: torch.randn(())):
        _raises_like(lambda: torch.nn.RNNCell(12, 40)(make_input()), lambda: b200rnn.RNNCell(12, 40)(make_input()))
    _raises_like(lambda: torch.nn.RNNCell(12, 40)(torch.randn(2, 12), torch.randn(1, 2, 40)),
                 lambda: b200rnn.RNNCell(12, 40)(torch.randn(2, 12), torch.randn(1, 2, 40)))
    # an unknown nonlinearity is accepted by the constructor and fails at forward
    _raises_like(lambda: torch.nn.RNNCell(12, 40, nonlinearity="gelu")(torch.randn(2, 12)),
                 lambda: b200rnn.RNNCell(12, 40, nonlinearity="gelu")(torch.randn(2, 12)))


def test_host_tensors_raise_no_cpu_path():
    with pytest.raises(_lib.NoCPUPathError):
        b200rnn.RNN(10, 32)(torch.randn(3, 2, 10))
    with pytest.raises(_lib.NoCPUPathError):
        b200rnn.RNNCell(10, 32, nonlinearity="relu")(torch.randn(2, 10))


def test_install_leaves_rnn_and_rnncell_stock():
    stock_rnn, stock_cell = torch.nn.RNN, torch.nn.RNNCell
    b200rnn.install()
    try:
        assert torch.nn.RNN is stock_rnn and torch.nn.RNNCell is stock_cell
    finally:
        b200rnn.uninstall()


def test_no_fused_paths():
    m = b200rnn.RNN(128, 128)
    for p in m.parameters():
        p.requires_grad_(False)
    assert m.frozen_weight_cache() is None


# ---- kernels ------------------------------------------------------------------------------------------------------
def _elman_kernels():
    """(STACK, LOCAL) of every elman_* kernel, by mangled name"""
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
        if m and name and re.search(r"\d(elman_\w+_kernel)[IE]", name):
            seen[name] = (int(m.group(1)), int(m.group(2)))
    return seen


def test_elman_cell_kernels_use_no_local_memory_and_no_stack():
    seen = _elman_kernels()
    names = sorted(re.search(r"\d(elman_\w+_kernel)", n).group(1) for n in seen)
    # the nonlinearity is a runtime flag: the cell forward x 3xTF32 / TF32 (2), the cell backward (1), the bias
    # reduction (1); the recurrence runs anyh_fwd_kernel / anyh_bwd_kernel (test_any_hidden_cpu.py)
    assert names == sorted(["elman_cell_fwd_kernel"] * 2 + ["elman_cell_bwd_kernel", "elman_bias_reduce_kernel"]), names
    assert all(v == (0, 0) for v in seen.values()), {n: v for n, v in seen.items() if v != (0, 0)}
