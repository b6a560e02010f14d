"""Hidden sizes other than 128 / 256 on the host side: which sizes the descriptor takes, that the model-shell entry
points refuse them, the modules' parameters and state_dict at those sizes, and that the runtime-sized recurrence
kernels (csrc/rnn_anyh.cu, GRU / LSTM / Elman) compile without stack or local memory."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest
import torch

from b200rnn import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "icassp2022-depression_b200", "lib", "libb200rnn.so")
UNSUPPORTED = -2


@pytest.mark.parametrize("H", [16, 48, 64, 96, 112, 128, 192, 256, 320, 384, 512, 768, 1008, 1024])
@pytest.mark.parametrize("mode", [_lib.GRU, _lib.LSTM])
def test_descriptor_takes_multiples_of_16_up_to_1024(mode, H):
    reserve, scratch = _lib.workspace_bytes(_lib.Desc(mode, 5, 7, 33, H, 2, 2, 1, 0.3, 0))
    G = 3 if mode == _lib.GRU else 4
    assert reserve >= 4 * 7 * 5 * 2 * 2 * (G + 1) * H      # gates + extra of every (layer, direction)
    assert scratch >= 4 * G * H * H                         # the transposed W_hh of the backward


@pytest.mark.parametrize("H", [8, 100, 1040, 0, 24 + 1])
def test_other_hidden_sizes_are_rejected_with_a_message(H):
    with pytest.raises(_lib.B200RNNError) as ei:
        _lib.workspace_bytes(_lib.Desc(_lib.GRU, 4, 4, 16, H, 1, 1, 0, 0.0, 0))
    assert "hidden_size" in str(ei.value)


def test_model_shell_entry_points_reject_other_hidden_sizes():
    lib = _lib.load()
    d = _lib.Desc(_lib.GRU, 2, 3, 128, 64, 1, 1, 0, 0.0, 0)
    n = ctypes.c_size_t(0)
    assert lib.b200rnn_wcache_bytes(ctypes.byref(d), ctypes.byref(n)) == UNSUPPORTED
    assert b"hidden_size" in lib.b200rnn_last_error()
    # desc, x, xs_t, xs_b, params, y, ys_t, ys_b, h_n, c_n, reserve, scratch, seed, offset, rng_state, ln_gamma,
    # ln_beta, ln_eps, y_pool, lengths, wcache, prologue_done, stream
    assert lib.b200rnn_forward_fused(ctypes.byref(d), None, 0, 0, None, None, 0, 0, None, None, None, None, 0, 0, None,
                                     None, None, 1e-5, None, None, None, None, None) == UNSUPPORTED
    assert b"hidden_size" in lib.b200rnn_last_error()
    d128 = _lib.Desc(_lib.GRU, 2, 3, 128, 128, 1, 1, 0, 0.0, 0)
    assert lib.b200rnn_wcache_bytes(ctypes.byref(d128), ctypes.byref(n)) == 0 and n.value > 0


def test_projection_keeps_its_sizes():
    for H, P in ((64, 16), (64, 32), (512, 128)):
        with pytest.raises(_lib.B200RNNError, match="proj_size"):
            d = _lib.Desc(_lib.LSTM, 2, 3, 16, H, 1, 1, 0, 0.0, _lib.FLAG_PROJ)
            d.proj_size = P
            _lib.workspace_bytes(d)


@pytest.mark.parametrize("kind, H", [("gru", 64), ("lstm", 48), ("gru", 512), ("lstm", 1024)])
def test_from_torch_and_state_dict_round_trip(kind, H):
    import b200rnn

    torch.manual_seed(1)
    stock = (torch.nn.GRU if kind == "gru" else torch.nn.LSTM)(21, H, num_layers=2, bidirectional=True)
    mine = b200rnn.from_torch(stock)
    assert mine.hidden_size == H
    for (n1, p1), (n2, p2) in zip(stock.named_parameters(), mine.named_parameters()):
        assert n1 == n2 and torch.equal(p1, p2)
    back = (torch.nn.GRU if kind == "gru" else torch.nn.LSTM)(21, H, num_layers=2, bidirectional=True)
    back.load_state_dict(mine.state_dict())
    for p1, p2 in zip(stock.parameters(), back.parameters()):
        assert torch.equal(p1, p2)
    fresh = (b200rnn.GRU if kind == "gru" else b200rnn.LSTM)(21, H, num_layers=2, bidirectional=True)
    fresh.load_state_dict(stock.state_dict())
    assert all(torch.equal(a, b) for a, b in zip(fresh.parameters(), stock.parameters()))


def _anyh_kernels():
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
        if m and name and re.search(r"\d(anyh_\w+_kernel)I", name):
            seen[name] = (int(m.group(1)), int(m.group(2)))
    return seen


def test_gru_lstm_elman_runtime_sized_kernels_use_no_local_memory_and_no_stack():
    seen = _anyh_kernels()
    # forward and backward x GRU / LSTM / Elman (one instantiation for tanh and relu) x fixed / ragged x shared-memory /
    # L2 weights
    assert len([n for n in seen if "anyh_fwd_kernel" in n]) == 12, sorted(seen)
    assert len([n for n in seen if "anyh_bwd_kernel" in n]) == 12, sorted(seen)
    assert all(v == (0, 0) for v in seen.values()), {n: v for n, v in seen.items() if v != (0, 0)}
