"""Mixed precision without a GPU: the validation of ``B200RNN_FLAG_F32_PARAMS`` (fp32 master parameters of a 16-bit
call), the workspace it sizes, the descriptor of a master-weight call, and the resource usage
of the rounding kernel."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest
import torch

import b200rnn
from b200rnn import _lib
from b200rnn.functional import RNNConfig, _make_desc

LIB = _lib.LIB_PATH
M = _lib.FLAG_F32_PARAMS


def _ws(flags, mode=_lib.LSTM, H=128, proj=0, L=2, D=1):
    lib = _lib.load()
    d = _lib.Desc(mode, 4, 5, 64, H, L, D, 1, 0.0, flags, proj)
    r, s = ctypes.c_size_t(0), ctypes.c_size_t(0)
    rc = lib.b200rnn_workspace_bytes(ctypes.byref(d), ctypes.byref(r), ctypes.byref(s))
    return rc, r.value, s.value


def test_flag_is_the_next_free_bit_and_the_abi_stays():
    assert M == 256
    assert _lib.load().b200rnn_version() == _lib.ABI_VERSION == 4


def test_flag_alone_is_invalid_and_with_proj_unsupported():
    lib = _lib.load()
    assert _ws(M)[0] == -1
    assert "B200RNN_FLAG_F16" in lib.b200rnn_last_error().decode()
    assert _ws(M | _lib.FLAG_TF32)[0] == -1
    assert _ws(M | _lib.FLAG_F16 | _lib.FLAG_PROJ, proj=32)[0] == -2
    assert _ws(M | _lib.FLAG_BF16 | _lib.FLAG_PROJ, H=256, proj=64)[0] == -2
    assert _ws(M | _lib.FLAG_F16 | _lib.FLAG_BF16)[0] == -2


def test_shell_entry_points_and_weight_cache_reject_the_flag():
    lib = _lib.load()
    for dt in (_lib.FLAG_F16, _lib.FLAG_BF16):
        d = _lib.Desc(_lib.GRU, 1, 1, 64, 256, 1, 1, 0, 0.0, dt | M)
        n = ctypes.c_size_t(0)
        assert lib.b200rnn_wcache_bytes(ctypes.byref(d), ctypes.byref(n)) == -2
        assert "float32 only" in lib.b200rnn_last_error().decode()
        # rejected before any pointer is read: the flag check comes first
        for fn in (lib.b200rnn_forward_fused, lib.b200rnn_backward_fused):
            assert fn(ctypes.byref(d), *_nulls(fn)) == -2
            assert "float32 only" in lib.b200rnn_last_error().decode()


def _nulls(fn):
    """NULL / zero for every argument after the descriptor"""
    return [0 if t in (ctypes.c_int, ctypes.c_int64, ctypes.c_uint64, ctypes.c_float) else None
            for t in fn.argtypes[1:]]


@pytest.mark.parametrize("mode,H,D", [(_lib.GRU, 256, 1), (_lib.LSTM, 128, 2), (_lib.GRU, 96, 2),
                                      (_lib.LSTM, 320, 1), (_lib.RNN_TANH, 64, 2)])
@pytest.mark.parametrize("dt", [_lib.FLAG_F16, _lib.FLAG_BF16])
def test_workspace_with_the_flag_covers_the_images(mode, H, D, dt):
    rc0, r0, s0 = _ws(dt, mode=mode, H=H, D=D)
    rc1, r1, s1 = _ws(dt | M, mode=mode, H=H, D=D)
    assert rc0 == rc1 == 0
    assert r1 == r0   # the reserve is the 16-bit call's
    # the scratch adds one 16-bit image of every weight_ih and weight_hh (each 256-byte aligned)
    G = {_lib.GRU: 3, _lib.LSTM: 4}.get(mode, 1)
    images = sum(G * H * (64 if l == 0 else D * H) * 2 + G * H * H * 2 for l in range(2) for _ in range(D))
    assert s1 >= s0 + images
    assert s1 - s0 <= images + 4 * D * 256


def test_descriptor_of_a_master_weight_config():
    cfg = RNNConfig(_lib.LSTM, 16, 32, 2, 1, 0.0, True, False, dtype=torch.float16, master_f32=True)
    desc = _make_desc(cfg, 2, 3, True)
    assert desc.flags & M and desc.flags & _lib.FLAG_F16 and not desc.flags & _lib.FLAG_BF16
    assert not _make_desc(RNNConfig(_lib.GRU, 16, 32, 1, 1, 0.0, True, False), 2, 3, True).flags & M
    assert b200rnn.LSTM(16, 32)._autocast_dtype() is None   # no autocast region
    assert not b200rnn.LSTM(16, 32)._config().master_f32


def test_rounding_kernel_uses_no_local_memory_and_no_stack():
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
        if m and name and "round16_multi_kernel" in name:
            seen[name] = (int(m.group(1)), int(m.group(2)))
    assert len(seen) == 1, sorted(seen)
    assert all(v == (0, 0) for v in seen.values()), seen
