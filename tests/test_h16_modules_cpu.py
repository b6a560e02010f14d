"""16-bit GRU / LSTM / RNN modules without a GPU: construction and conversion, parameter dtypes, the state dict and
init against stock torch, pickling and repr, torch's dtype errors, what stays float32 only, the ABI's flag checks, the
on-chip tier bounds of the 16-bit runtime-sized forward, and the resource usage of the new kernels."""
import io
import os
import re
import shutil
import subprocess

import pytest
import torch

import b200rnn
from b200rnn import _lib

DTYPES = (torch.float16, torch.bfloat16)
KINDS = {"gru": (b200rnn.GRU, torch.nn.GRU, {}), "lstm": (b200rnn.LSTM, torch.nn.LSTM, {}),
         "relu": (b200rnn.RNN, torch.nn.RNN, {"nonlinearity": "relu"})}
LIB = _lib.LIB_PATH


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("kind", sorted(KINDS))
def test_init_state_dict_pickle_repr_match_stock(kind, dt):
    mine_cls, stock_cls, kw = KINDS[kind]
    torch.manual_seed(7)
    mine = mine_cls(24, 48, num_layers=2, bidirectional=True, dtype=dt, **kw)
    torch.manual_seed(7)
    stock = stock_cls(24, 48, num_layers=2, bidirectional=True, dtype=dt, **kw)
    assert all(p.dtype == dt for p in mine.parameters())
    assert list(mine.state_dict()) == list(stock.state_dict())
    for a, b in zip(mine.state_dict().values(), stock.state_dict().values()):
        assert a.dtype == b.dtype and torch.equal(a, b)
    back = mine_cls(24, 48, num_layers=2, bidirectional=True, dtype=dt, **kw)
    back.load_state_dict(stock.state_dict())
    buf = io.BytesIO()
    torch.save(back, buf)
    buf.seek(0)
    again = torch.load(buf, weights_only=False)
    assert all(torch.equal(a, b) for a, b in zip(again.parameters(), stock.parameters()))
    assert repr(mine).split("(", 1)[1] == repr(stock).split("(", 1)[1]


@pytest.mark.parametrize("kind", sorted(KINDS))
def test_half_bfloat16_and_to(kind):
    mine_cls, _, kw = KINDS[kind]
    m = mine_cls(8, 16, **kw)
    assert all(p.dtype == torch.float16 for p in m.half().parameters())
    assert all(p.dtype == torch.bfloat16 for p in m.bfloat16().parameters())
    assert all(p.dtype == torch.float32 for p in m.to(torch.float32).parameters())
    assert m.frozen_weight_cache() is None


@pytest.mark.parametrize("dt", DTYPES)
def test_input_dtype_mismatch_raises_what_torch_raises(dt):
    torch.manual_seed(0)
    mine, stock = b200rnn.GRU(4, 16, dtype=dt), torch.nn.GRU(4, 16, dtype=dt)
    x = torch.randn(3, 2, 4)

    def raised(f):
        with pytest.raises(Exception) as e:
            f()
        return type(e.value), str(e.value)

    assert raised(lambda: mine(x)) == raised(lambda: stock(x))


def test_float64_and_16bit_projection_raise():
    with pytest.raises(NotImplementedError):
        b200rnn.GRU(4, 16, dtype=torch.float64)
    for dt in DTYPES:
        with pytest.raises(NotImplementedError):
            b200rnn.LSTM(4, 128, proj_size=32, dtype=dt)
    with pytest.raises(NotImplementedError):
        b200rnn.GRUCell(4, 16, dtype=torch.float16)


def test_shell_fusions_reject_16bit_parameters():
    m = b200rnn.GRU(8, 16).half()
    with pytest.raises(_lib.B200RNNError, match="float32"):
        b200rnn.dp.GradBucket(m)
    with pytest.raises(_lib.B200RNNError, match="float32"):
        _lib.require_fp32_params(m.parameters(), "TrainStep")


def test_abi_flag_validation():
    lib = _lib.load()
    import ctypes
    both = _lib.FLAG_F16 | _lib.FLAG_BF16

    def ws(flags, proj=0, mode=_lib.LSTM, H=128):
        d = _lib.Desc(mode, 4, 5, 64, H, 2, 1, 1, 0.0, flags, proj)
        r, s = ctypes.c_size_t(0), ctypes.c_size_t(0)
        rc = lib.b200rnn_workspace_bytes(ctypes.byref(d), ctypes.byref(r), ctypes.byref(s))
        return rc, r.value, s.value

    assert ws(both)[0] == -2
    assert ws(_lib.FLAG_F16 | _lib.FLAG_PROJ, proj=32)[0] == -2
    assert ws(_lib.FLAG_BF16 | _lib.FLAG_PROJ, proj=64)[0] == -2
    rc32, r32, s32 = ws(0)
    rc16, r16, s16 = ws(_lib.FLAG_F16)
    assert rc32 == rc16 == 0 and r16 > r32 and s16 > s32   # the 16-bit extras sit behind the fp32 layout
    d = _lib.Desc(_lib.GRU, 1, 1, 64, 256, 1, 1, 0, 0.0, _lib.FLAG_F16)
    n = ctypes.c_size_t(0)
    assert lib.b200rnn_wcache_bytes(ctypes.byref(d), ctypes.byref(n)) == -2
    assert "float32 only" in lib.b200rnn_last_error().decode()


# The on-chip tier of the runtime-sized kernels: a hidden size keeps W_hh in shared memory when one of plan_anyh's
# candidate shapes (C in 2..16 with C <= H / 8, BS in 2..64, NT = HS * BS in whole warps up to 512) fits the 227 KB opt-in
# limit, by the library's own anyh_smem (exported for tests as b200rnn_debug_anyh_smem)
MAX_SMEM, MAX_NT = 232448, 512


def _smem():
    import ctypes
    lib = _lib.load()
    f = lib.b200rnn_debug_anyh_smem
    f.restype = ctypes.c_size_t
    f.argtypes = [ctypes.c_int] * 7
    return f


def _onchip(G, H, bwd, wbytes):
    smem = _smem()
    for C in (2, 4, 8, 16):
        if C > H // 8:
            continue
        HS = 8 * ((H // 8 + C - 1) // C)
        for BS in (2, 4, 8, 16, 32, 64):
            if (HS * BS + 31) // 32 * 32 <= MAX_NT and smem(G, H, C, BS, int(bwd), 1, wbytes) <= MAX_SMEM:
                return True
    return False


def _bound(G, bwd, wbytes):
    return max(H for H in range(16, 1025, 16) if _onchip(G, H, bwd, wbytes))


def test_onchip_tier_bounds_of_the_16bit_kernels():
    # forward: fp32 weights GRU 512, LSTM 432; 16-bit GRU 752, LSTM 640, every Elman size
    assert (_bound(3, False, 4), _bound(4, False, 4)) == (512, 432)
    assert (_bound(3, False, 2), _bound(4, False, 2), _bound(1, False, 2)) == (752, 640, 1024)
    # backward (BPTT): fp32 weights GRU 512, LSTM 384; 16-bit GRU 672, LSTM 592, every Elman size
    assert (_bound(3, True, 4), _bound(4, True, 4)) == (512, 384)
    assert (_bound(3, True, 2), _bound(4, True, 2), _bound(1, True, 2)) == (672, 592, 1024)
    for G in (3, 4):  # every size up to the bound is on chip, every one above it in the L2 tier
        for bwd in (False, True):
            top = _bound(G, bwd, 2)
            assert all(_onchip(G, H, bwd, 2) == (H <= top) for H in range(16, 1025, 16))


def test_new_kernels_use_no_local_memory_and_no_stack():
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
        if m and name and re.search(r"anyh16_(fwd|bwd)_kernel|gemm_n16_kernel|widen16_kernel|narrow16_kernel|"
                                    r"copy16_kernel|whh_prep16_kernel", name):
            seen[name] = (int(m.group(1)), int(m.group(2)))
    # 3 modes x VL x tier x 2 types, forward and backward
    assert len([n for n in seen if "anyh16_fwd_kernel" in n]) == 24, sorted(seen)
    assert len([n for n in seen if "anyh16_bwd_kernel" in n]) == 24, sorted(seen)
    assert len([n for n in seen if "whh_prep16_kernel" in n]) == 1
    assert len([n for n in seen if "gemm_n16_kernel" in n]) == 2
    assert all(v == (0, 0) for v in seen.values()), seen
