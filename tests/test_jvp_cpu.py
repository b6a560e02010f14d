"""Forward-mode AD (b200rnn_forward_tangent, functional._RNNFunction.jvp, func._Tangent) without a GPU: the binding,
the descriptor checks of the tangent entry point, the tangent kernels' resources and the Python refusals."""
import ctypes
import dataclasses
import os
import re
import shutil
import subprocess

import pytest
import torch

from b200rnn import _lib
from b200rnn import functional as F

OK, ERR_INVALID, ERR_UNSUPPORTED = 0, -1, -2
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "icassp2022-depression_b200", "lib", "libb200rnn.so")
HEADER = os.path.join(ROOT, "include", "b200rnn.h")


def _cfg(mode=_lib.GRU, H=64, L=2, D=2, **kw):
    return F.RNNConfig(mode=mode, input_size=24, hidden_size=H, num_layers=L, num_dirs=D, dropout=0.25, training=True,
                       batch_first=False, **kw)


def _tangent_call(desc, lengths=None):
    """the entry point on dummy (never dereferenced) pointers: every refusal comes before any launch"""
    lib = _lib.load()
    fake = 1 << 40
    n = 4 * desc.num_layers * desc.num_dirs
    params = _lib.ptr_array([fake] * n)
    lstm = desc.mode == _lib.LSTM
    rc = lib.b200rnn_forward_tangent(ctypes.byref(desc), fake, 1, 1, params, fake, 1, 1, None, None, fake, lengths,
                                     fake, None, None, None, fake, 1, 1, fake, fake if lstm else None, fake, None)
    return rc, lib.b200rnn_last_error().decode()


def test_header_binding_and_exports_include_the_tangent_entry():
    for name in ("b200rnn_forward_tangent", "b200rnn_tangent_workspace_bytes"):
        assert name in _lib.SYMBOLS
        assert re.search(rf"B200RNN_API int {name}\(", open(HEADER).read())
    lib = _lib.load()
    assert len(lib.b200rnn_forward_tangent.argtypes) == 23
    assert lib.b200rnn_forward_tangent.restype is ctypes.c_int
    assert _lib.ABI_VERSION == 4 == lib.b200rnn_version()


@pytest.mark.parametrize("what", ["proj", "f16", "bf16", "f32_params", "fused_ln", "lengths"])
def test_tangent_entry_refuses_what_forward_mode_does_not_run(what):
    cfg = _cfg(mode=_lib.LSTM, H=128, proj_size=32) if what == "proj" else _cfg()
    desc = F._make_desc(cfg, 8, 3, True)
    flags = {"f16": _lib.FLAG_F16, "bf16": _lib.FLAG_BF16, "f32_params": _lib.FLAG_F16 | _lib.FLAG_F32_PARAMS,
             "fused_ln": _lib.FLAG_FUSED_LN}
    desc.flags |= flags.get(what, 0)
    lengths = 1 << 40 if what == "lengths" else None
    rc, msg = _tangent_call(desc, lengths)
    assert rc == ERR_UNSUPPORTED, msg
    want = {"proj": "proj_size", "f16": "float32 only", "bf16": "float32 only", "f32_params": "float32 only",
            "fused_ln": "model-shell", "lengths": "lengths"}[what]
    assert want in msg and "forward mode" in msg, msg


@pytest.mark.parametrize("what", ["proj", "f16", "fused_ln"])
def test_tangent_workspace_query_refuses_the_same_descriptors(what):
    cfg = _cfg(mode=_lib.LSTM, H=128, proj_size=32) if what == "proj" else _cfg()
    desc = F._make_desc(cfg, 8, 3, True)
    desc.flags |= {"proj": 0, "f16": _lib.FLAG_F16, "fused_ln": _lib.FLAG_FUSED_LN}[what]
    with pytest.raises(_lib.B200RNNError, match="forward mode"):
        _lib.tangent_workspace_bytes(desc)


@pytest.mark.parametrize("mode", [_lib.GRU, _lib.LSTM, _lib.RNN_TANH])
def test_tangent_scratch_is_one_gemm_workspace_and_per_direction_tangent_buffers(mode):
    """per direction: D pre-activation blocks [T,B,G*H] (+ the GRU's [T,B,H] h side) and two inner-layer outputs
    [T,B,D*H], rounded to 256 bytes; the GEMM workspace is shared by every direction"""
    T, B, H, L, D = 5, 4, 48, 3, 2
    G = {_lib.GRU: 3, _lib.LSTM: 4, _lib.RNN_TANH: 1}[mode]
    cfg = _cfg(mode=mode, H=H, L=L, D=D)
    rnd = lambda n: (n + 63) // 64 * 64 * 4  # noqa: E731
    block = D * rnd(T * B * G * H) + (D * rnd(T * B * H) if mode == _lib.GRU else 0) + 2 * rnd(T * B * D * H)
    one = _lib.tangent_workspace_bytes(F._make_desc(cfg, B, T, True))
    many = _lib.tangent_workspace_bytes(F._make_desc(dataclasses.replace(cfg, models=160), B, T, True))
    assert many - one == 159 * block
    assert one - block < 4 << 20   # the shared GEMM workspace of this shape, not a backward's scratch per direction


def test_tangent_entry_checks_its_outputs_and_initial_states():
    desc = F._make_desc(_cfg(), 8, 3, True)
    lib = _lib.load()
    fake = 1 << 40
    params = _lib.ptr_array([fake] * 8)
    # a GRU has no cell state
    rc = lib.b200rnn_forward_tangent(ctypes.byref(desc), fake, 1, 1, params, fake, 1, 1, None, None, fake, None, fake,
                                     None, None, fake, fake, 1, 1, fake, None, fake, None)
    assert rc == ERR_INVALID and "cell state" in lib.b200rnn_last_error().decode()
    # y_dot and h_n_dot are required
    rc = lib.b200rnn_forward_tangent(ctypes.byref(desc), fake, 1, 1, params, fake, 1, 1, None, None, fake, None, fake,
                                     None, None, None, None, 1, 1, fake, None, fake, None)
    assert rc == ERR_INVALID and "y_dot" in lib.b200rnn_last_error().decode()


def test_tangent_kernels_use_no_local_memory_and_no_stack():
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
        if m and name and "anyh_tangent_kernel" in name:
            seen[name] = (int(m.group(1)), int(m.group(2)))
    # GRU / LSTM / Elman x shared-memory / L2 weights
    assert len(seen) == 6, sorted(seen)
    assert all(v == (0, 0) for v in seen.values()), seen


@pytest.mark.parametrize("case", ["proj", "f16", "autocast", "packed"])
def test_forward_mode_refusals_name_what_is_unsupported(case):
    cfg = {"proj": _cfg(mode=_lib.LSTM, H=128, proj_size=32), "f16": _cfg(dtype=torch.float16),
           "autocast": _cfg(dtype=torch.float16, master_f32=True), "packed": _cfg()}[case]
    lengths = torch.ones(8, dtype=torch.int32) if case == "packed" else None
    with pytest.raises(_lib.B200RNNError, match="forward-mode AD") as e:
        F.check_forward_ad(cfg, lengths)
    assert {"proj": "proj_size", "f16": "float32", "autocast": "autocast", "packed": "PackedSequence"}[case] in str(e.value)


def test_dual_tensors_are_detected_only_inside_a_dual_level():
    import torch.autograd.forward_ad as fwAD
    x = torch.randn(3)
    assert not F.forward_ad_active(x, None)
    with fwAD.dual_level():
        d = fwAD.make_dual(x, torch.ones(3))
        assert F.forward_ad_active(x, d)
        assert not F.forward_ad_active(x, None)
