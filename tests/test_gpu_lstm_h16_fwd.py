"""The no-grad forward of the model-shell entry (``b200rnn_forward_fused`` without SAVE_FOR_BACKWARD, the frozen text
BiLSTM of the fuse step) runs the LSTM-128 recurrence on fp16 pairs (lstm_fwd_h16_kernel, ``tcl8``: 2-CTA clusters of
8 batch rows); the module forward keeps the scalar FFMA kernels.

Against the float64 oracle (oracle/rnn_numpy.py), bidirectional and two layers at T = 30: per-step outputs and the final
h and c within 1e-5, and no more than 1.25 x the error of the FFMA module path on the same inputs, at B = 128, ragged,
and at a batch that needs more than one wave of clusters. Runs are bitwise deterministic, CUDA-graph replays equal the
eager call, and an in-place weight edit reaches the next call."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TCL8_LINE = "[b200rnn] fwd cfg tcl8 C=2 BS=8 mma.sync f16x3"
T, I, H = 30, 1024, 128


def _lstm(seed=0):
    import b200rnn

    torch.manual_seed(seed)
    return b200rnn.LSTM(I, H, num_layers=2, bidirectional=True).to(DEV)


def _fused(lstm, x_tm, lengths=None):
    """y [T,B,2H], h_n, c_n [4,B,H] of b200rnn_forward_fused without SAVE_FOR_BACKWARD (lengths: PackedSequence
    semantics)"""
    from b200rnn import _lib
    from b200rnn.functional import _make_desc, _stream_ptr

    lib = _lib.load()
    T_, B, _ = x_tm.shape
    desc = _make_desc(lstm._config(), B, T_, False)
    _, sbytes = _lib.workspace_bytes(desc)
    scratch = torch.empty(sbytes, dtype=torch.uint8, device=DEV)
    y = torch.empty(T_, B, 2 * H, device=DEV)
    h_n = torch.empty(4, B, H, device=DEV)
    c_n = torch.empty(4, B, H, device=DEV)
    params = _lib.ptr_array([w.data_ptr() for w in lstm._flat_weights])
    lens = lengths.to(DEV, torch.int32).contiguous() if lengths is not None else None
    rc = lib.b200rnn_forward_fused(ctypes.byref(desc), x_tm.data_ptr(), x_tm.stride(0), x_tm.stride(1), params,
                                   y.data_ptr(), B * 2 * H, 2 * H, h_n.data_ptr(), c_n.data_ptr(), None,
                                   scratch.data_ptr(), 0, 0, None, None, None, 0.0, None,
                                   lens.data_ptr() if lens is not None else None, None, None, _stream_ptr(DEV))
    _lib.check(rc, "b200rnn_forward_fused")
    return y, h_n, c_n


def _oracle(lstm, x_tm, lengths=None):
    from oracle.rnn_numpy import NumpyRNN

    w = [p.detach().double().cpu().numpy() for p in lstm._flat_weights]
    return NumpyRNN("lstm", w, 2, True).forward(x_tm.double().cpu().numpy(),
                                                None if lengths is None else lengths.numpy())


def _err(outs, refs):
    return max(np.abs(o.cpu().double().numpy() - r).max() for o, r in zip(outs, refs))


# B = 300: 38 slices x 2 directions = 76 clusters, more than the 66 two-CTA cluster slots of a 132-SM card
@pytest.mark.parametrize("B, ragged", [(128, False), (128, True), (300, False)], ids=["b128", "b128_ragged", "b300"])
def test_fused_forward_matches_fp64_t30(B, ragged):
    from b200rnn.functional import rnn_forward

    lstm = _lstm()
    g = torch.Generator().manual_seed(B + ragged)
    x = torch.randn(T, B, I, generator=g)
    lens = None
    if ragged:
        lens = torch.randint(1, T + 1, (B,), generator=g)
        lens[B // 3] = T
    x_d = x.to(DEV)
    with torch.no_grad():
        out = _fused(lstm, x_d, lens)
        ref = rnn_forward(x_d, lstm._flat_weights, lstm._config(), lengths=lens)  # the module path: FFMA
    torch.cuda.synchronize()
    o64 = _oracle(lstm, x, lens)
    err = _err(out, o64)
    err_ffma = _err(ref[:3], o64)
    print(f"B={B} ragged={ragged}: max |y - y64| f16x3 {err:.3e}, FFMA {err_ffma:.3e}")
    assert err < 1e-5
    assert err <= 1.25 * err_ffma, (err, err_ffma)
    if ragged:  # past its length a row emits exact zeros
        y = out[0]
        for b in range(B):
            if lens[b] < T:
                assert y[lens[b]:, b].abs().max().item() == 0


def test_deterministic_graph_replays_and_weight_edits():
    from b200rnn.functional import rnn_forward_fused

    B = 128
    lstm = _lstm(2)
    x = torch.randn(T, B, I, device=DEV)
    with torch.no_grad():
        a = rnn_forward_fused(x, lstm._flat_weights, lstm._config())
        b = rnn_forward_fused(x, lstm._flat_weights, lstm._config())
        assert all(torch.equal(u, v) for u, v in zip(a, b))
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            rnn_forward_fused(x, lstm._flat_weights, lstm._config())
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            static = rnn_forward_fused(x, lstm._flat_weights, lstm._config())[0]
        for i in range(20):
            xi = torch.randn_like(x)
            x.copy_(xi)
            graph.replay()
            eager = rnn_forward_fused(xi, lstm._flat_weights, lstm._config())[0]
            torch.cuda.synchronize()
            assert torch.equal(static, eager), f"replay {i}"
        # an in-place edit of weight_hh reaches the next call: the same result as a fresh copy of the edited weights
        before = rnn_forward_fused(x, lstm._flat_weights, lstm._config())[0]
        lstm.weight_hh_l0_reverse.mul_(0.5)
        after = rnn_forward_fused(x, lstm._flat_weights, lstm._config())[0]
        fresh = [w.clone() for w in lstm._flat_weights]
        ref = rnn_forward_fused(x, fresh, lstm._config())[0]
        assert not torch.equal(before, after)
        assert torch.equal(after, ref)


_CHILD = """
import sys
sys.path[:0] = [{root!r}, {pkg!r}]
import torch, b200rnn
from b200rnn.functional import rnn_forward_fused
torch.manual_seed(0)
lstm = b200rnn.LSTM(64, 128, num_layers=2, bidirectional=True).to("cuda:0")
for path in ("fused", "module", "train"):
    x = torch.randn(8, 24, 64, device="cuda:0", requires_grad=path == "train")
    if path == "train":
        lstm(x)[0].sum().backward()
    else:
        with torch.no_grad():
            rnn_forward_fused(x, lstm._flat_weights, lstm._config()) if path == "fused" else lstm(x)
    torch.cuda.synchronize()
    print("[b200rnn] ran", path, file=sys.stderr, flush=True)
"""


def test_debug_line_names_the_fp16_pair_config_on_the_fused_path_only():
    env = dict(os.environ, B200RNN_DEBUG="1")
    code = _CHILD.format(root=ROOT, pkg=os.path.join(ROOT, "icassp2022-depression_b200"))
    proc = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert proc.returncode == 0, proc.stdout + proc.stderr
    ran, seen = [], []
    for ln in proc.stderr.splitlines():
        if ln.startswith("[b200rnn] fwd cfg"):
            seen.append(ln.split(":")[0])
        elif ln.startswith("[b200rnn] ran"):
            ran.append((ln.split()[2], set(seen)))
            seen = []
    assert [r[0] for r in ran] == ["fused", "module", "train"], proc.stderr
    for path, cfgs in ran:   # every layer of the fused call runs the fp16-pair config, no layer of the others does
        assert cfgs == {TCL8_LINE} if path == "fused" else (cfgs and TCL8_LINE not in cfgs), (path, cfgs)
