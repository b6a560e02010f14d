"""The no-grad forward of the model-shell entry (``b200rnn_forward_fused`` without SAVE_FOR_BACKWARD, the frozen
audio encoder of the fuse step) runs the GRU-256 8-row recurrence on fp16 pairs (rec_fwd_h16_kernel, ``f16x3``); the
module forward keeps 3xTF32 (``tc8``).

Against the float64 oracle (oracle/rnn_numpy.py) at T = 120: per-step outputs within 1e-5, and no more than 1.25 x the
error of the 3xTF32 module path on the same inputs; the pooled LayerNorm + GRU + time-sum features within 1e-4. Runs are
bitwise deterministic, CUDA-graph replays equal the eager call, and an in-place weight edit reaches the next call (the
split is made per launch, nothing is cached)."""
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
H16_LINE = "[b200rnn] fwd cfg tc8 C=4 BS=8 mma.sync f16x3"
TC8_LINE = "[b200rnn] fwd cfg tc8 C=4 BS=8 mma.sync 3xTF32"


def _gru(seed=0):
    import b200rnn

    torch.manual_seed(seed)
    return b200rnn.GRU(256, 256, num_layers=2).to(DEV)


def _fused(gru, x_tm, lengths=None):
    """y [T,B,256] of b200rnn_forward_fused without SAVE_FOR_BACKWARD (lengths: PackedSequence semantics)"""
    from b200rnn import _lib
    from b200rnn.functional import _make_desc, _stream_ptr

    lib = _lib.load()
    T, B, _ = x_tm.shape
    desc = _make_desc(gru._config(), B, T, False)
    _, sbytes = _lib.workspace_bytes(desc)
    scratch = torch.empty(sbytes, dtype=torch.uint8, device=DEV)
    y = torch.empty(T, B, 256, device=DEV)
    h_n = torch.empty(2, B, 256, device=DEV)
    params = _lib.ptr_array([w.data_ptr() for w in gru._flat_weights])
    lens = lengths.to(DEV, torch.int32).contiguous() if lengths is not None else None
    rc = lib.b200rnn_forward_fused(ctypes.byref(desc), x_tm.data_ptr(), x_tm.stride(0), x_tm.stride(1), params,
                                   y.data_ptr(), B * 256, 256, h_n.data_ptr(), None, None, scratch.data_ptr(), 0, 0,
                                   None, None, None, 0.0, None, lens.data_ptr() if lens is not None else None, None,
                                   None, _stream_ptr(DEV))
    _lib.check(rc, "b200rnn_forward_fused")
    return y, h_n


def _oracle(gru, x_tm, lengths=None):
    from oracle.rnn_numpy import NumpyRNN

    w = [p.detach().double().cpu().numpy() for p in gru._flat_weights]
    y, h = NumpyRNN("gru", w, 2, False).forward(x_tm.double().cpu().numpy(),
                                                None if lengths is None else lengths.numpy())
    return y, h


@pytest.mark.parametrize("B, ragged", [(128, False), (128, True), (160, False)], ids=["b128", "b128_ragged", "b160"])
def test_fused_forward_matches_fp64_t120(B, ragged):
    from b200rnn.functional import rnn_forward

    T = 120
    gru = _gru()
    g = torch.Generator().manual_seed(B + ragged)
    x = torch.randn(T, B, 256, generator=g)
    lens = None
    if ragged:
        lens = torch.randint(1, T + 1, (B,), generator=g)
        lens[B // 3] = T
    x_d = x.to(DEV)
    with torch.no_grad():
        y, h_n = _fused(gru, x_d, lens)
        y_tc8, h_tc8 = rnn_forward(x_d, gru._flat_weights, gru._config(), lengths=lens)  # the module path: 3xTF32
    torch.cuda.synchronize()
    y64, h64 = _oracle(gru, x, lens)
    err = max(np.abs(y.cpu().double().numpy() - y64).max(), np.abs(h_n.cpu().double().numpy() - h64).max())
    err_tc8 = max(np.abs(y_tc8.cpu().double().numpy() - y64).max(), np.abs(h_tc8.cpu().double().numpy() - h64).max())
    print(f"B={B} ragged={ragged}: max |y - y64| f16x3 {err:.3e}, 3xTF32 {err_tc8:.3e}")
    assert err < 1e-5
    assert err <= 1.25 * err_tc8, (err, err_tc8)
    if ragged:  # past its length a row emits exact zeros
        for b in range(B):
            if lens[b] < T:
                assert y[lens[b]:, b].abs().max().item() == 0


def test_pooled_features_match_fp64():
    """forward_ln_sum, the fuse step's audio branch: LayerNorm prologue, streamed projection, time sum"""
    T, B = 120, 128
    gru = _gru(1)
    ln = torch.nn.LayerNorm(256).to(DEV)
    with torch.no_grad():
        ln.weight.uniform_(0.5, 1.5)
        ln.bias.uniform_(-0.2, 0.2)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(T, B, 256, generator=g)
    with torch.no_grad():
        pooled = gru.forward_ln_sum(x.to(DEV), ln)
    torch.cuda.synchronize()
    xd = x.double()
    xn = torch.nn.functional.layer_norm(xd, (256,), ln.weight.detach().cpu().double(), ln.bias.detach().cpu().double(),
                                        ln.eps)
    y64, _ = _oracle(gru, xn)
    err = np.abs(pooled.cpu().double().numpy() - y64.sum(axis=0)).max()
    print(f"pooled: max |p - p64| {err:.3e}")
    assert err < 1e-4


def test_deterministic_graph_replays_and_weight_edits():
    from b200rnn.functional import rnn_forward_fused

    T, B = 120, 128
    gru = _gru(2)
    x = torch.randn(T, B, 256, device=DEV)
    with torch.no_grad():
        a = rnn_forward_fused(x, gru._flat_weights, gru._config())[0]
        b = rnn_forward_fused(x, gru._flat_weights, gru._config())[0]
        assert torch.equal(a, b)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            rnn_forward_fused(x, gru._flat_weights, gru._config())
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            static = rnn_forward_fused(x, gru._flat_weights, gru._config())[0]
        for i in range(50):
            xi = torch.randn_like(x)
            x.copy_(xi)
            graph.replay()
            eager = rnn_forward_fused(xi, gru._flat_weights, gru._config())[0]
            torch.cuda.synchronize()
            assert torch.equal(static, eager), f"replay {i}"
        # an in-place edit of weight_hh reaches the next call: the same result as a fresh copy of the edited weights
        before = rnn_forward_fused(x, gru._flat_weights, gru._config())[0]
        gru.weight_hh_l0.mul_(0.5)
        after = rnn_forward_fused(x, gru._flat_weights, gru._config())[0]
        fresh = [w.clone() for w in gru._flat_weights]
        ref = rnn_forward_fused(x, fresh, gru._config())[0]
        assert not torch.equal(before, after)
        assert torch.equal(after, ref)


_CHILD = """
import sys
sys.path[:0] = [{root!r}, {pkg!r}]
import torch, b200rnn
from b200rnn.functional import rnn_forward_fused
torch.manual_seed(0)
gru = b200rnn.GRU(256, 256, num_layers=2).to("cuda:0")
for B, path in ((128, "fused"), (128, "module"), (160, "fused"), (160, "module"), (128, "train")):
    x = torch.randn(16, B, 256, device="cuda:0", requires_grad=path == "train")
    if path == "train":
        gru(x)[0].sum().backward()
    else:
        with torch.no_grad():
            rnn_forward_fused(x, gru._flat_weights, gru._config()) if path == "fused" else gru(x)
    torch.cuda.synchronize()
    print("[b200rnn] ran", path, B, file=sys.stderr, flush=True)
"""


def test_debug_line_names_the_contraction_of_each_path():
    env = dict(os.environ, B200RNN_DEBUG="1")
    code = _CHILD.format(root=ROOT, pkg=os.path.join(ROOT, "icassp2022-depression_b200"))
    proc = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert proc.returncode == 0, proc.stdout + proc.stderr
    ran, seen = [], []
    for ln in proc.stderr.splitlines():
        if ln.startswith("[b200rnn] fwd cfg"):
            seen.append(ln.split(":")[0])
        elif ln.startswith("[b200rnn] ran"):
            ran.append((ln.split()[2], seen[-1] if seen else None, set(seen)))
            seen = []
    assert [r[:2] for r in ran] == [("fused", H16_LINE), ("module", TC8_LINE), ("fused", H16_LINE),
                                    ("module", TC8_LINE), ("train", TC8_LINE)], proc.stderr
    for path, _, cfgs in ran:   # every layer of a call runs the same contraction
        assert (H16_LINE in cfgs) == (path == "fused"), (path, cfgs)
