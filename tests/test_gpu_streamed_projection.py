"""Streamed input projection: for a unidirectional layer whose recurrence fits one wave on at most half of the SMs, the
layer's x-projection GEMM publishes a ready counter per 128-row tile and the recurrence starts while the GEMM still
runs, waiting per step for the tiles it reads (csrc/api.cu, DESIGN.md §4). The arithmetic is that of the serial order,
so results match stock torch at the usual thresholds, and a CUDA graph replays bit for bit what an eager call computes
(counters that were not reset, or a step read before its tile was published, would show as a difference).

B200RNN_DEBUG prints one "[b200rnn] streamed x-projection" line per streamed GEMM and is read once per process, so the
dispatch checks run in child processes."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STREAMED = "[b200rnn] streamed x-projection"


def _gru_errors(B, T, ragged, seed=11):
    """max |y - y_ref|, |h_n - h_n_ref|; max |dx - dx_ref| / max |dx_ref|; max |dW - dW_ref| / max |dW_ref|"""
    import b200rnn

    torch.manual_seed(seed)
    ref = torch.nn.GRU(256, 256, num_layers=2, batch_first=True)
    mine = b200rnn.from_torch(ref).to(DEV)
    x = torch.randn(B, T, 256)
    lens = torch.randint(1, T + 1, (B,)) if ragged else torch.full((B,), T)
    lens[0] = T
    xr = x.clone().requires_grad_(True)
    xm = x.to(DEV).requires_grad_(True)
    outs = []
    for model, inp in ((ref, xr), (mine, xm)):
        if ragged:
            pk = torch.nn.utils.rnn.pack_padded_sequence(inp, lens, batch_first=True, enforce_sorted=False)
            y, h = model(pk)
            y = torch.nn.utils.rnn.pad_packed_sequence(y, batch_first=True, total_length=T)[0]
        else:
            y, h = model(inp)
        outs.append((y, h))
    (yr, hr), (ym, hm) = outs
    wy = torch.randn(B, T, 256)
    wh = torch.randn_like(hr)
    ((yr * wy).sum() + (hr * wh).sum()).backward()
    ((ym * wy.to(DEV)).sum() + (hm * wh.to(DEV)).sum()).backward()
    torch.cuda.synchronize()
    err_y = max((ym.detach().cpu() - yr.detach()).abs().max().item(), (hm.detach().cpu() - hr.detach()).abs().max().item())
    err_dx = ((xm.grad.cpu() - xr.grad).abs().max() / xr.grad.abs().max()).item()
    g_ref = torch.cat([p.grad.reshape(-1) for p in ref.parameters()])
    g_mine = torch.cat([p.grad.reshape(-1).cpu() for p in mine.parameters()])
    err_g = ((g_mine - g_ref).abs().max() / g_ref.abs().max()).item()
    return err_y, err_dx, err_g


@pytest.mark.parametrize("B, ragged", [(128, False), (128, True), (64, False)], ids=["b128", "b128_ragged", "c2_b64"])
def test_streamed_gru_matches_torch_t120(B, ragged):
    # B = 128: the benchmark's audio GRU (tc8); B = 64: the c2 training shape (bs4), whose recurrence overwrites the
    # gates the streamed GEMM wrote with the activated gates the backward reads
    err_y, err_dx, err_g = _gru_errors(B, 120, ragged)
    assert err_y < 1e-5, err_y
    assert err_dx < 1e-4 and err_g < 1e-4, (err_dx, err_g)


def test_graph_replays_match_eager_bitwise():
    import b200rnn

    torch.manual_seed(3)
    B, T = 128, 120
    mine = b200rnn.from_torch(torch.nn.GRU(256, 256, num_layers=2, batch_first=True)).to(DEV).eval()
    static_x = torch.randn(B, T, 256, device=DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.no_grad(), torch.cuda.stream(side):
        for _ in range(3):
            mine(static_x)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.no_grad(), torch.cuda.graph(graph):
        static_y, static_h = mine(static_x)
    for i in range(50):
        x = torch.randn(B, T, 256, device=DEV)
        static_x.copy_(x)
        graph.replay()
        with torch.no_grad():
            y, h = mine(x)
        torch.cuda.synchronize()
        assert torch.equal(static_y, y) and torch.equal(static_h, h), f"replay {i} differs from the eager call"


_CHILD = """
import sys
sys.path[:0] = [{root!r}, {pkg!r}]
import torch, b200rnn
torch.manual_seed(0)
kind, B, T = {kind!r}, {B}, {T}
if kind == "gru":
    ref = torch.nn.GRU(256, 256, num_layers=2, batch_first=True)
    x = torch.randn(B, T, 256, device="cuda:0")
else:
    ref = torch.nn.LSTM(1024, 256, num_layers=2, bidirectional=True, batch_first=True)
    x = torch.randn(B, T, 1024, device="cuda:0")
mine = b200rnn.from_torch(ref).to("cuda:0")
with torch.no_grad():
    mine(x)
torch.cuda.synchronize()
print("DONE", flush=True)
"""


def _streamed_lines(kind, B, T):
    code = _CHILD.format(root=ROOT, pkg=os.path.join(ROOT, "icassp2022-depression_b200"), kind=kind, B=B, T=T)
    proc = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, B200RNN_DEBUG="1"), capture_output=True,
                          text=True, timeout=600)
    assert proc.returncode == 0 and "DONE" in proc.stdout, proc.stdout + proc.stderr
    return [ln for ln in proc.stderr.splitlines() if ln.startswith(STREAMED)], proc.stderr


@pytest.mark.parametrize("kind, B, T, n_streamed", [("gru", 128, 120, 2), ("gru", 160, 120, 0), ("lstm", 64, 30, 0)],
                         ids=["gru_b128_streams", "gru_b160_serial", "bilstm_serial"])
def test_which_shapes_stream(kind, B, T, n_streamed):
    # B = 160 takes tc8 on 80 SMs (more than half of the card) and a bidirectional layer walks t both ways: both keep
    # GEMM and recurrence one after the other
    lines, err = _streamed_lines(kind, B, T)
    assert len(lines) == n_streamed, err
