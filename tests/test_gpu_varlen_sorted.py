"""Ragged batches with skewed lengths: the recurrence kernels put the rows into batch slots sorted by descending length
and run each cluster only for its longest sequence (rnn_kernels.cuh, RecFwdParams::order). The skipped steps must look
exactly like masked ones: zero outputs, zero gradients, states and gradients as stock torch computes them.

Oracle: stock torch.nn.GRU / LSTM on CPU fed the same PackedSequence (enforce_sorted=False). Tolerances as
tests/test_gpu_varlen.py: outputs and states 1e-5 absolute, gradients 1e-4 relative to the largest entry. The GRU-256 batch
sizes reach each forward config of a unidirectional layer (B = 16: bs2, 64: bs4, 128: tc8, checked in a child process
with B200RNN_DEBUG, which is read once per process)."""
import os
import subprocess
import sys

import pytest
import torch
from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT_TOL = 1e-5
GRAD_RTOL = 1e-4


def _lengths(B, T, skew, seed=0):
    """one_long: every row short but one, in the middle of the batch, at T; rising: lengths grow with the row index, so
    the slot order reverses the rows"""
    g = torch.Generator().manual_seed(seed)
    if skew == "one_long":
        lens = torch.randint(1, max(2, T // 4) + 1, (B,), generator=g)
        lens[B // 2] = T
    else:
        lens = 1 + (torch.arange(B) * (T - 1)) // max(B - 1, 1)
    return lens


def _models(kind, I, H, L, bi, seed=0):
    import b200rnn

    torch.manual_seed(seed)
    cls = torch.nn.GRU if kind == "gru" else torch.nn.LSTM
    ref = cls(I, H, num_layers=L, bidirectional=bi, batch_first=True)
    return ref, b200rnn.from_torch(ref).to(DEV)


def _states(out):
    return out[1] if isinstance(out[1], tuple) else (out[1],)


def _run(model, x, lens, wy, ws, dev):
    """padded output, states, dx and parameter gradients of sum(y * wy) + sum(state * ws) for a packed batch"""
    model.zero_grad()
    xx = x.clone().to(dev).requires_grad_(True)
    out = model(pack_padded_sequence(xx, lens, batch_first=True, enforce_sorted=False))
    y = pad_packed_sequence(out[0], batch_first=True, total_length=x.shape[1])[0]
    loss = (y * wy.to(dev)).sum()
    for s, w in zip(_states(out), ws):
        loss = loss + (s * w.to(dev)).sum()
    loss.backward()
    return (y.detach().cpu(), [s.detach().cpu() for s in _states(out)], xx.grad.cpu(),
            [p.grad.cpu() for p in model.parameters()])


def _check_against_torch(kind, B, T, I, H, L, bi, skew):
    ref, mine = _models(kind, I, H, L, bi)
    g = torch.Generator().manual_seed(11)
    lens = _lengths(B, T, skew)
    x = torch.randn(B, T, I, generator=g)
    D = 2 if bi else 1
    wy = torch.randn(B, T, D * H, generator=g)
    ws = [torch.randn(L * D, B, H, generator=g) for _ in range(1 if kind == "gru" else 2)]
    y_r, s_r, dx_r, gp_r = _run(ref, x, lens, wy, ws, "cpu")
    y_m, s_m, dx_m, gp_m = _run(mine, x, lens, wy, ws, DEV)
    assert (y_m - y_r).abs().max().item() <= OUT_TOL
    for a, b in zip(s_m, s_r):
        assert (a - b).abs().max().item() <= OUT_TOL
    assert ((dx_m - dx_r).abs().max() / dx_r.abs().max()).item() <= GRAD_RTOL
    for (n, _), a, b in zip(ref.named_parameters(), gp_m, gp_r):
        assert ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item() <= GRAD_RTOL, n


CASES = [
    # kind, B, T, I, H, L, bidirectional
    ("gru", 16, 48, 256, 256, 2, False),    # bs2
    ("gru", 64, 48, 256, 256, 2, False),    # bs4 (batch-paired)
    ("gru", 128, 48, 256, 256, 2, False),   # tc8 (tensor cores)
    ("gru", 16, 48, 256, 256, 1, True),
    ("lstm", 16, 30, 64, 128, 1, False),
    ("lstm", 64, 30, 256, 128, 2, True),
    ("lstm", 64, 30, 256, 256, 2, True),    # the text BiLSTM's hidden size
]


@pytest.mark.parametrize("skew", ["one_long", "rising"])
@pytest.mark.parametrize("kind,B,T,I,H,L,bi", CASES)
def test_skewed_packed_batch_matches_torch_cpu(kind, B, T, I, H, L, bi, skew):
    _check_against_torch(kind, B, T, I, H, L, bi, skew)


_CHILD = """
import sys
sys.path[:0] = [{root!r}, {pkg!r}]
import torch, b200rnn
from torch.nn.utils.rnn import pack_padded_sequence
torch.manual_seed(0)
gru = b200rnn.from_torch(torch.nn.GRU(256, 256, batch_first=True)).to("cuda:0")
for B in (16, 64, 128):
    lens = torch.randint(1, 9, (B,))
    lens[B // 2] = 8
    x = torch.randn(B, 8, 256, device="cuda:0")
    with torch.no_grad():
        gru(pack_padded_sequence(x, lens, batch_first=True, enforce_sorted=False))
    torch.cuda.synchronize()
    print("[b200rnn] ran B=%d" % B, file=sys.stderr, flush=True)
"""


def test_gru256_batch_sizes_reach_each_forward_config():
    env = dict(os.environ, B200RNN_DEBUG="1")
    code = _CHILD.format(root=ROOT, pkg=os.path.join(ROOT, "icassp2022-depression_b200"))
    proc = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert proc.returncode == 0, proc.stdout + proc.stderr
    # the last config line before each "ran" line is the config that ran
    ran, last = [], None
    for ln in proc.stderr.splitlines():
        if ln.startswith("[b200rnn] fwd cfg"):
            last = ln.split(":")[0]
        elif ln.startswith("[b200rnn] ran"):
            ran.append(last)
    assert ran == ["[b200rnn] fwd cfg C=4 BS=2 KL=16 UPL=8 RG=0 PB=0", "[b200rnn] fwd cfg C=4 BS=4 KL=16 UPL=4 RG=1 PB=1",
                   "[b200rnn] fwd cfg tc8 C=4 BS=8 mma.sync 3xTF32"], proc.stderr


def test_padding_garbage_reaches_nothing_tc8():
    """B = 128 (tc8): values past each length of 1e3 * randn change no output, state or gradient by a single bit, and
    the padded output and dx rows are exactly 0."""
    B, T, I, H = 128, 40, 256, 256
    _, mine = _models("gru", I, H, 2, False)
    g = torch.Generator().manual_seed(5)
    lens = _lengths(B, T, "one_long", seed=5)
    x = torch.randn(B, T, I, generator=g)
    for b in range(B):
        x[b, lens[b]:] = 0.0
    x2 = x.clone()
    for b in range(B):
        x2[b, lens[b]:] = 1e3 * torch.randn(T - int(lens[b]), I, generator=g)
    wy, ws = torch.randn(B, T, H, generator=g), [torch.randn(2, B, H, generator=g)]
    r1 = _run(mine, x, lens, wy, ws, DEV)
    r2 = _run(mine, x2, lens, wy, ws, DEV)
    assert torch.equal(r1[0], r2[0]) and torch.equal(r1[2], r2[2])
    for a, b in zip(r1[1] + r1[3], r2[1] + r2[3]):
        assert torch.equal(a, b)
    y, _, dx, _ = r1
    for b in range(B):
        if lens[b] < T:
            assert y[b, lens[b]:].abs().max().item() == 0 and dx[b, lens[b]:].abs().max().item() == 0


@pytest.mark.parametrize("kind,bi", [("gru", False), ("lstm", True)])
def test_rows_do_not_depend_on_batch_order_or_neighbours(kind, bi):
    """The same sequences (distinct lengths) in another batch order sort into the same slots: h_n and every per-row
    result are bit-identical after un-permuting. With extra shorter rows appended they keep their slots too; the
    results then agree within tolerance (another batch size may take another config)."""
    B, T, I, H = 48, 64, 128, 256
    _, mine = _models(kind, I, H, 2, bi)
    D = 2 if bi else 1
    g = torch.Generator().manual_seed(7)
    lens = torch.randperm(T - 1, generator=g)[:B] + 2    # distinct, in [2, T]
    x = torch.randn(B, T, I, generator=g)
    for b in range(B):
        x[b, lens[b]:] = 0.0
    wy = torch.randn(B, T, D * H, generator=g)
    ws = [torch.randn(2 * D, B, H, generator=g) for _ in range(1 if kind == "gru" else 2)]
    base = _run(mine, x, lens, wy, ws, DEV)

    perm = torch.randperm(B, generator=g)
    inv = torch.argsort(perm)
    pr = _run(mine, x[perm], lens[perm], wy[perm], [w[:, perm] for w in ws], DEV)
    assert torch.equal(pr[0][inv], base[0])
    for a, b in zip(pr[1], base[1]):
        assert torch.equal(a[:, inv], b)
    assert torch.equal(pr[2][inv], base[2])

    E = 8   # extra rows of length 1, shorter than every original one
    lens_x = torch.cat([lens, torch.ones(E, dtype=lens.dtype)])
    x_x = torch.cat([x, torch.randn(E, T, I, generator=g)])
    for b in range(B, B + E):
        x_x[b, 1:] = 0.0
    wy_x = torch.cat([wy, torch.randn(E, T, D * H, generator=g)])
    ws_x = [torch.cat([w, torch.randn(2 * D, E, H, generator=g)], dim=1) for w in ws]
    ex = _run(mine, x_x, lens_x, wy_x, ws_x, DEV)
    assert (ex[0][:B] - base[0]).abs().max().item() <= OUT_TOL
    for a, b in zip(ex[1], base[1]):
        assert (a[:, :B] - b).abs().max().item() <= OUT_TOL
    assert ((ex[2][:B] - base[2]).abs().max() / base[2].abs().max()).item() <= GRAD_RTOL


def test_packed_runs_are_bitwise_deterministic():
    for kind, B, T, I, H, bi in (("gru", 128, 60, 256, 256, False), ("lstm", 64, 30, 256, 256, True)):
        _, mine = _models(kind, I, H, 2, bi)
        g = torch.Generator().manual_seed(13)
        lens = _lengths(B, T, "one_long", seed=13)
        x = torch.randn(B, T, I, generator=g)
        D = 2 if bi else 1
        wy = torch.randn(B, T, D * H, generator=g)
        ws = [torch.randn(2 * D, B, H, generator=g) for _ in range(1 if kind == "gru" else 2)]
        r1 = _run(mine, x, lens, wy, ws, DEV)
        r2 = _run(mine, x, lens, wy, ws, DEV)
        assert torch.equal(r1[0], r2[0]) and torch.equal(r1[2], r2[2]), kind
        for a, b in zip(r1[1] + r1[3], r2[1] + r2[3]):
            assert torch.equal(a, b), kind


@pytest.mark.parametrize("kind,B,bi", [("gru", 128, False), ("lstm", 64, True)])
def test_full_length_packed_batch_matches_dense(kind, B, bi):
    """lengths == T for every row (non-increasing, so the slot order is the identity): the packed run matches the dense
    run of the same rows."""
    import b200rnn

    T, I, H = 30, 256, 256
    torch.manual_seed(3)
    cls = b200rnn.GRU if kind == "gru" else b200rnn.LSTM
    mine = cls(I, H, num_layers=2, bidirectional=bi, batch_first=True).to(DEV)
    x = torch.randn(B, T, I, device=DEV)
    with torch.no_grad():
        dense = mine(x)
        packed = mine(pack_padded_sequence(x, torch.full((B,), T), batch_first=True))
    y = pad_packed_sequence(packed[0], batch_first=True)[0]
    assert (y - dense[0]).abs().max().item() <= 1e-6
    for a, b in zip(_states(packed), _states(dense)):
        assert (a - b).abs().max().item() <= 1e-6
